"""Host-only check that the configuration table of tests/test_gpu_ew_classes.py covers every launch that is not a
tensor-core convolution in the traced programs: the training step of every architecture with and without deferred
BatchNorm cells, the attention-head variants, and the evaluation with its output assembly and scoring tail
(tools/trace_step.py --eval --assembly). Keys come from tools/ew_classes.py, for the traced launches from the recorded
arguments (LAUNCH_ARGS), for the table rows from the arguments they hand to the C ABI."""
import ast
import functools
import json
import os
import subprocess
import sys

import test_conv_plans as conv_plans
import test_gpu_ew_classes as rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ew_classes  # noqa: E402


def _programs():
    """conv_plans._programs() with the evaluation traced through its output assembly."""
    return [p + ["--assembly"] if "--eval" in p else p for p in conv_plans._programs()]


_TRACE = """import importlib, importlib.util, json, os, sys
sys.path.insert(0, %r)
classes = importlib.import_module(sys.argv[1])
spec = importlib.util.spec_from_file_location("trace_step", os.path.join(%r, "trace_step.py"))
ts = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ts)
sys.argv = ["trace_step.py"] + sys.argv[2:]
stdout, sys.stdout = sys.stdout, open(os.devnull, "w")
ts.main()
sys.stdout = stdout
keys = {}
for i, args in sorted(ts.LAUNCH_ARGS.items()):
    key = classes.launch_key(ts.EVENTS[i][0], args)
    if key is not None:
        keys.setdefault(repr(key), repr(args))
print(json.dumps(keys))
""" % ((os.path.join(ROOT, "tools"),) * 2)


def trace_keys(progs, key_module):
    """{repr(key): (program, repr(arguments of its first launch))} over the programs (argument lists of
    tools/trace_step.py), keyed by launch_key of tools/<key_module>.py; one process per program (trace_step runs with
    -O), as many at once as there are CPUs."""
    running, keys = [], {}

    def reap(proc, prog):
        out, err = proc.communicate(timeout=900)
        assert proc.returncode == 0, (prog, err[-2000:])
        for k, a in json.loads(out.strip().splitlines()[-1]).items():
            keys.setdefault(k, (" ".join(prog), a))
    for prog in progs:
        if len(running) >= (os.cpu_count() or 4):
            reap(*running.pop(0))
        running.append((subprocess.Popen([sys.executable, "-O", "-c", _TRACE, key_module] + prog,
                                         stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True), prog))
    while running:
        reap(*running.pop(0))
    return keys


@functools.lru_cache(maxsize=None)
def _step_keys():
    return trace_keys(_programs(), "ew_classes")


def _row_keys():
    table = {}
    for row in rows.ROWS:
        table.setdefault(repr(ew_classes.launch_key(row[0], row[1])), []).append(rows.row_id(row))
    return table


def test_every_row_has_a_runner_and_a_key():
    for row in rows.ROWS:
        assert row[0] in rows.RUNNERS, row
        assert ew_classes.launch_key(row[0], row[1]) is not None, row


def test_ew_table_covers_every_launch_of_the_programs():
    """Every key of every launch that is not OUT_OF_SCOPE has a row (launch_key raises for an entry point it does not
    know), and every entry point with a key has a runner."""
    keys = _step_keys()
    assert len(keys) > 100, len(keys)
    table = _row_keys()
    missing = ["%s  (%s: %s)" % (k, prog, args) for k, (prog, args) in sorted(keys.items()) if k not in table]
    assert not missing, ("launch configurations without a row in tests/test_gpu_ew_classes.py:\n" + "\n".join(missing))
    assert {ast.literal_eval(k)[0] for k in keys} <= set(rows.RUNNERS)
