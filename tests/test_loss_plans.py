"""Host-only check that the configuration table of tests/test_gpu_loss_classes.py covers every loss launch of the traced
training steps: every architecture under each criterion (CE, RMI, image-weighted CE with and without the binary16
rounding of its weights), the two-scale architectures with the supervised multi-scale terms, and RMI on the OCR
auxiliary head. The attention-head variants and deferred BatchNorm cells change no loss key (traced once, every key of
theirs is one of the default programs'), so they are not in the list. Keys come from tools/loss_classes.py, for the traced
launches from the recorded arguments (tools/trace_step.py LAUNCH_ARGS), for the table rows from the arguments they hand
to the C ABI."""
import ast
import functools
import os
import sys

import test_ew_plans as ew_plans
import test_gpu_loss_classes as rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import loss_classes  # noqa: E402
from b200seg import arch as A  # noqa: E402

CRITERIA = ("ce", "rmi", "img_wt:1.0", "img_wt:2.5:half")


def _programs():
    """tools/trace_step.py arguments of every training step whose loss launches the table must cover."""
    progs = []
    for arch in A.ARCHS:
        for crit in CRITERIA:
            progs.append(["--arch", arch, "--criterion", crit])
            if A.is_two_scale(arch):
                progs.append(["--arch", arch, "--criterion", crit, "--sup-wt", "0.05"])
        if A.has_ocr(arch):
            progs.append(["--arch", arch, "--criterion", "rmi", "--ocr-aux-rmi"])
            if A.is_two_scale(arch):
                progs.append(["--arch", arch, "--criterion", "rmi", "--ocr-aux-rmi", "--sup-wt", "0.05"])
    return progs


@functools.lru_cache(maxsize=None)
def _step_keys():
    return ew_plans.trace_keys(_programs(), "loss_classes")


def _row_keys():
    table = {}
    for row in rows.ROWS:
        table.setdefault(repr(loss_classes.launch_key(row[0], row[1])), []).append(rows.row_id(row))
    return table


def test_every_row_has_a_runner_and_a_key():
    for row in rows.ROWS:
        assert row[0] in rows.RUNNERS, row
        assert loss_classes.launch_key(row[0], row[1]) is not None, row


def test_loss_table_covers_every_launch_of_the_programs():
    """Every key of every loss launch of the programs has a row, and every entry point with a key has a runner."""
    progs = _programs()
    keys = _step_keys()
    print("\n%d programs, %d loss configuration keys, %d table rows" % (len(progs), len(keys), len(rows.ROWS)))
    assert {ast.literal_eval(k)[0] for k in keys} == set(loss_classes.LOSS_ENTRY_POINTS)
    table = _row_keys()
    missing = ["%s  (%s: %s)" % (k, prog, args) for k, (prog, args) in sorted(keys.items()) if k not in table]
    assert not missing, ("loss launch configurations without a row in tests/test_gpu_loss_classes.py:\n" +
                         "\n".join(missing))
    assert {ast.literal_eval(k)[0] for k in keys} <= set(rows.RUNNERS)
