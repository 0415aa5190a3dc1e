"""Joins the static step trace (tools/trace_step.py: shapes, FLOPs, bytes of every convolution launch, program order) with
an ncu launch list of the same step (a .csv.gz: measured duration of every kernel, launch order) and prints, per
convolution class (kind, shape), launches, measured time, roofline time and their ratio. The launch list starts somewhere
inside a step, so the expected kernel-name sequence is rotated onto the observed one first.

    python -O tools/conv_classes.py launches.csv.gz
    python -O tools/conv_classes.py gpurun_out/abi_launches.csv --abi gpurun_out/abi_calls.json

With --abi (the log tools/gpu_abi_log.py wrote in the SAME run as the launch list) nothing is guessed: the k-th b200seg
kernel of the list belongs to the ABI call whose cumulative launch count covers k.
"""
import collections
import csv
import gzip
import importlib.util
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, B = 1386.7e12, 6650e9


def load_trace():
    spec = importlib.util.spec_from_file_location("trace_step", os.path.join(ROOT, "tools", "trace_step.py"))
    ts = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ts)
    argv, sys.argv = sys.argv, ["trace_step.py"]
    stdout, sys.stdout = sys.stdout, open(os.devnull, "w")
    try:
        ts.main()
    finally:
        sys.stdout, sys.argv = stdout, argv
    exp = []        # (kernel name, kind, detail, flops, bytes) per expected tensor-core kernel launch
    for name, nbytes, flops, detail in ts.EVENTS:
        m = re.match(r"(\d+)x(\d+) c(\d+)->(\d+) k(\d) s(\d)", detail or "")
        if not m:
            continue
        h, w, cin, cout, k, s = map(int, m.groups())
        if name.startswith("conv2d_fwd"):
            halo = k == 3 and s == 1 and cout % 16 == 0 and cout != 19 and cout != 1
            exp.append(("conv3x3_halo_kernel" if halo else "conv_igemm_kernel", "fwd", detail, flops, nbytes))
        elif name == "conv2d_dgrad":
            if k == 3 and s == 1 and cin % 16 == 0:
                exp.append(("conv3x3_halo_kernel", "dgrad", detail, flops, nbytes))
            else:
                reps = 4 if (k == 3 and s == 2) else 1
                for _ in range(reps):
                    exp.append(("conv_igemm_kernel", "dgrad", detail, flops / reps, nbytes / reps))
        elif name == "conv2d_wgrad":
            exp.append(("wgrad_igemm_kernel", "wgrad", detail, flops, nbytes))
    return exp


def open_text(path):
    return gzip.open(path, "rt") if path.endswith(".gz") else open(path, "rt")


def join_with_abi_log(csv_path, abi_path):
    import json
    with open(abi_path) as f:
        log = json.load(f)
    rows = list(csv.reader(open_text(csv_path)))
    for i, r in enumerate(rows):
        if "Kernel Name" in r:
            hdr, start = r, i
            break
    ki, mi = hdr.index("Kernel Name"), hdr.index("Metric Value")
    dur = []
    for r in rows[start + 2:]:
        if len(r) > mi and "b200seg::" in r[ki]:
            try:
                dur.append(float(r[mi].replace(",", "")) / 1000.0)
            except ValueError:
                pass
    calls = log["calls"]
    total = sum(c[4] for c in calls)
    print("ABI log: %d calls, %d kernels; launch list: %d b200seg kernels" % (len(calls), total, len(dur)))
    if total != len(dur):
        print("COUNT MISMATCH: the two files are not from the same run (or a launch count passed to check() is wrong)")
    first = log["step_starts"][-1]           # the last logged step (allocator warm, kernels loaded)
    k = sum(c[4] for c in calls[:first])
    agg, per_entry = collections.OrderedDict(), collections.OrderedDict()
    for name, detail, flops, nbytes, launches in calls[first:]:
        t = sum(dur[k:k + launches])
        k += launches
        if launches == 0:
            continue
        roof = max(flops / P, nbytes / B) * 1e6
        for key, table in (((name, detail), agg), ((name, ""), per_entry)):
            a = table.setdefault(key, [0, 0, 0.0, 0.0])
            a[0] += 1; a[1] += launches; a[2] += t; a[3] += roof
    for title, table in (("per entry point", per_entry), ("per convolution class", agg)):
        print("\n%s\n%-18s %-30s %6s %8s %10s %10s %8s" % (title, "entry point", "shape", "calls", "kernels", "meas ms",
                                                         "roof ms", "ratio"))
        tot = [0.0, 0.0]
        for (name, detail), (c, l, t, rt) in sorted(table.items(), key=lambda kv: -kv[1][2]):
            if table is agg and not detail:
                continue
            print("%-18s %-30s %6d %8d %10.3f %10.3f %8.1f" % (name, detail, c, l, t / 1e3, rt / 1e3, t / max(rt, 1e-9)))
            tot[0] += t; tot[1] += rt
        print("%-18s %-30s %6s %8s %10.3f %10.3f %8.1f" % ("sum", "", "", "", tot[0] / 1e3, tot[1] / 1e3,
                                                          tot[0] / max(tot[1], 1e-9)))


def load_launches(path):
    rows = list(csv.reader(open_text(path)))
    for i, r in enumerate(rows):
        if "Kernel Name" in r:
            hdr, start = r, i
            break
    ki, mi = hdr.index("Kernel Name"), hdr.index("Metric Value")
    obs = []
    for r in rows[start + 2:]:
        if len(r) <= mi:
            continue
        try:
            v = float(r[mi].replace(",", ""))
        except ValueError:
            continue
        name = r[ki].split("(")[0].replace("b200seg::", "")
        if name in ("conv3x3_halo_kernel", "conv_igemm_kernel", "wgrad_igemm_kernel"):
            obs.append((name, v / 1000.0))          # us
    return obs


def main():
    if "--abi" in sys.argv:
        join_with_abi_log(sys.argv[1], sys.argv[sys.argv.index("--abi") + 1])
        return
    exp = load_trace()
    obs = load_launches(sys.argv[1])
    print("expected %d tensor-core launches per step, launch list holds %d" % (len(exp), len(obs)))
    n = len(exp)
    en = [e[0] for e in exp]
    on = [o[0] for o in obs]
    best = (-1, 0)
    for rot in range(n):
        m = sum(1 for i in range(min(n, len(on))) if en[(i + rot) % n] == on[i])
        if m > best[0]:
            best = (m, rot)
    m, rot = best
    print("best rotation %d: %d of %d kernel names agree" % (rot, m, min(n, len(on))))
    if m < 0.98 * min(n, len(on)):
        print("sequence mismatch: the launch list is from a different program version; classes below are unreliable")
    agg = collections.OrderedDict()
    for i in range(min(n, len(on))):
        name, kind, detail, flops, nbytes = exp[(i + rot) % n]
        if name != on[i]:
            continue
        a = agg.setdefault((kind, detail), [0, 0.0, 0.0])
        a[0] += 1
        a[1] += obs[i][1]
        a[2] += max(flops / P, nbytes / B) * 1e6
    print("%-6s %-30s %6s %10s %10s %8s %10s" % ("kind", "shape", "n", "meas ms", "roof ms", "ratio", "us/launch"))
    tot = [0, 0.0, 0.0]
    for (kind, detail), (c, t, rt) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-6s %-30s %6d %10.3f %10.3f %8.1f %10.1f" % (kind, detail, c, t / 1e3, rt / 1e3, t / max(rt, 1e-9), t / c))
        tot[0] += c; tot[1] += t; tot[2] += rt
    print("%-6s %-30s %6d %10.3f %10.3f %8.1f" % ("all", "", tot[0], tot[1] / 1e3, tot[2] / 1e3, tot[1] / tot[2]))


if __name__ == "__main__":
    main()
