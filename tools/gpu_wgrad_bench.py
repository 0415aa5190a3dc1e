"""Times every distinct weight-gradient launch (b200seg_conv2d_wgrad: wgrad_igemm_kernel, plus wgrad_reduce_kernel when the
plan splits the pixels) of the traced training step, one crop, and prints per shape the launches per step, the plan,
microseconds per launch, TFLOP/s and the share of the H100 SXM's dense bf16 data-sheet rate (989 TFLOP/s), then the
launch-weighted total per step. The shapes and counts come from tools/trace_step.py's recorder (meta tensors, no
device), run in a child `python -O`. Each shape is timed with CUDA events around a CUDA-graph replay of --launches
back-to-back launches on random bf16 inputs, after a warm-up replay; the median of --reps replays is kept. Inputs of the
smaller shapes stay in L2 across the replay, as they partly do in the step. The card's name, power limit and maximum SM
clock are read in the same run. B200SEG_LIB_VARIANT=<tag> times lib/libb200seg_<tag>.so (see b200seg/_lib.py).

    python tools/gpu_wgrad_bench.py [--arch ocrnet.HRNet_Mscale] [--height 1024 --width 2048] [--out wgrad.json]"""
import argparse
import collections
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

PEAK_TFLOPS = 989.0   # H100 SXM, dense bf16, data sheet (700 W)


def record_calls(arch, height, width, key):
    """Counter {key(name, args): calls per step} over the launching entry points of the traced step, for the calls whose
    key is not None (tools/trace_step.py's recorder: meta tensors, no device; run under python -O)."""
    spec = importlib.util.spec_from_file_location("trace_step", os.path.join(ROOT, "tools", "trace_step.py"))
    ts = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ts)
    seen = collections.Counter()
    base = ts.Recorder

    class KeyRecorder(base):
        def __getattr__(self, name):
            fake = base.__getattr__(self, name)
            if ts.QUERY.search(name):
                return fake

            def record(*args):
                k = key(name, args, ts.SIZES)
                if k is not None:
                    seen[k] += 1
                return fake(*args)
            return record

    ts.Recorder = KeyRecorder
    argv, sys.argv = sys.argv, ["trace_step.py", "--arch", arch, "--height", str(height), "--width", str(width),
                                "--bn-cells"]
    stdout, sys.stdout = sys.stdout, open(os.devnull, "w")
    try:
        ts.main()
    finally:
        sys.stdout, sys.argv = stdout, argv
    return seen


def trace_launches(arch, height, width):
    """[(ConvDesc field values, dy_ld, launches per step)] of the step's weight gradients (run under python -O)."""
    from b200seg import _lib

    def key(name, args, sizes):
        if name != "b200seg_conv2d_wgrad":
            return None
        d, dy_ld = args[0]._obj, args[3]
        return tuple(getattr(d, f) for f, _ in _lib.ConvDesc._fields_), dy_ld
    seen = record_calls(arch, height, width, key)
    return [(list(desc), dy_ld, n) for (desc, dy_ld), n in seen.items()]


def time_replay(launch, launches, reps):
    """Microseconds per launch: CUDA events around a CUDA-graph replay of `launches` back-to-back calls of launch(),
    after three eager calls and one warm-up replay; returns (median of `reps` replays, all replays)."""
    import torch
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            launch()
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1000.0 / launches)
    return sorted(times)[len(times) // 2], times


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        import torch
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="ocrnet.HRNet_Mscale")
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=20, help="launches per CUDA-graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per shape (the median is kept)")
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    ap.add_argument("--trace-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.trace_only:
        if __debug__:
            sys.exit("--trace-only runs under python -O (the wrappers assert is_cuda)")
        print(json.dumps(trace_launches(args.arch, args.height, args.width)))
        return

    out = subprocess.run([sys.executable, "-O", os.path.abspath(__file__), "--trace-only", "--arch", args.arch,
                          "--height", str(args.height), "--width", str(args.width)],
                         capture_output=True, text=True, check=True).stdout
    shapes = json.loads(out.strip().splitlines()[-1])

    import torch
    from b200seg import _lib
    from b200seg._lib import ptr, stream_ptr
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    L = _lib.lib()
    name, power, sm_clock = card()
    print("%s, power limit %s, max SM clock %s; library %s" % (name, power, sm_clock, os.path.basename(_lib.LIB_PATH)))
    print("%-34s %6s %-22s %9s %8s %7s %10s" % ("shape (HxW cin->cout kK sS)", "per", "plan (Nw tpg splits)", "us",
                                               "TFLOP/s", "of 989", "us/step"))
    rows, total_us, total_flop = [], 0.0, 0.0
    torch.manual_seed(0)
    for fields, dy_ld, count in sorted(shapes, key=lambda s: (s[0][1] * s[0][2], s[0][3], s[0][4], s[0][5]),
                                       reverse=True):
        d = _lib.ConvDesc(*fields)
        dil = max(1, d.dilation)
        ho = (d.h + 2 * d.pad - dil * (d.ksize - 1) - 1) // d.stride + 1
        wo = (d.w + 2 * d.pad - dil * (d.ksize - 1) - 1) // d.stride + 1
        flop = 2.0 * d.n * ho * wo * d.cin * d.cout * d.ksize * d.ksize
        plan = (ctypes.c_int32 * 10)()
        rc = L.b200seg_conv2d_wgrad_plan_info(ctypes.byref(d), plan)
        if rc:
            sys.exit("plan_info failed (%d) for %s" % (rc, fields))
        x = (torch.randn((d.n, d.h, d.w, d.x_ld), device="cuda") * 0.5).to(torch.bfloat16)
        dy = (torch.randn((d.n, ho, wo, dy_ld), device="cuda") * 0.5).to(torch.bfloat16)
        dw = torch.zeros((d.cout * d.ksize * d.ksize * d.cin,), device="cuda")
        nbytes = L.b200seg_conv2d_wgrad_ws_bytes(ctypes.byref(d))
        ws = torch.empty((max(nbytes, 16) // 4,), device="cuda")

        def launch():
            rc = L.b200seg_conv2d_wgrad(ctypes.byref(d), ptr(x), ptr(dy), dy_ld, ptr(dw), ptr(ws), nbytes, stream_ptr())
            if rc:
                raise RuntimeError("b200seg_conv2d_wgrad returned %d for %s" % (rc, fields))

        us, times = time_replay(launch, args.launches, args.reps)
        tflops = flop / us / 1e6
        label = "%dx%d c%d->%d k%d s%d" % (d.h, d.w, d.cin, d.cout, d.ksize, d.stride)
        print("%-34s %6d %-22s %9.1f %8.1f %6.1f%% %10.1f" % (label, count, "%d %d %d" % (plan[0], plan[2], plan[4]),
                                                             us, tflops, 100.0 * tflops / PEAK_TFLOPS, us * count),
              flush=True)
        rows.append(dict(desc=fields, dy_ld=dy_ld, launches_per_step=count, ntile_w=plan[0], taps_per_group=plan[2],
                         splits=plan[4], us=round(us, 2), us_reps=[round(t, 2) for t in times],
                         tflops=round(tflops, 1)))
        total_us += us * count
        total_flop += flop * count
        del x, dy, dw, ws
    tflops = total_flop / total_us / 1e6
    print("per step: %d launches, %.3f TFLOP, %.3f ms, %.1f TFLOP/s (%.1f%% of 989)" %
          (sum(r["launches_per_step"] for r in rows), total_flop / 1e12, total_us / 1e3, tflops,
           100.0 * tflops / PEAK_TFLOPS))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=dict(name=name, power_limit=power, max_sm_clock=sm_clock),
                           library=os.path.basename(_lib.LIB_PATH), shapes=rows,
                           total=dict(ms=round(total_us / 1e3, 3), tflop=round(total_flop / 1e12, 4))), f, indent=1)


if __name__ == "__main__":
    main()
