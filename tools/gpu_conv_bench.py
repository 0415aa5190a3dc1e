"""Times every distinct forward and data-gradient convolution launch (conv3x3_halo_kernel / conv_igemm_kernel) of the
traced training step, one crop, through the entry point and with the epilogue the step asks for (batch statistics, BN
fold cells, residual addend, affine), and prints per shape the launches per step, the plan, microseconds per launch,
TFLOP/s, GB/s and the share of the roofline max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s) (H100 SXM dense bf16 and HBM3,
data sheet), then the launch-weighted total per step. Bytes are the sizes of the tensors handed to the launch, as
tools/trace_step.py counts them. Shapes and counts come from that tool's recorder (meta tensors, no device) in a child
`python -O`; each shape is timed with tools/gpu_wgrad_bench.py's CUDA-graph replay on random bf16 inputs. The card's
name, power limit and maximum SM clock are read in the same run. B200SEG_LIB_VARIANT=<tag> times
lib/libb200seg_<tag>.so (see b200seg/_lib.py). --planes hands every halo launch a plane-ordered weight image (random
bf16, include/b200seg.h), as the training and evaluation steps do.

    python tools/gpu_conv_bench.py [--arch ocrnet.HRNet_Mscale] [--height 1024 --width 2048] [--planes] [--out conv.json]"""
import argparse
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
_spec = importlib.util.spec_from_file_location("gpu_wgrad_bench", os.path.join(ROOT, "tools", "gpu_wgrad_bench.py"))
WB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(WB)

PEAK_TFLOPS = 989.0   # H100 SXM, dense bf16, data sheet (700 W)
PEAK_GBS = 3350.0     # H100 SXM HBM3, data sheet
ENTRIES = ("b200seg_conv2d_fwd", "b200seg_conv2d_fwd_add", "b200seg_conv2d_fwd_bn", "b200seg_conv2d_fwd_affine",
           "b200seg_conv2d_dgrad")


def _key(name, args, sizes):
    """(entry, ConvDesc fields, pitches and epilogue options, bytes handed to the launch) of one recorded call."""
    if name not in ENTRIES:
        return None
    from b200seg import _lib
    desc = tuple(getattr(args[0]._obj, f) for f, _ in _lib.ConvDesc._fields_)
    nbytes = sum(sizes.get(a, 0) for a in args if isinstance(a, int))
    if name == "b200seg_conv2d_dgrad":        # (d, dy, dy_ld, w, addend, addend_ld, dx, dx_ld, stream)
        opt = (args[2], args[4] is not None, args[5], args[7])
    elif name == "b200seg_conv2d_fwd_add":    # (d, x, w, bias, addend, addend_ld, y, stats, grid, stream)
        opt = (args[5], args[7] is not None)
    elif name == "b200seg_conv2d_fwd_bn":     # (d, x, w, bias, y, fold, stream)
        opt = ()
    elif name == "b200seg_conv2d_fwd_affine":  # (d, x, w, scale, shift, relu, addend, addend_ld, y, stream)
        opt = (args[5], args[6] is not None, args[7])
    else:                                     # (d, x, w, bias, y, stats, grid, stream)
        opt = (args[5] is not None,)
    return name, desc, opt, nbytes


def out_hw(d):
    dil = max(1, d.dilation)
    return ((d.h + 2 * d.pad - dil * (d.ksize - 1) - 1) // d.stride + 1,
            (d.w + 2 * d.pad - dil * (d.ksize - 1) - 1) // d.stride + 1)


def make_launch(L, name, d, opt, torch):
    """A closure that runs the recorded call once on random inputs (and the buffers it keeps alive)."""
    from b200seg import _lib
    from b200seg._lib import ptr, stream_ptr
    bf16, dev = torch.bfloat16, "cuda"
    ho, wo = out_hw(d)
    taps = d.ksize * d.ksize

    def rnd(*shape):
        return (torch.randn(shape, device=dev) * 0.5).to(bf16)

    def check(rc):
        if rc:
            raise RuntimeError("%s returned %d for %s" % (name, rc, d))

    if name == "b200seg_conv2d_dgrad":
        dy_ld, has_add, add_ld, dx_ld = opt
        dy, w = rnd(d.n, ho, wo, dy_ld), rnd(d.cin, taps, d.cout)
        dx = rnd(d.n, d.h, d.w, dx_ld)
        add = dx if has_add else None
        keep = (dy, w, dx)
        return (lambda: check(L.b200seg_conv2d_dgrad(ctypes.byref(d), ptr(dy), dy_ld, ptr(w), ptr(add), add_ld, ptr(dx),
                                                     dx_ld, stream_ptr()))), keep
    x, w = rnd(d.n, d.h, d.w, d.x_ld), rnd(d.cout, taps, d.cin)
    bias = torch.randn(d.cout, device=dev) * 0.1 if d.has_bias else None
    y = torch.empty((d.n, ho, wo, d.y_ld), dtype=torch.float32 if d.out_fp32 else bf16, device=dev)
    stats = torch.empty(max(1, L.b200seg_conv2d_stats_elems(ctypes.byref(d))), device=dev)
    grid = ctypes.c_int32(0)
    keep = (x, w, bias, y, stats)
    if name == "b200seg_conv2d_fwd":
        st = stats if opt[0] else None
        return (lambda: check(L.b200seg_conv2d_fwd(ctypes.byref(d), ptr(x), ptr(w), ptr(bias), ptr(y), ptr(st),
                                                   ctypes.byref(grid), stream_ptr()))), keep
    if name == "b200seg_conv2d_fwd_add":
        add_ld, has_stats = opt
        add, st = rnd(d.n, ho, wo, add_ld), (stats if has_stats else None)
        return (lambda: check(L.b200seg_conv2d_fwd_add(ctypes.byref(d), ptr(x), ptr(w), ptr(bias), ptr(add), add_ld,
                                                       ptr(y), ptr(st), ctypes.byref(grid), stream_ptr()))), keep + (add,)
    if name == "b200seg_conv2d_fwd_affine":
        relu, has_add, add_ld = opt
        scale, shift = torch.rand(d.cout, device=dev) + 0.5, torch.randn(d.cout, device=dev) * 0.1
        add = rnd(d.n, ho, wo, add_ld) if has_add else None
        return (lambda: check(L.b200seg_conv2d_fwd_affine(ctypes.byref(d), ptr(x), ptr(w), ptr(scale), ptr(shift), relu,
                                                          ptr(add), add_ld, ptr(y), stream_ptr()))), keep + (add,)
    # fwd_bn: statistics added to the layer's fp64 cells (deferred finalisation, as in the step)
    cells = torch.zeros(2 * ((d.cout + 15) // 16 * 16), dtype=torch.float64, device=dev)
    f = _lib.BnFold()
    f.accum, f.c = ptr(cells), d.cout
    return (lambda: check(L.b200seg_conv2d_fwd_bn(ctypes.byref(d), ptr(x), ptr(w), ptr(bias), ptr(y), ctypes.byref(f),
                                                  stream_ptr()))), keep + (cells, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="ocrnet.HRNet_Mscale")
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=20, help="launches per CUDA-graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per shape (the median is kept)")
    ap.add_argument("--planes", action="store_true", help="halo launches stream their weights from the image")
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    ap.add_argument("--trace-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.trace_only:
        if __debug__:
            sys.exit("--trace-only runs under python -O (the wrappers assert is_cuda)")
        seen = WB.record_calls(args.arch, args.height, args.width, _key)
        print(json.dumps([[name, list(desc), list(opt), nbytes, n] for (name, desc, opt, nbytes), n in seen.items()]))
        return

    out = subprocess.run([sys.executable, "-O", os.path.abspath(__file__), "--trace-only", "--arch", args.arch,
                          "--height", str(args.height), "--width", str(args.width)],
                         capture_output=True, text=True, check=True).stdout
    calls = json.loads(out.strip().splitlines()[-1])

    import torch
    from b200seg import _lib
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    L = _lib.lib()
    name, power, sm_clock = WB.card()
    print("%s, power limit %s, max SM clock %s; library %s%s" % (name, power, sm_clock, os.path.basename(_lib.LIB_PATH),
                                                             ", weight images" if args.planes else ""))
    print("%-12s %-34s %5s %-14s %9s %8s %8s %7s %10s" % ("entry", "shape (HxW cin->cout kK sS)", "calls",
                                                         "kern BN occ", "us", "TFLOP/s", "GB/s", "roof", "us/step"))
    rows, total_us, total_flop, total_roof = [], 0.0, 0.0, 0.0
    torch.manual_seed(0)
    for entry, fields, opt, nbytes, count in sorted(calls, key=lambda c: -conv_flop(c[1]) * c[4]):
        d = _lib.ConvDesc(*fields)
        flop = conv_flop(fields)
        plan = (ctypes.c_int32 * 12)()
        which = 1 if entry == "b200seg_conv2d_dgrad" else 0
        pd = _lib.ConvDesc(*fields)
        if L.b200seg_conv2d_plan_info(ctypes.byref(pd), which, plan) != 0:
            plan[0] = plan[1] = plan[6] = -1    # stride-2 data gradients: four sub-lattice launches, no plan query
        launch, keep = make_launch(L, entry, d, tuple(opt), torch)
        if args.planes and plan[0] == 1:
            img_rows = ctypes.c_int32(0)
            n_img = L.b200seg_conv2d_planes_elems(ctypes.byref(d), which, ctypes.byref(img_rows))
            img = (torch.randn(n_img, device="cuda") * 0.5).to(torch.bfloat16)
            d.w_planes, d.w_planes_rows = img.data_ptr(), img_rows.value
            keep = keep + (img,)
        us, times = WB.time_replay(launch, args.launches, args.reps)
        roof_us = max(flop / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_GBS * 1e9)) * 1e6
        label = "%dx%d c%d->%d k%d s%d" % (d.h, d.w, d.cin, d.cout, d.ksize, d.stride)
        short = entry[len("b200seg_conv2d_"):]
        kern = {1: "halo", 0: "igemm"}.get(plan[0], "igemm4")
        print("%-12s %-34s %5d %-14s %9.1f %8.1f %8.1f %6.1f%% %10.1f" % (
            short, label, count, "%s %d %d" % (kern, plan[1], plan[6]), us, flop / us / 1e6, nbytes / us / 1e3,
            100.0 * roof_us / us, us * count), flush=True)
        rows.append(dict(entry=short, desc=fields, options=opt, launches_per_step=count, kernel=kern, BN=plan[1],
                         occ=plan[6], us=round(us, 2), us_reps=[round(t, 2) for t in times],
                         tflops=round(flop / us / 1e6, 1), gbs=round(nbytes / us / 1e3, 1),
                         roofline_share=round(roof_us / us, 4)))
        total_us += us * count
        total_flop += flop * count
        total_roof += roof_us * count
        del keep
    print("per step: %d calls, %.3f TFLOP, %.3f ms, %.1f TFLOP/s, roofline %.3f ms (%.1f%%)" %
          (sum(r["launches_per_step"] for r in rows), total_flop / 1e12, total_us / 1e3, total_flop / total_us / 1e6,
           total_roof / 1e3, 100.0 * total_roof / total_us))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=dict(name=name, power_limit=power, max_sm_clock=sm_clock),
                           library=os.path.basename(_lib.LIB_PATH), shapes=rows,
                           total=dict(ms=round(total_us / 1e3, 3), tflop=round(total_flop / 1e12, 4),
                                      roofline_ms=round(total_roof / 1e3, 3))), f, indent=1)


def conv_flop(fields):
    """2 x MAC of the convolution a ConvDesc describes (data gradients: the same GEMM with the channel roles swapped)."""
    from b200seg import _lib
    d = _lib.ConvDesc(*fields)
    ho, wo = out_hw(d)
    return 2.0 * d.n * ho * wo * d.cin * d.cout * d.ksize * d.ksize


if __name__ == "__main__":
    main()
