"""Static trace of one training step on the CPU (no GPU, no kernels): runs the real step program (b200seg.model /
b200seg.engine / b200seg.raw) on `meta` tensors with every launching C-ABI entry point replaced by a recorder, and
prints, per kernel class, the number of launches, the algorithmic FLOPs / bytes and the roofline time
sum_launches max(FLOPs / P, bytes / B). Host-only planner queries (stats_elems, ws_bytes, grids ...) still go to the real
library, so buffer sizes are the real ones.

    python -O tools/trace_step.py [--arch ocrnet.HRNet_Mscale] [--height 1024 --width 2048] [--tflops 1386.7 --gbs 6650]
    python -O tools/trace_step.py --eval [--arch ...]      # the evaluation forwards at 0.5x, 1.0x and 2.0x instead
    python -O tools/trace_step.py --eval --assembly        # ... as b200seg.evaltail.eval_minibatch runs them, with the
                                                           # output assembly, flips and the scoring tail
    python -O tools/trace_step.py --criterion rmi --ocr-aux-rmi [--sup-wt 0.05]   # the training step with another loss

-O is required: the wrappers assert `is_cuda`, and the point of this tool is to run them without a device.
Bytes of a launch = sizes of the tensors handed to it (views count with their own extent), i.e. what the kernel must at
least read or write once; FLOPs are counted for the convolutions (2 x MAC) only."""
import argparse
import collections
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

import torch  # noqa: E402

from b200seg import _lib, engine as EN, model as M, raw  # noqa: E402

QUERY = re.compile(r"(_elems|_ws_bytes|_grid|_launches|_chunk|_splits|_abi_version|_build_info|_plan_info)$")
SIZES = {}          # fake address -> bytes
EVENTS = []         # (entry point, bytes, flops, detail)
CONV_DESCS = {}     # index into EVENTS -> ((n, h, w, cin, cout, k, stride, dilation), emit_stats, out_fp32, has_bias):
                    # the descriptor of a convolution as the step hands it over (a data gradient's cout is padded)
LAUNCH_ARGS = {}    # index into EVENTS -> the arguments of every other launch (tools/ew_classes.py keys them): scalars as
                    # they are, pointers as PTR (present) or None (absent), a fuse descriptor as ("fuse", n, h, w, c,
                    # relu, ((h, w, ld, affine) per term)), a BatchNorm fold as ("fold", c, count, gamma, running, batch),
                    # a loss descriptor as ("ms", n, h, w, hq, wq, hm, wm, hl, wl, nheads, sup_wt, ignore_index, loss_kind)
PTR = "ptr"
_next = [0x7F0000000000]     # far above any scalar argument (pixel counts, pitches ...) the entry points take


def fake_ptr(t):
    if t is None:
        return None
    a = _next[0]
    _next[0] += 0x1000
    SIZES[a] = t.numel() * t.element_size()
    return a


class Recorder:
    def __init__(self, real):
        self.real = real

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if QUERY.search(name):
            return fn

        def fake(*args):
            nbytes, flops, detail = 0, 0.0, ""
            rec = []
            for a in args:
                if isinstance(a, int) and a in SIZES:
                    nbytes += SIZES[a]
                    rec.append(PTR)
                elif hasattr(a, "_obj"):                      # ctypes.byref(...)
                    obj = a._obj
                    rec.append(PTR)                           # any other descriptor (a SyncBN exchange ...)
                    if isinstance(obj, _lib.FuseDesc):
                        rec[-1] = ("fuse", obj.n, obj.h, obj.w, obj.c, obj.relu,
                                   tuple((t.h, t.w, t.ld, bool(t.scale)) for t in obj.term[:obj.nterms]))
                    elif isinstance(obj, _lib.BnFold):
                        rec[-1] = ("fold", obj.c, obj.count, bool(obj.gamma), bool(obj.running_mean),
                                   bool(obj.batch_stats_out))
                    elif isinstance(obj, _lib.MscaleDesc):
                        rec[-1] = ("ms", obj.n, obj.h, obj.w, obj.hq, obj.wq, obj.hm, obj.wm, obj.hl, obj.wl,
                                   obj.nheads, obj.sup_wt, obj.ignore_index, obj.loss_kind)
                    if isinstance(obj, _lib.ConvDesc):
                        k, s = obj.ksize, obj.stride
                        dil = max(1, getattr(obj, "dilation", 1))
                        ho = (obj.h + 2 * obj.pad - dil * (k - 1) - 1) // s + 1
                        wo = (obj.w + 2 * obj.pad - dil * (k - 1) - 1) // s + 1
                        flops = 2.0 * obj.n * ho * wo * obj.cin * obj.cout * k * k
                        detail = "%dx%d c%d->%d k%d s%d" % (obj.h, obj.w, obj.cin, obj.cout, k, s)
                        if dil > 1:
                            detail += " d%d" % dil
                        CONV_DESCS[len(EVENTS)] = ((obj.n, obj.h, obj.w, obj.cin, obj.cout, k, s, dil),
                                                   obj.emit_stats, obj.out_fp32, obj.has_bias)
                    elif isinstance(obj, ctypes.c_int32):
                        obj.value = 148                       # stats_grid of the convolutions
                else:
                    rec.append(a)
            if not detail:
                LAUNCH_ARGS[len(EVENTS)] = tuple(rec)
            EVENTS.append((name[len("b200seg_"):], nbytes, flops, detail))
            return 0
        return fake


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="ocrnet.HRNet_Mscale")
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    pk = dict(bf16_tflops_sustained=1386.7, hbm_gbs=6572.9)       # this pool's measured values; refreshed from the file
    try:
        import json
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            pk.update(json.load(f))
    except (OSError, ValueError):
        pass
    ap.add_argument("--tflops", type=float, default=pk["bf16_tflops_sustained"],
                    help="sustained dense bf16 TFLOP/s (MEASURED_PEAKS.json)")
    ap.add_argument("--gbs", type=float, default=pk["hbm_gbs"], help="HBM copy bandwidth GB/s (MEASURED_PEAKS.json)")
    ap.add_argument("--top", type=int, default=0, help="also list the N largest launches by roofline time")
    ap.add_argument("--bn-cells", action="store_true",
                    help="trace the training default with per-GPU statistics: deferred BatchNorm finalisation inside "
                         "the consuming apply passes; without the flag: the program with separate bn_finalize / "
                         "bn_bwd_finalize launches (SyncBN)")
    ap.add_argument("--attn-head", default="default", choices=["default", "no3x3", "dropout", "oldarch", "no3x3_dropout"],
                    help="attention-head ablation of the multi-scale archs (--mscale_no3x3 / --mscale_dropout / "
                         "--mscale_old_arch of the reference's train.py)")
    ap.add_argument("--eval", action="store_true",
                    help="trace the evaluation forward instead of the training step: BatchNorm from the running "
                         "statistics, one scale pass each at 0.5x, 1.0x and 2.0x of --height x --width")
    ap.add_argument("--assembly", action="store_true",
                    help="with --eval: run the evaluation as b200seg.evaltail.eval_minibatch does, with flips and the "
                         "output assembly of b200seg.evalpath (multi-scale archs: N_SCALES 0.5, 1.0, 2.0 inside the "
                         "network; the others: scales 0.5, 1.0, 2.0 around it)")
    ap.add_argument("--criterion", default="ce",
                    help="loss of the training step, as B200SegModule takes it: ce, rmi or img_wt[:upper_bound[:half]]")
    ap.add_argument("--sup-wt", type=float, default=0.0,
                    help="supervised_mscale_wt of the two-scale archs (cfg.LOSS.SUPERVISED_MSCALE_WT)")
    ap.add_argument("--ocr-aux-rmi", action="store_true",
                    help="with --criterion rmi: RMI on the OCR auxiliary head too (cfg.LOSS.OCR_AUX_RMI)")
    args = ap.parse_args()
    if __debug__:
        sys.exit("run with python -O (the wrappers assert is_cuda)")

    rec = Recorder(_lib.lib())
    _lib.lib = lambda: rec
    raw.lib = lambda: rec
    raw.ptr = fake_ptr
    raw.stream_ptr = lambda: 0

    from b200seg.module import B200SegModule
    from b200seg import arch as A
    flags = dict(no3x3=dict(mscale_inner_3x3=False), dropout=dict(mscale_dropout=True),
                 oldarch=dict(mscale_oldarch=True),
                 no3x3_dropout=dict(mscale_inner_3x3=False, mscale_dropout=True)).get(args.attn_head, {})
    net = B200SegModule(args.arch, 19, criterion=args.criterion, ocfg=dict(A.OCR_DEFAULT, **flags),
                        supervised_mscale_wt=args.sup_wt, ocr_aux_rmi=args.ocr_aux_rmi)
    dev = torch.device("meta")
    tensors = {k: torch.empty(v.shape, dtype=v.dtype, device=dev) for k, v in net._tensors().items()}
    packed, grads = {}, {}
    for n, p in net.named_parameters():
        if p.dim() == 4:
            o, i, k, _ = p.shape
            i = 16 if i == 3 else i
            packed[n[: -len(".weight")]] = (torch.empty((o, k * k, i), dtype=torch.bfloat16, device=dev),
                                            torch.empty((i, k * k, (o + 7) // 8 * 8), dtype=torch.bfloat16, device=dev))
            grads[n] = torch.empty((o, k * k, i), dtype=torch.float32, device=dev)
        else:
            grads[n] = torch.empty(p.shape, dtype=torch.float32, device=dev)
    images = torch.empty((1, 3, args.height, args.width), dtype=torch.float32, device=dev)
    if args.eval:
        E = EN.Engine(tensors, {}, packed, False, None)
        E.eval_bn = {n[: -len(".running_mean")]: (torch.empty(v.shape, dtype=torch.float32, device=dev),
                                                  torch.empty(v.shape, dtype=torch.float32, device=dev))
                     for n, v in tensors.items() if n.endswith(".running_mean")}
        if args.assembly:
            from b200seg import evaltail
            evaltail.eval_minibatch(_EvalNet(net, tensors, packed, E.eval_bn), images,
                                    torch.empty((1, args.height, args.width), dtype=torch.long, device=dev),
                                    scales=(0.5, 1.0, 2.0), do_flip=True)
            report(args, "evaluation with output assembly: %d launches" % len(EVENTS))
            return
        for s in (0.5, 1.0, 2.0):
            hw = (int(args.height * s), int(args.width * s))
            if A.has_wrn38_trunk(args.arch) and not A.is_two_scale(args.arch):
                M.deepv3_pass(E, images, net.hcfg, hw, None)
            else:
                M.scale_pass(E, images, hw, args.arch, net.hcfg, net.ocfg)
        report(args, "evaluation forward at 0.5x, 1.0x and 2.0x: %d launches" % len(EVENTS))
        return
    gts = torch.empty((1, args.height, args.width), dtype=torch.long, device=dev)
    if A.has_wrn38_trunk(args.arch):
        n_sets = 2 if A.is_two_scale(args.arch) else 1        # one Dropout2d mask set per scale pass
        mask = torch.empty((n_sets * sum(c for _b, c, _p in A.wrn_drop_layout(net.hcfg)),), dtype=torch.float32,
                           device=dev)
    else:
        mask = torch.empty((1, net.ocfg["mid_channels"]), dtype=torch.float32, device=dev)
    bncells = None
    if args.bn_cells:
        bncells = {n[: -len(".running_mean")]: (torch.empty(2 * ((v.shape[0] + 15) // 16 * 16), dtype=torch.float64, device=dev),
                                                torch.empty(2 * v.shape[0], dtype=torch.float64, device=dev))
                   for n, v in tensors.items() if n.endswith(".running_mean")}
    E = EN.Engine(tensors, grads, packed, True, mask, bncells=bncells,
                  attn_seed=torch.empty((1,), dtype=torch.int64, device=dev))
    M.train_loss(E, images, gts, args.arch, net.hcfg, net.ocfg, net.lo_scale, net.ocr_alpha, net.sup_wt,
                 net.ignore_index, loss_kind=net.loss_kind, img_wt=net.img_wt, ocr_aux_rmi=net.ocr_aux_rmi)
    n_fwd = len(EVENTS)
    M.run_backward(E)
    report(args, "one crop: %d launches (%d forward + loss, %d backward)" % (len(EVENTS), n_fwd, len(EVENTS) - n_fwd))


class _EvalNet:
    """What b200seg.evalpath.eval_forward and b200seg.evaltail.eval_minibatch read of a B200SegModule in eval mode, over
    the traced meta tensors."""
    training = False
    lo_scale = 0.5

    def __init__(self, net, tensors, packed, eval_bn):
        from b200seg import arch as A
        self.arch, self.hcfg, self.ocfg = net.arch, net.hcfg, net.ocfg
        self.n_scales = (0.5, 1.0, 2.0) if A.is_two_scale(net.arch) else None
        self._tensors = lambda: tensors
        self._packed = packed
        self._planes = {}       # the weight images change which bytes a halo launch reads, not the launches
        self._eval_bn_params = lambda: eval_bn
        self._ensure_device_state = self._repack = lambda: None

    def __call__(self, inputs):
        from b200seg import evalpath
        return evalpath.eval_forward(self, inputs["images"])


def report(args, what):
    P, B = args.tflops * 1e12, args.gbs * 1e9
    agg = collections.OrderedDict()
    tot = [0, 0.0, 0.0, 0.0]
    for i, (name, nbytes, flops, detail) in enumerate(EVENTS):
        t = max(flops / P, nbytes / B)
        a = agg.setdefault(name, [0, 0.0, 0.0, 0.0])
        for acc in (a, tot):
            acc[0] += 1; acc[1] += flops; acc[2] += nbytes; acc[3] += t
    print("%s  %dx%d  %s" % (args.arch, args.height, args.width, what))
    print("%-24s %8s %12s %12s %12s" % ("entry point", "launches", "TFLOP", "GB", "roofline ms"))
    for name, (c, f, b, t) in sorted(agg.items(), key=lambda kv: -kv[1][3]):
        print("%-24s %8d %12.3f %12.2f %12.3f" % (name, c, f / 1e12, b / 1e9, t * 1e3))
    print("%-24s %8d %12.3f %12.2f %12.3f" % ("total", tot[0], tot[1] / 1e12, tot[2] / 1e9, tot[3] * 1e3))
    print("(peaks: %.1f TFLOP/s, %.0f GB/s; roofline ms = sum over launches of max(FLOPs/P, bytes/B))" %
          (args.tflops, args.gbs))
    if args.top:
        big = sorted(EVENTS, key=lambda e: -max(e[2] / P, e[1] / B))[: args.top]
        for name, nbytes, flops, detail in big:
            print("  %-22s %-28s %8.1f MB %8.2f GFLOP %8.1f us" %
                  (name, detail, nbytes / 1e6, flops / 1e9, max(flops / P, nbytes / B) * 1e6))


if __name__ == "__main__":
    main()
