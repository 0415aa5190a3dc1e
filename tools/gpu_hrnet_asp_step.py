"""Step time and peak memory of the basic.HRNet_ASP and mscale.HRNet_ASP training steps (W48 trunk, one 1024x2048 crop
per GPU, CE, CUDA-graph replay, FusedSGD), and the time of the step's dilated ASPP launches: the three 720 -> 256 3x3
branches (dilation 12 / 24 / 36) of every scale pass, forward with batch statistics, data gradient (accumulated into
the trunk map's gradient) and weight gradient, each timed in isolation with CUDA events at the step's shapes and summed
per step. Prints one JSON line per arch with the GPU name and power limit it ran on; an arch that fails (out of memory,
a refused launch) reports its error instead of a time.

    python tools/gpu_hrnet_asp_step.py [--steps 10 --warmup 3] [--archs basic.HRNet_ASP,mscale.HRNet_ASP]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from b200seg import arch as A, raw  # noqa: E402
from b200seg.module import B200SegModule  # noqa: E402
from b200seg.optim import FusedSGD  # noqa: E402
from gpu_mscale_deepv3_step import gpu_info  # noqa: E402

# tools/trace_step.py --arch <arch> (convolutions, 2 x MAC, one 1024x2048 crop)
TFLOP_PER_CROP_1024x2048 = {"basic.HRNet_ASP": 9.33, "mscale.HRNet_ASP": 12.20}


def step(arch, h, w, steps, warmup):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    net = B200SegModule(arch, 19, criterion="ce").cuda().train()
    opt = FusedSGD(net.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator().manual_seed(0)
    images = torch.randn((1, 3, h, w), generator=g).cuda()
    gts = torch.randint(0, 19, (1, h, w), generator=g).cuda()
    for it in range(warmup + steps):
        if it == warmup:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        opt.zero_grad(set_to_none=True)
        loss = net({"images": images, "gts": gts})
        loss.backward()
        opt.step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = dict(ms_per_step=round(ms, 2), crops_per_s=round(1000.0 / ms, 3),
               peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2), loss=float(loss),
               kernels_per_step=getattr(net, "kernels_per_step", None),
               tflops_per_s=round(TFLOP_PER_CROP_1024x2048[arch] / (ms * 1e-3), 1))
    del net, opt
    return res


def _timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def dilated_aspp_ms(h4, w4, red=256, cin=720, reps=20):
    """ms of the forward, data-gradient and weight-gradient launches of the three dilated branches on one h4 x w4
    map."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn((1, h4, w4, cin), generator=g).to(torch.bfloat16).cuda()
    dy = torch.randn((1, h4, w4, red), generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn((red, 9, cin), generator=g) * 0.01).to(torch.bfloat16).cuda()
    w_d = wt.flip(1).permute(2, 1, 0).contiguous()
    cat = torch.empty((1, h4, w4, 5 * red), dtype=torch.bfloat16, device="cuda")
    dx = torch.zeros((1, h4, w4, cin), dtype=torch.bfloat16, device="cuda")
    dw = torch.zeros((red, 9, cin), dtype=torch.float32, device="cuda")
    ws = [None]
    out = dict(fwd=0.0, dgrad=0.0, wgrad=0.0)
    for i, r in enumerate(A.ASPP_RATES):
        c0 = (2 + i) * red
        out["fwd"] += _timed(lambda: raw.conv2d_fwd(x, wt, emit_stats=True, dilation=r, out=cat[..., c0:c0 + red]),
                             reps)
        out["dgrad"] += _timed(lambda: raw.conv2d_dgrad(dy, w_d, (1, h4, w4, cin), 3, 1, addend=dx, out=dx, dilation=r),
                               reps)
        out["wgrad"] += _timed(lambda: raw.conv2d_wgrad(x, dy, dw, red, 3, 1, ws_holder=ws, dilation=r), reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--archs", default="basic.HRNet_ASP,mscale.HRNet_ASP")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    h, w = 1024, 2048
    for arch in args.archs.split(","):
        res = dict(arch=arch, size="%dx%d" % (h, w))
        try:
            res.update(step(arch, h, w, args.steps, args.warmup))
            passes = [(h // 4, w // 4)] + ([(h // 8, w // 8)] if A.is_two_scale(arch) else [])
            parts = [dilated_aspp_ms(ph, pw) for ph, pw in passes]
            res["dilated_aspp_ms_per_step"] = {k: round(sum(p[k] for p in parts), 2) for k in ("fwd", "dgrad", "wgrad")}
            res["dilated_aspp_ms_per_step"]["total"] = round(sum(res["dilated_aspp_ms_per_step"].values()), 2)
        except Exception as e:  # noqa: BLE001 - out of memory or a refused launch: report it for this arch, go on
            res.update(error="%s: %s" % (type(e).__name__, str(e).splitlines()[0]),
                       peak_gb=torch.cuda.max_memory_allocated() / 1e9)
        res.update(info)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
