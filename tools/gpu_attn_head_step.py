"""Step time and peak memory of the multi-scale training steps with each attention-head ablation (--mscale_no3x3,
--mscale_dropout, --mscale_old_arch, and no3x3 + dropout; mscale.DeepV3W38 takes no3x3 only) against the default head: W48 / WRN-38 trunk, one 1024x2048
crop, CE, CUDA-graph replay, FusedSGD. Each variant is timed against the default model in the same process, alternating
round after round, so that drift on a shared GPU hits both alike; the line reports the medians over the rounds. Also
times the attention head's last BatchNorm apply and backward passes at the 1.0x map with and without the fused dropout.
Peak memory is the step's own (allocated beyond what the default model already holds). Prints one JSON line per
arch and variant with the GPU name and power limit it ran on.

    python tools/gpu_attn_head_step.py [--steps 6 --warmup 3 --rounds 3] [--archs ocrnet.HRNet_Mscale,...]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from b200seg import arch as A, raw  # noqa: E402
from b200seg.module import B200SegModule  # noqa: E402
from b200seg.optim import FusedSGD  # noqa: E402
from gpu_mscale_deepv3_step import gpu_info  # noqa: E402

ARCHS = ("ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.HRNet_ASP", "mscale.DeepV3W38")
VARIANTS = {"default": {}, "no3x3": dict(mscale_inner_3x3=False), "dropout": dict(mscale_dropout=True),
            "oldarch": dict(mscale_oldarch=True), "no3x3_dropout": dict(mscale_inner_3x3=False, mscale_dropout=True)}


def build(arch, variant):
    net = B200SegModule(arch, 19, criterion="ce", ocfg=dict(A.OCR_DEFAULT, **VARIANTS[variant])).cuda().train()
    return net, FusedSGD(net.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4)


def run(net, opt, images, gts, iters):
    for _ in range(iters):
        opt.zero_grad(set_to_none=True)
        loss = net({"images": images, "gts": gts})
        loss.backward()
        opt.step()
    return loss


def timed_steps(net, opt, images, gts, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(net, opt, images, gts, steps)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bn_pass_ms(n, h, w, c=256, reps=50):
    """ms of the BatchNorm apply (+ ReLU) and backward passes on one [n, h, w, c] map, without and with the fused
    dropout."""
    g = torch.Generator().manual_seed(1)
    y = torch.randn((n, h, w, c), generator=g).to(torch.bfloat16).cuda()
    dz = torch.randn((n, h, w, c), generator=g).to(torch.bfloat16).cuda()
    scale, shift = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    mean, invstd = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    dg, db = torch.zeros(c, device="cuda"), torch.zeros(c, device="cuda")
    cells = torch.zeros(2 * c, dtype=torch.float64, device="cuda")
    seed = torch.tensor([7], dtype=torch.int64, device="cuda")
    z = torch.empty_like(y)
    dy = torch.empty_like(y)
    out = {}
    for tag, drop in (("plain", None), ("dropout", (seed, 1))):
        for what, fn in (("apply", lambda: raw.bn_apply(y, scale, shift, None, None, True, out=z, dropout=drop)),
                         ("bwd", lambda: raw.bn_bwd(dz, z, None, y, mean, invstd, scale, dg, db, dy_out=dy,
                                                    cells=cells, dropout=drop))):
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out["%s_%s_ms" % (what, tag)] = round(e0.elapsed_time(e1) / reps, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--archs", default=",".join(ARCHS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    h, w = 1024, 2048
    g = torch.Generator().manual_seed(0)
    images = torch.randn((1, 3, h, w), generator=g).cuda()
    gts = torch.randint(0, 19, (1, h, w), generator=g).cuda()
    for arch in args.archs.split(","):
        # mscale.DeepV3W38 takes --mscale_no3x3 only
        variants = [v for v in VARIANTS if arch != "mscale.DeepV3W38" or v in ("default", "no3x3")]
        base, peak0 = None, None
        for v in variants:
            # two models alive at a time: the default and the variant, timed alternately in the same rounds
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            cand = build(arch, v)
            run(*cand, images, gts, args.warmup)
            torch.cuda.synchronize()
            peak = (torch.cuda.max_memory_allocated() - before) / 1e9
            if base is None:
                base, peak0 = cand, peak
                continue
            run(*base, images, gts, args.warmup)      # the default re-warmed after the variant's build
            times = {"default": [], v: []}
            for _ in range(args.rounds):
                times["default"].append(timed_steps(*base, images, gts, args.steps))
                times[v].append(timed_steps(*cand, images, gts, args.steps))
            ms0, ms = statistics.median(times["default"]), statistics.median(times[v])
            res = dict(arch=arch, variant=v, size="%dx%d" % (h, w), ms_per_step=round(ms, 2),
                       default_ms_per_step=round(ms0, 2), rounds=[[round(a, 2), round(b, 2)] for a, b in
                                                                  zip(times["default"], times[v])],
                       vs_default=round(ms / ms0, 4), peak_gb=round(peak, 2), default_peak_gb=round(peak0, 2))
            res.update(info)
            print(json.dumps(res), flush=True)
            del cand
            torch.cuda.empty_cache()
        del base
        torch.cuda.empty_cache()
        f = 2 if arch == "mscale.DeepV3W38" else 4
        res = dict(arch=arch, what="attention head BN passes at the 1.0x map", map=[1, h // f, w // f, 256])
        res.update(bn_pass_ms(1, h // f, w // f))
        res.update(info)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
