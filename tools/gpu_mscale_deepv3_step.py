"""Step time and peak memory of the mscale.DeepV3W38 two-scale training step (full-width WideResNet-38, one crop per
GPU, CE, CUDA-graph replay, FusedSGD) at the 1024x2048 Cityscapes crop and the 800x800 crop of the reference's
train_cityscapes_deepv3.yml. Prints one JSON line per size with the GPU name and power limit it ran on; a size that fails
(out of memory, a refused launch) reports its error instead of a time.

    python tools/gpu_mscale_deepv3_step.py [--steps 10 --warmup 3] [--sizes 1024x2048,800x800]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

import torch  # noqa: E402

from b200seg.module import B200SegModule  # noqa: E402
from b200seg.optim import FusedSGD  # noqa: E402

TFLOP_PER_CROP_1024x2048 = 46.13      # tools/trace_step.py --arch mscale.DeepV3W38 (convolutions, 2 x MAC)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa
        return dict(gpu=torch.cuda.get_device_name(0), power_limit="unknown (%r)" % e)


def run(h, w, steps, warmup):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    net = B200SegModule("mscale.DeepV3W38", 19, criterion="ce").cuda().train()
    opt = FusedSGD(net.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator().manual_seed(0)
    images = torch.randn((1, 3, h, w), generator=g).cuda()
    gts = torch.randint(0, 19, (1, h, w), generator=g).cuda()
    try:
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
    except Exception as e:  # noqa: BLE001 - out of memory or a refused launch: report it for this size, go on
        return dict(size="%dx%d" % (h, w), error="%s: %s" % (type(e).__name__, str(e).splitlines()[0]),
                    peak_gb=torch.cuda.max_memory_allocated() / 1e9)
    ms = e0.elapsed_time(e1) / steps
    res = dict(size="%dx%d" % (h, w), ms_per_step=round(ms, 2), crops_per_s=round(1000.0 / ms, 3),
               peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2), loss=float(loss),
               kernels_per_step=getattr(net, "kernels_per_step", None))
    if (h, w) == (1024, 2048):
        res["tflops_per_s"] = round(TFLOP_PER_CROP_1024x2048 / (ms * 1e-3), 1)
    del net, opt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="1024x2048,800x800")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    for s in args.sizes.split(","):
        h, w = (int(v) for v in s.split("x"))
        res = run(h, w, args.steps, args.warmup)
        res.update(info)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
