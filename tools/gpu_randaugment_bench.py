"""RandAugment on the device input pipeline at a 1024x2048 crop: the device time of each op's kernels (torch.profiler,
CUDA activities), the bytes each op moves and their share of the H100 SXM's 3.35 TB/s HBM bound; the time of one whole
DeviceTrainTransform call (1024x2048 frame -> 1024x2048 crop, colour jitter) with and without RandAugment(2, 9) (CUDA
events around a loop of calls, host work included); and, labelled as a CPU number, Pillow's time per sample for the same
chain (oracle replay). Prints the card name and power limit read in the same run.

    python tools/gpu_randaugment_bench.py [--iters 20] [--out randaugment_bench.json]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# bytes per pixel each op moves at least (uint8 RGB, int64 labels): the geometric ops read and write both; the point
# ops and the blends read and write the RGB bytes; the histogram ops read them once more for the histogram
BYTES_PER_PIXEL = {"affine": 3 + 8 + 3 + 8, "hist": 3 + 3 + 3, "lut": 3 + 3, "enhance": 3 + 3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def op_times(h, w, iters, m=9):
    from torch.profiler import ProfilerActivity, profile
    from b200seg import augment as AUG
    from b200seg import raw
    rgb = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda")
    lab = torch.randint(0, 19, (h, w), dtype=torch.int64, device="cuda")
    spare = torch.empty_like(lab)
    rows = []
    for op, (name, lo, hi) in enumerate(AUG.RA_OPS):
        steps = AUG.randaugment_steps([(op, (float(m) / 30) * float(hi - lo) + lo, False)], h, w)
        if not steps:
            continue
        for _ in range(3):
            raw.rand_augment(rgb, lab, spare, steps)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                raw.rand_augment(rgb, lab, spare, steps)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith("_ZN7b200seg") or "aug_" in e.key)
        us /= iters
        nbytes = BYTES_PER_PIXEL[steps[0][0]] * h * w
        rows.append(dict(op=name, kind=steps[0][0], device_us=round(us, 2), bytes=nbytes,
                         hbm_share=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3) if us > 0 else None))
    return rows


def transform_ms(h, w, iters, rand_augment):
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    img_u8, mask_u8 = AO.synth_frame(h, w, 3)
    x, m = torch.from_numpy(img_u8).cuda(), torch.from_numpy(mask_u8).cuda()
    t = AUG.DeviceTrainTransform((h, w), rand_augment=rand_augment)
    out_i = torch.empty((3, h, w), dtype=torch.float32, device="cuda")
    out_l = torch.empty((h, w), dtype=torch.int64, device="cuda")
    random.seed(0)
    np.random.seed(0)
    for _ in range(3):
        t(x, m, out_image=out_i, out_label=out_l)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        t(x, m, out_image=out_i, out_label=out_l)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def pil_ms_per_sample(h, w, samples, rand_augment):
    """CPU: the Pillow replay of the same chain (resize / crop / flip, RandAugment, jitter, ToTensor, Normalize)."""
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    from oracle import randaugment_oracle as RO
    img_u8, mask_u8 = AO.synth_frame(h, w, 3)
    random.seed(0)
    np.random.seed(0)
    params = [AUG.draw_params(w, h, (h, w), rand_augment=rand_augment) for _ in range(samples)]
    t0 = time.perf_counter()
    for p in params:
        RO.reference_chain(img_u8, mask_u8, p, (h, w))
    return (time.perf_counter() - t0) * 1e3 / samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--pil-samples", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU: no CUDA device"
    name, power = card()
    h, w = a.height, a.width
    res = dict(card=name, power_limit=power, crop=[h, w], ops=op_times(h, w, a.iters))
    res["transform_ms"] = transform_ms(h, w, a.iters, None)
    res["transform_ms_rand_augment_2_9"] = transform_ms(h, w, a.iters, (2, 9))
    res["cpu_pil_ms_per_sample"] = pil_ms_per_sample(h, w, a.pil_samples, None)
    res["cpu_pil_ms_per_sample_rand_augment_2_9"] = pil_ms_per_sample(h, w, a.pil_samples, (2, 9))
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
