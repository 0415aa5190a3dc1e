"""Step time of the two-scale ocrnet.HRNet_Mscale training step (1024x2048, one crop, CUDA graph) under four losses,
timed in alternating rounds in one process: CE, image-weighted CE (--img_wt_loss --wt_bound 2.0, fp16 weights),
RMI with supervised multi-scale weight 0.05, and the same with RMI on the OCR auxiliary head (--ocr_aux_loss_rmi).
Prints the card name and power limit, per-round milliseconds per step, and each option's added time over CE.

    python tools/gpu_loss_options_bench.py [--steps 10] [--rounds 4] [--out loss_options.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

import torch  # noqa: E402

CONFIGS = [("ce", dict(criterion="ce", supervised_mscale_wt=0.0)),
           ("img_wt", dict(criterion="img_wt:2.0:half", supervised_mscale_wt=0.0)),
           ("rmi_sup0.05", dict(criterion="rmi", supervised_mscale_wt=0.05)),
           ("rmi_sup0.05_aux_rmi", dict(criterion="rmi", supervised_mscale_wt=0.05, ocr_aux_rmi=True))]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from b200seg.module import B200SegModule
    from oracle import seg_oracle as O
    images, gts = O.synth_batch(1, args.height, args.width, seed=1)
    images, gts = images.cuda(), gts.cuda()
    nets = {}
    for name, kw in CONFIGS:
        torch.manual_seed(0)
        net = B200SegModule("ocrnet.HRNet_Mscale", 19, **kw).cuda().train()
        with torch.no_grad():
            for n_, p_ in net.named_parameters():
                if p_.dim() == 4 and n_.startswith("backbone"):
                    p_.normal_(0, (2.0 / (p_.shape[1] * p_.shape[2] * p_.shape[3])) ** 0.5)
        nets[name] = net

    def step(net):
        net.zero_grad(set_to_none=True)
        net({"images": images, "gts": gts}).backward()

    for name, net in nets.items():              # eager warm-up, capture, replays
        for _ in range(4):
            step(net)
    torch.cuda.synchronize()
    times = {name: [] for name in nets}
    for _ in range(args.rounds):
        for name, net in nets.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.steps):
                step(net)
            end.record()
            end.synchronize()
            times[name].append(start.elapsed_time(end) / args.steps)
    gpu, power = card()
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = dict(gpu=gpu, power_limit=power, shape=[1, args.height, args.width], steps_per_round=args.steps,
               ms_per_step_rounds=times, ms_per_step_median=med,
               added_ms_vs_ce={k: med[k] - med["ce"] for k in med if k != "ce"},
               added_ms_aux_rmi_vs_rmi=med["rmi_sup0.05_aux_rmi"] - med["rmi_sup0.05"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
