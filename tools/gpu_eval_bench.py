#!/usr/bin/env python
"""cfg5 timing (GPU): ocrnet.HRNet_Mscale three-scale inference {0.5, 1.0, 2.0} of one 1024x2048 frame + device-side
argmax / confusion matrix, eager and CUDA-graph replay. Prints one JSON line."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
import torch  # noqa: E402

from b200seg.evaltail import eval_minibatch  # noqa: E402
from b200seg.module import B200SegModule  # noqa: E402


def main():
    torch.manual_seed(0)
    net = B200SegModule("ocrnet.HRNet_Mscale", 19, n_scales=[0.5, 1.0, 2.0]).cuda().eval()
    g = torch.Generator().manual_seed(0)
    images = torch.randn((1, 3, 1024, 2048), generator=g).cuda()
    gts = torch.randint(0, 19, (1, 1024, 2048), generator=g).cuda()
    out = {}
    with torch.no_grad():
        for it in range(2 + 6):          # call 1 eager, call 2 captures, then replays
            if it == 2:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
            res = eval_minibatch(net, images, gts, scales=(1.0,), do_flip=False)
        e1.record()
        torch.cuda.synchronize()
        out["ms_per_frame"] = e0.elapsed_time(e1) / 6
        pred = net({"images": images})["pred"]
        out["pred_checksum"] = float(pred.float().abs().mean())
        out["argmax_hist"] = torch.bincount(pred.argmax(1).flatten(), minlength=19)[:6].tolist()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
