"""Device-side evaluation tail: the scoring half of the reference's eval_minibatch (utils/trnval_utils.py:84-196).

The reference sums the network output over flips / scales on the GPU, then moves the [N,19,H,W] fp32 logits to the host
for softmax, argmax and the numpy bincount of fast_hist (utils/misc.py:50-85). Here the whole tail stays on the device:
only the 19x19 int64 confusion matrix (and, on request, the class map) ever crosses PCIe.
"""
import torch

from . import raw


@torch.no_grad()
def eval_minibatch(net, images, gts, scales=(1.0,), do_flip=False, mscale=None, hist=None):
    """images fp32 [N,3,H,W], gts int64 [N,H,W] (device tensors). Mirrors eval_minibatch: with a multi-scale model
    (cfg.MODEL.MSCALE) the scales are handled inside the network, so ``scales`` is (1.0,) (trnval_utils.py:97-101).
    Returns dict(predictions int64 [N,H,W], prob_mask fp32 [N,H,W], hist int64 [19,19] accumulated into ``hist``)."""
    assert not net.training
    if mscale is None:
        mscale = net.arch in ("ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.HRNet_ASP") and bool(net.n_scales)
    if mscale:
        scales = (1.0,)
    n, _, H, W = images.shape
    flips = (1, 0) if do_flip else (0,)
    out = None
    for flip in flips:
        for s in scales:
            x = images
            if flip:
                x = raw.accum_pred(x.contiguous(), None, flip=True)          # mirrored copy of the input
            if s != 1.0:
                x = raw.resize_nchw(x.contiguous(), round(H * s), round(W * s))
            pred = net({"images": x})["pred"]
            if s != 1.0:
                pred = raw.resize_nchw(pred, H, W)
            out = raw.accum_pred(pred.contiguous(), out, flip=bool(flip))
    scale = 1.0 / (len(scales) * len(flips))
    predictions, max_probs, hist = raw.argmax_hist(out, gts.contiguous().long(), scale, hist)
    return dict(predictions=predictions, prob_mask=max_probs, hist=hist)


def iou_from_hist(hist):
    """utils/misc.py:110-114 / eval_metrics: per-class IoU = diag / (row + col - diag)."""
    h = hist.double()
    d = torch.diagonal(h)
    return d / (h.sum(0) + h.sum(1) - d).clamp_min(1.0)
