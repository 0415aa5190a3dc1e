"""fp32 restatement of ImageBasedCrossEntropyLoss2d (loss/utils.py:70-118), the criterion of --img_wt_loss, and the
batch with unequal class mixes its tests use. Test infrastructure only, next to oracle/seg_oracle.py, whose criteria
have the same (logits, gts, do_rmi) signature; pinned to the reference by tests/golden/reference_losses.pt."""
import torch
import torch.nn.functional as F

from oracle import seg_oracle as O


def img_wt_class_weights(gts, upper_bound, num_classes=19):
    """Class weights over the whole batch (loss/utils.py:86-99, norm=False): counts b of the labels in
    [0, num_classes), then w = (b != 0) * upper_bound * (1 - b / sum b) + 1, each step an fp32 operation."""
    inside = (gts >= 0) & (gts < num_classes)
    bins = torch.bincount(gts[inside].flatten(), minlength=num_classes)
    share = bins.float() / bins.sum().float()
    return (bins != 0).float() * upper_bound * (1.0 - share) + 1.0


def criterion_img_wt(upper_bound=1.0, batch_weights=False, fp16=False, ignore_index=255, num_classes=19):
    """The criterion as get_loss builds it: one set of class weights from the whole batch (rounded through binary16
    when batch_weights is off and fp16 is on), and the loss is the SUM over images of the class-weighted mean NLL of
    the image's valid pixels. An image without a valid pixel contributes NaN to the loss and nothing to the gradient.
    do_rmi is ignored."""
    def crit(logits, gts, do_rmi=None):
        w = img_wt_class_weights(gts, upper_bound, num_classes).to(logits.device)
        if fp16 and not batch_weights:
            w = w.half().float()
        valid = gts != ignore_index
        y = torch.where(valid, gts, torch.zeros_like(gts))
        nll = -F.log_softmax(logits, dim=1).gather(1, y.unsqueeze(1)).squeeze(1)
        pw = w[y] * valid.float()
        num, den = (pw * nll).flatten(1).sum(1), pw.flatten(1).sum(1)
        per_image = torch.where(den > 0, num / torch.where(den > 0, den, torch.ones_like(den)),
                                torch.full_like(den, float("nan")))
        return per_image.sum()
    return crit


def synth_batch_mixed(n, h, w, seed=0, empty_second=False):
    """oracle.seg_oracle.synth_batch with unequal class mixes: image 1 only uses classes 0-4 (the others are absent
    from it), and with empty_second every label of image 1 is 255 (no valid pixel)."""
    images, gts = O.synth_batch(n, h, w, seed=seed)
    second = gts[1]
    if empty_second:
        second.fill_(255)
    else:
        second.copy_(torch.where(second != 255, second % 5, second))
    return images, gts
