"""RandAugment on the GPU (--rand_augment N,M; b200seg.augment.DeviceTrainTransform, csrc/randaugment_kernels.cu) against
the Pillow replay of the reference's ops (oracle/randaugment_oracle.py, itself pinned to the unmodified reference by
tests/test_randaugment_host.py): every op alone and composed chains are bit-exact - the uint8 crop after RandAugment,
the labels with their fill, and the normalised fp32 image."""
import hashlib
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

pytestmark = pytest.mark.gpu


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _identity_params(h, w, ra):
    """The whole frame as the crop (scale 1, no padding, no flip, no jitter) and the given RandAugment decisions."""
    from b200seg import augment as AUG
    p = AUG.AugParams()
    p.scale, p.rs_w, p.rs_h, p.pad_x, p.pad_y, p.x1, p.y1, p.flip, p.ops = 1.0, w, h, 0, 0, 0, 0, False, []
    p.ra = list(ra)
    return p


def _check(t, img_u8, mask_u8, p, crop):
    from oracle import randaugment_oracle as RO
    ref_img, ref_lab, ref_u8 = RO.reference_chain(img_u8, mask_u8, p, crop, 255, t.mean, t.std)
    img, lab = t(torch.from_numpy(img_u8).cuda(), torch.from_numpy(mask_u8).cuda(), params=p)
    torch.cuda.synchronize()
    got_u8 = t.last_rgb_u8.cpu().numpy()
    assert np.array_equal(got_u8, ref_u8), (p, int((got_u8 != ref_u8).any(-1).sum()))
    assert torch.equal(lab.cpu(), ref_lab), (p, int((lab.cpu() != ref_lab).sum()))
    assert torch.equal(img.cpu(), ref_img), p
    return ref_lab


@pytest.mark.parametrize("hw", [(67, 131), (1024, 2048)])
def test_every_op_alone_matches_pillow(hw):
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    h, w = hw
    img_u8, mask_u8 = AO.synth_frame(h, w, 17)
    t = AUG.DeviceTrainTransform((h, w), color_aug=0.0)
    fills = 0
    for op, (name, lo, hi) in enumerate(AUG.RA_OPS):
        for m in (0, 1, 15, 29, 30):
            val = (float(m) / 30) * float(hi - lo) + lo
            for neg in ((False, True) if op in AUG.RA_SIGNED else (False,)):
                lab = _check(t, img_u8, mask_u8, _identity_params(h, w, [(op, val, neg)]), (h, w))
                fills += int((lab == 255).any())
    assert fills >= 20          # the geometric ops exercise the label fill


def test_composed_chains_match_the_reference_golden():
    """The golden's chains (tests/golden/reference_randaugment.pt: the unmodified reference under fixed seeds), drawn by
    the product and run on the device: the digests of the fp32 image and the labels are the reference's."""
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "reference_randaugment.pt"), weights_only=False)
    full = 0
    for i, (h, w, crop, smin, smax, caug, seed, n, m) in enumerate(gold["chains"]):
        img_u8, mask_u8 = AO.synth_frame(h, w, seed)
        t = AUG.DeviceTrainTransform(tuple(crop), smin, smax, caug, rand_augment="%d,%d" % (n, m))
        random.seed(seed)
        np.random.seed(seed)
        img, lab = t(torch.from_numpy(img_u8).cuda(), torch.from_numpy(mask_u8).cuda())
        assert random.random() == gold["chain_next_random"][i]
        img, lab = img.cpu(), lab.cpu()
        assert (_sha(img.numpy()), _sha(lab.numpy())) == tuple(gold["chain_sha256"][i]), i
        if full < len(gold["image"]) and n >= 2:
            assert torch.equal(img, gold["image"][full]) and torch.equal(lab, gold["label"][full])
            full += 1


def test_long_chains_at_full_size():
    """Every op of augment_list() in one chain on a 1024x2048 crop of a 1024x2048 frame, twice (odd and even number of
    geometric ops: the label ping-pong ends in the caller's buffer either way)."""
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    img_u8, mask_u8 = AO.synth_frame(1024, 2048, 23)
    t = AUG.DeviceTrainTransform((1024, 2048))
    for seed, order in ((1, range(14)), (2, (5, 8, 1, 13, 6, 3, 11, 10))):
        random.seed(seed)
        np.random.seed(seed)
        p = t.draw(2048, 1024)
        p.ra = [(op, (15 / 30) * float(AUG.RA_OPS[op][2] - AUG.RA_OPS[op][1]) + AUG.RA_OPS[op][1], bool(k % 2))
                for k, op in enumerate(order)]
        _check(t, img_u8, mask_u8, p, (1024, 2048))


def test_batch_wrapper_draws_in_loader_order():
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    from oracle import randaugment_oracle as RO
    frames = [AO.synth_frame(96, 160, s) for s in (41, 42, 43, 44)]
    imgs = torch.from_numpy(np.stack([f[0] for f in frames])).pin_memory()
    masks = torch.from_numpy(np.stack([f[1] for f in frames])).pin_memory()
    t = AUG.DeviceTrainTransform((64, 96), rand_augment="3,15")
    random.seed(7)
    np.random.seed(7)
    batch = next(iter(AUG.DeviceAugmentedBatches([(imgs, masks)], t)))
    torch.cuda.synchronize()
    random.seed(7)
    np.random.seed(7)
    for i, (img_u8, mask_u8) in enumerate(frames):
        p = t.draw(160, 96)
        assert len(p.ra) == 3
        ref_img, ref_lab, _ = RO.reference_chain(img_u8, mask_u8, p, (64, 96), 255, t.mean, t.std)
        assert torch.equal(batch["images"][i].cpu(), ref_img) and torch.equal(batch["gts"][i].cpu(), ref_lab), i


def test_histogram_ops_do_not_synchronise():
    """AutoContrast and Equalize build their histogram and LUT on the device: one transform call runs under
    torch.cuda.set_sync_debug_mode("error")."""
    from b200seg import augment as AUG
    from oracle import augment_oracle as AO
    from oracle import randaugment_oracle as RO
    img_u8, mask_u8 = AO.synth_frame(96, 160, 31)
    x, m = torch.from_numpy(img_u8).cuda(), torch.from_numpy(mask_u8).cuda()
    t = AUG.DeviceTrainTransform((64, 96), rand_augment="4,20")
    random.seed(3)
    np.random.seed(3)
    p = t.draw(160, 96)
    p.ra = [(6, 1.0, False), (1, 0.2, True), (8, 1.0, False), (9, 110 * 20 / 30, False)]
    out_i = torch.empty((3, 64, 96), dtype=torch.float32, device="cuda")
    out_l = torch.empty((64, 96), dtype=torch.int64, device="cuda")
    t(x, m, params=p)                  # first call: uploads the label-id table
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t(x, m, params=p, out_image=out_i, out_label=out_l)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    ref_img, ref_lab, _ = RO.reference_chain(img_u8, mask_u8, p, (64, 96), 255, t.mean, t.std)
    assert torch.equal(out_i.cpu(), ref_img) and torch.equal(out_l.cpu(), ref_lab)
