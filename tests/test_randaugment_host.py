"""RandAugment on the device input pipeline (--rand_augment N,M, datasets/randaugment.py), host half, no GPU:
(1) b200seg.augment.draw_params consumes `random` exactly like RandAugment.__call__ and the ops' sign draws, and the
Pillow replay of those decisions (oracle/randaugment_oracle.py) reproduces the UNMODIFIED reference bit for bit
(tests/golden/reference_randaugment.pt), chains and every op alone; (2) the NEAREST source tables and 16.16 matrices the
product hands to its geometric kernel are Pillow's; (3) the argument checks; (4) without RandAugment nothing changes."""
import hashlib
import os
import random
import sys

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

from b200seg import augment as AUG  # noqa: E402
from oracle import augment_oracle as AO  # noqa: E402
from oracle import randaugment_oracle as RO  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "reference_randaugment.pt")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _gold():
    return torch.load(GOLD, weights_only=False)


def test_draws_and_oracle_chain_reproduce_the_reference():
    gold = _gold()
    seen = set()
    for i, (h, w, crop, smin, smax, caug, seed, n, m) in enumerate(gold["chains"]):
        img_u8, mask_u8 = AO.synth_frame(h, w, seed)
        random.seed(seed)
        np.random.seed(seed)
        p = AUG.draw_params(w, h, tuple(crop), smin, smax, caug, rand_augment=(n, m))
        assert random.random() == gold["chain_next_random"][i], (i, p)          # `random` left in the same state
        drawn = [(RO.OPS[op], neg if op in AUG.RA_SIGNED else None) for op, _, neg in p.ra]
        assert drawn == [tuple(x) for x in gold["chain_ops"][i]], (i, p)
        image, label, _ = RO.reference_chain(img_u8, mask_u8, p, tuple(crop), 255, gold["mean"], gold["std"])
        assert (_sha(image.numpy()), _sha(label.numpy())) == tuple(gold["chain_sha256"][i]), (i, p)
        seen.update(RO.OPS[op] for op, _, _ in p.ra)
    assert len(seen) >= 12, seen
    for k in range(len(gold["image"])):
        assert gold["image"][k].dtype == torch.float32 and gold["label"][k].dtype == torch.int64


def test_every_op_alone_reproduces_the_reference():
    gold = _gold()
    h, w, seed = gold["single_frame"]
    img_u8, mask_u8 = AO.synth_frame(h, w, seed)
    lo_hi = {RO.OPS[i]: AUG.RA_OPS[i][1:] for i in range(len(RO.OPS))}
    for name, m, neg, sha_img, sha_mask in gold["single"]:
        op = RO.OPS.index(name)
        lo, hi = lo_hi[name]
        val = (float(m) / 30) * float(hi - lo) + lo
        im, lab = RO.apply_ops(img_u8, mask_u8, [(op, val, neg and op in AUG.RA_SIGNED)])
        assert (_sha(im), _sha(lab.astype(np.uint8))) == (sha_img, sha_mask), (name, m, neg)


def _gather(plan, src, fill):
    """The geometric kernel's NEAREST gather with the product's plan (numpy, test only)."""
    h, w = src.shape[:2]
    ys, xs = np.mgrid[0:h, 0:w]
    if plan["scale"]:
        xi, yi = plan["tab_x"][xs], plan["tab_y"][ys]
    else:
        f = [np.int64(v) for v in plan["fixed"]]
        xi = (f[2] + ys * f[1] + xs * f[0]) >> 16
        yi = (f[5] + ys * f[4] + xs * f[3]) >> 16
    ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
    out = np.full_like(src, fill)
    out[ok] = src[yi[ok], xi[ok]]
    return out


@pytest.mark.parametrize("hw", [(67, 131), (64, 96), (1024, 2048)])
def test_nearest_plans_are_pillows(hw):
    """Labels of every geometric op, and the image of Rotate: both of Pillow's NEAREST paths (per-axis tables for
    translations, 16.16 fixed point for shears and rotations), both signs, fill 255."""
    h, w = hw
    _, mask_u8 = AO.synth_frame(h, w, 5)
    mk = Image.fromarray(mask_u8)
    for op in (1, 2, 3, 4, 5):
        for m in ((0, 1, 15, 29, 30) if h < 1000 else (7, 30)):
            val = (float(m) / 30) * float(AUG.RA_OPS[op][2] - AUG.RA_OPS[op][1]) + AUG.RA_OPS[op][1]
            for neg in (False, True):
                steps = AUG.randaugment_steps([(op, val, neg)], h, w)
                _, ref = RO.apply_ops(np.zeros((h, w, 3), np.uint8), mask_u8, [(op, val, neg)])
                if not steps:                                # Rotate by 0: Pillow returns a copy
                    assert op == 5 and m == 0 and np.array_equal(ref, mask_u8)
                    continue
                (kind, plan), = steps
                assert kind == "affine" and plan["bilinear"] == (op != 5) and plan["scale"] == (op in (3, 4) or m == 0)
                assert np.array_equal(_gather(plan, mask_u8, 255), ref), (op, m, neg)
    assert mk.size == (w, h)


def test_static_luts_are_pillows():
    from PIL import ImageOps
    img_u8, _ = AO.synth_frame(40, 50, 9)
    im = Image.fromarray(img_u8)
    for m in (0, 1, 15, 29, 30):
        for op, ref in ((7, lambda v: ImageOps.invert(im)), (9, lambda v: ImageOps.solarize(im, v)),
                        (10, lambda v: ImageOps.posterize(im, int(v)))):
            lo, hi = AUG.RA_OPS[op][1:]
            val = (float(m) / 30) * float(hi - lo) + lo
            (kind, lut), = AUG.randaugment_steps([(op, val, False)], 40, 50)
            lut = np.asarray(lut).reshape(3, 256)
            got = np.stack([lut[c][img_u8[..., c]] for c in range(3)], -1)
            assert kind == "lut" and np.array_equal(got, np.array(ref(val))), (op, m)


def test_rand_augment_argument_checks():
    assert AUG.parse_rand_augment("2,9") == (2, 9) and AUG.parse_rand_augment((0, 30)) == (0, 30)
    assert AUG.DeviceTrainTransform((64, 96), rand_augment="3,15").rand_augment == (3, 15)
    assert AUG.DeviceTrainTransform((64, 96)).rand_augment is None
    for bad in ("2", "2,9,1", "a,9", "2;9", "", "-1,9", "2,31", "2,-1", (2, 9.0), (2,), (-1, 0), (1, 31), (True, 3)):
        with pytest.raises((ValueError, TypeError)):
            AUG.DeviceTrainTransform((64, 96), rand_augment=bad)


def test_without_rand_augment_the_draws_are_unchanged():
    """rand_augment=None: the same draws and the same `random` / `numpy.random` state as the default chain."""
    for seed in range(5):
        random.seed(seed)
        np.random.seed(seed)
        a = AUG.draw_params(160, 96, (64, 96))
        ra, na = random.random(), np.random.random()
        random.seed(seed)
        np.random.seed(seed)
        b = AUG.draw_params(160, 96, (64, 96), rand_augment=None)
        assert repr(a) == repr(b) and a.ra == [] and (ra, na) == (random.random(), np.random.random())
        t = AUG.DeviceTrainTransform((64, 96))
        assert t.tables(b, 160, 96)["ra"] == []
    # with RandAugment the numpy ColorJitter draws keep their stream
    for seed in range(5):
        random.seed(seed)
        np.random.seed(seed)
        a = AUG.draw_params(160, 96, (64, 96))
        random.seed(seed)
        np.random.seed(seed)
        c = AUG.draw_params(160, 96, (64, 96), rand_augment=(4, 9))
        assert c.ops == a.ops and len(c.ra) == 4
