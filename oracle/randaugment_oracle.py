"""TEST INFRASTRUCTURE (oracle): the reference's --rand_augment N,M (datasets/randaugment.py RandAugment, appended to the
joint transforms after the flip, datasets/__init__.py:83-87) replayed with Pillow for GIVEN random decisions, written from
what each op does to the image / label pair:

    Identity                                    nothing
    ShearX / ShearY / TranslateX / TranslateY   Image.transform(AFFINE, matrix): image BILINEAR, fill black;
                                                labels NEAREST, fill 255 (Translate: the value times the crop size)
    Rotate                                      Image.rotate(degrees): NEAREST (Pillow's default), same fills
    AutoContrast / Invert / Equalize            ImageOps.autocontrast / invert / equalize of the image
    Solarize / Posterize                        ImageOps.solarize(threshold) / posterize(int(bits)) of the image
    Color / Brightness / Sharpness              ImageEnhance.<op>(image).enhance(value)

Pinned by tests/test_randaugment_host.py against the UNMODIFIED reference (tests/golden/reference_randaugment.pt). Only
tests/ may import this module; the product (b200seg/augment.py + csrc/randaugment_kernels.cu) never does."""
import copy

import numpy as np
import torch
from PIL import Image, ImageEnhance, ImageOps

from oracle import augment_oracle as AO

# the op order of augment_list(); random.choices draws the index
OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "AutoContrast", "Invert", "Equalize",
       "Solarize", "Posterize", "Color", "Brightness", "Sharpness")
LABEL_FILL = 255


def apply_op(img, mask, op, val, neg):
    """One op on PIL images (RGB image, L labels); `neg`: the op's sign draw came out > 0.5 (signed ops only)."""
    name = OPS[op]
    v = -val if neg else val

    def affine(m):
        return (img.transform(img.size, Image.AFFINE, m, resample=Image.BILINEAR, fillcolor=(0, 0, 0)),
                mask.transform(mask.size, Image.AFFINE, m, resample=Image.NEAREST, fillcolor=LABEL_FILL))

    if name == "ShearX":
        return affine((1, v, 0, 0, 1, 0))
    if name == "ShearY":
        return affine((1, 0, 0, v, 1, 0))
    if name == "TranslateX":
        return affine((1, 0, v * img.size[0], 0, 1, 0))
    if name == "TranslateY":
        return affine((1, 0, 0, 0, 1, v * img.size[1]))
    if name == "Rotate":
        return img.rotate(v, fillcolor=(0, 0, 0)), mask.rotate(v, resample=Image.NEAREST, fillcolor=LABEL_FILL)
    if name == "AutoContrast":
        return ImageOps.autocontrast(img), mask
    if name == "Invert":
        return ImageOps.invert(img), mask
    if name == "Equalize":
        return ImageOps.equalize(img), mask
    if name == "Solarize":
        return ImageOps.solarize(img, v), mask
    if name == "Posterize":
        return ImageOps.posterize(img, int(v)), mask
    if name == "Color":
        return ImageEnhance.Color(img).enhance(v), mask
    if name == "Brightness":
        return ImageEnhance.Brightness(img).enhance(v), mask
    if name == "Sharpness":
        return ImageEnhance.Sharpness(img).enhance(v), mask
    return img, mask


def apply_ops(img_u8, label, ra):
    """uint8 [h,w,3] + integer labels [h,w] (0..255) -> (uint8 [h,w,3], int64 labels) after the ops of `ra`
    ((op, value, negated) in order, b200seg.augment.AugParams.ra)."""
    img, mask = Image.fromarray(np.ascontiguousarray(img_u8)), Image.fromarray(np.asarray(label, dtype=np.uint8))
    for op, val, neg in ra:
        img, mask = apply_op(img, mask, op, val, neg)
    return np.array(img), np.array(mask).astype(np.int64)


def reference_chain(img_u8, mask_u8, p, crop_hw, ignore_label=255, mean=(0.485, 0.456, 0.406),
                    std=(0.229, 0.224, 0.225), id_to_trainid=None, full_size=False):
    """augment_oracle.reference_chain with RandAugment between the flip and the colour jitter. Returns (fp32 tensor
    [3,th,tw], int64 tensor [th,tw], uint8 crop [th,tw,3] after RandAugment, before the colour jitter)."""
    q = copy.copy(p)
    q.ops = []
    _, lab, crop_u8 = AO.reference_chain(img_u8, mask_u8, q, crop_hw, ignore_label, mean, std, id_to_trainid, full_size)
    crop_u8, lab = apply_ops(crop_u8, lab.numpy(), p.ra)
    img = Image.fromarray(crop_u8)
    for kind, factor in p.ops:                       # ColorJitter, as augment_oracle.reference_chain applies it
        if kind == 0:
            img = ImageEnhance.Brightness(img).enhance(factor)
        elif kind == 1:
            img = ImageEnhance.Contrast(img).enhance(factor)
        elif kind == 2:
            img = ImageEnhance.Color(img).enhance(factor)
        else:
            img = AO.adjust_hue(img, factor)
    t = torch.from_numpy(np.array(img)).permute(2, 0, 1).contiguous().to(torch.float32).div(255)     # ToTensor
    m, s = torch.as_tensor(mean, dtype=torch.float32), torch.as_tensor(std, dtype=torch.float32)
    t = t.sub_(m[:, None, None]).div_(s[:, None, None])                                              # Normalize
    return t, torch.from_numpy(lab), crop_u8
