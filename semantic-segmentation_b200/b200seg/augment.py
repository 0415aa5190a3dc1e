"""Device-side training input pipeline (SURVEY.md §8 row f4): the reference's per-sample transform chain

    RandomSizeAndCrop (transforms/joint_transforms.py:433-472: PIL BICUBIC resize of the image, NEAREST of the mask,
    RandomCrop with ImageOps.expand padding :143-182) -> RandomHorizontallyFlip (:276-281) -> ColorJitter
    (transforms/transforms.py:297-362: ImageEnhance brightness / contrast / saturation + HSV hue shift, random order)
    -> ToTensor -> Normalize (datasets/__init__.py:102-104) and MaskToTensor, after the label-id remap of
    datasets/base_loader.py:177-181

as three sm_90a kernels (csrc/augment_kernels.cu) on the DECODED uint8 frame, so a 1024x2048 crop costs microseconds on
the GPU instead of a PIL worker process per GPU. Results are bit-exact with PIL 12 on the uint8 stages and with
torchvision's ToTensor / Normalize arithmetic on the fp32 stage (tests/test_gpu_augment.py): the host side below draws
the random parameters with the reference's own generator calls in the reference's order (`random` for the geometry,
`numpy.random` for the colour jitter), builds PIL's fixed-point resampling tables exactly as Pillow's
precompute_coeffs / normalize_coeffs_8bpc do (double arithmetic, 22 fractional bits) and hands them to the kernels.
There is no CPU image path here: the tables are a few KB of integers, the pixels never touch the host."""
import math
import random

import numpy as np
import torch

from . import raw

PRECISION_BITS = 32 - 8 - 2      # Pillow's 8 bits-per-channel resampler
OP_BRIGHTNESS, OP_CONTRAST, OP_SATURATION, OP_HUE = 0, 1, 2, 3


# ----------------------------------------------------------------------------------------------- Pillow's tables
def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def bicubic_tables(in_size, out_size, lo=0, hi=None):
    """Pillow's ImagingResample coefficient tables (BICUBIC, 8 bpc) of output positions [lo, hi): int32 kk[hi-lo, ksize]
    (22-bit fixed point, rows zero padded) and int32 bounds[hi-lo, 2] = (first source index, tap count).
    Vectorised over the output positions; every double operation and the left-to-right order of the normalising sum are
    those of precompute_coeffs / normalize_coeffs_8bpc (tests/test_augment_host.py compares with Image.resize)."""
    hi = out_size if hi is None else hi
    scale = filterscale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    n = max(0, hi - lo)
    kk = np.zeros((n, ksize), dtype=np.int32)
    bounds = np.zeros((n, 2), dtype=np.int32)
    if n == 0:
        return kk, bounds
    ss = 1.0 / filterscale
    center = (np.arange(lo, hi, dtype=np.float64) + 0.5) * scale
    xmin = np.trunc(center - support + 0.5).astype(np.int64)          # (int) of a double: truncation
    xmin = np.maximum(xmin, 0)
    xmax = np.trunc(center + support + 0.5).astype(np.int64)
    xmax = np.minimum(xmax, in_size) - xmin
    a = -0.5
    w = np.zeros((n, ksize), dtype=np.float64)
    ww = np.zeros(n, dtype=np.float64)
    for x in range(ksize):                                             # taps in order: ww accumulates left to right
        live = x < xmax
        t = np.abs((x + xmin - center + 0.5) * ss)
        f = np.where(t < 1.0, ((a + 2.0) * t - (a + 3.0)) * t * t + 1, np.where(t < 2.0, (((t - 5) * t + 8) * t - 4) * a, 0.0))
        f = np.where(live, f, 0.0)
        w[:, x] = f
        ww = np.where(live, ww + f, ww)
    nz = ww != 0.0
    w = np.where(nz[:, None], w / np.where(nz, ww, 1.0)[:, None], w)
    fixed = np.where(w < 0, np.trunc(-0.5 + w * (1 << PRECISION_BITS)), np.trunc(0.5 + w * (1 << PRECISION_BITS)))
    kk[:] = np.where(np.arange(ksize)[None, :] < xmax[:, None], fixed, 0).astype(np.int32)
    bounds[:, 0], bounds[:, 1] = xmin, xmax
    return kk, bounds


def nearest_table(in_size, out_size, lo=0, hi=None):
    """Source index of every NEAREST output position in [lo, hi): Pillow's affine scaler accumulates xo += in/out in
    double starting at in/out * 0.5 (the accumulated value, not (x + 0.5) * scale, decides ties); numpy's cumsum adds
    left to right in double, i.e. the same sequence of roundings."""
    hi = out_size if hi is None else hi
    if hi <= lo:
        return np.zeros(0, dtype=np.int32)
    a0 = float(in_size) / out_size
    steps = np.full(hi, a0, dtype=np.float64)
    steps[0] = a0 * 0.5
    xo = np.cumsum(steps)
    return np.clip(np.floor(xo[lo:hi]), 0, in_size - 1).astype(np.int32)


# ----------------------------------------------------------------------------------------------- parameters
class AugParams:
    """One sample's random decisions, drawn like the reference draws them."""
    __slots__ = ("scale", "rs_w", "rs_h", "pad_x", "pad_y", "x1", "y1", "flip", "ops")

    def __repr__(self):
        return "AugParams(%s)" % ", ".join("%s=%r" % (k, getattr(self, k)) for k in self.__slots__)


def draw_params(w, h, crop_hw, scale_min=0.5, scale_max=2.0, color_aug=0.25, centroid=None, pre_size=None,
                full_size=False, rng=random, nprng=np.random):
    """Consumes `random` / `numpy.random` exactly like RandomSizeAndCrop.__call__ -> RandomCrop.__call__ (nopad=False,
    TRANSLATE_AUG_FIX off) -> RandomHorizontallyFlip -> ColorJitter.get_params do for one sample."""
    p = AugParams()
    scale_amt = rng.uniform(scale_min, scale_max)                      # joint_transforms.py:446
    if pre_size is not None:                                           # :448-456
        scale_amt *= pre_size / (w if w > h else h)
    th, tw = (h, w) if full_size else crop_hw                          # :458-459 (crop.size = (h, w) of the input)
    p.scale = scale_amt
    p.rs_w, p.rs_h = int(w * scale_amt), int(h * scale_amt)            # :461
    if centroid is not None:
        centroid = [int(c * scale_amt) for c in centroid]              # :463-464
    rw, rh = p.rs_w, p.rs_h
    p.pad_x = p.pad_y = 0
    p.x1 = p.y1 = 0
    if not (rw == tw and rh == th):                                    # RandomCrop.__call__ :143-182
        if th > rh:
            p.pad_y = (th - rh) // 2 + 1
        if tw > rw:
            p.pad_x = (tw - rw) // 2 + 1
        rw, rh = rw + 2 * p.pad_x, rh + 2 * p.pad_y
        if centroid is not None:                                       # crop_in_image :104-126
            c_x, c_y = centroid
            x1 = rng.randint(c_x - tw, c_x)
            p.x1 = min(rw - tw, max(0, x1))
            y1 = rng.randint(c_y - th, c_y)
            p.y1 = min(rh - th, max(0, y1))
        else:
            p.x1 = 0 if rw == tw else rng.randint(0, rw - tw)
            p.y1 = 0 if rh == th else rng.randint(0, rh - th)
    p.flip = rng.random() < 0.5                                        # :278
    ops = []
    if color_aug and color_aug > 0:                                    # transforms.py:326-348
        ops.append((OP_BRIGHTNESS, float(nprng.uniform(max(0, 1 - color_aug), 1 + color_aug))))
        ops.append((OP_CONTRAST, float(nprng.uniform(max(0, 1 - color_aug), 1 + color_aug))))
        ops.append((OP_SATURATION, float(nprng.uniform(max(0, 1 - color_aug), 1 + color_aug))))
        ops.append((OP_HUE, float(nprng.uniform(-color_aug, color_aug))))
        nprng.shuffle(ops)
    p.ops = [(int(k), float(f)) for k, f in ops]
    return p


# ----------------------------------------------------------------------------------------------- the transform
class DeviceTrainTransform:
    """image uint8 [H, W, 3] + label-id mask uint8 [H, W] (CUDA tensors) -> (fp32 [3, th, tw] normalised image, int64
    [th, tw] train-id labels), the outputs of the reference's train_joint_transform_list + train_input_transform +
    target_transform (datasets/__init__.py:72-108) for the same random decisions."""

    def __init__(self, crop_hw, scale_min=0.5, scale_max=2.0, color_aug=0.25, ignore_label=255,
                 mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), id_to_trainid=None, pre_size=None,
                 full_size=False):
        self.crop_hw = tuple(crop_hw)
        self.scale_min, self.scale_max, self.color_aug = scale_min, scale_max, color_aug
        self.ignore_label = int(ignore_label)
        self.mean, self.std = tuple(float(m) for m in mean), tuple(float(s) for s in std)
        self.pre_size, self.full_size = pre_size, full_size
        lut = np.arange(256, dtype=np.uint8)
        if id_to_trainid:                      # datasets/base_loader.py:177-181 (applied to the decoded label ids)
            for k, v in id_to_trainid.items():
                if 0 <= int(k) < 256:
                    lut[int(k)] = int(v) & 0xFF
        self._lut_host = torch.from_numpy(lut)
        self._lut = None

    def draw(self, w, h, centroid=None, rng=random, nprng=np.random):
        return draw_params(w, h, self.crop_hw, self.scale_min, self.scale_max, self.color_aug, centroid, self.pre_size,
                           self.full_size, rng, nprng)

    def tables(self, p, w, h):
        """Resampling tables of the crop window only (host integers, a few KB)."""
        th, tw = (h, w) if self.full_size else self.crop_hw
        # output column c (before the flip) shows padded-resized column x1 + c, i.e. resized column x1 + c - pad_x
        lo_x, hi_x = max(0, p.x1 - p.pad_x), min(p.rs_w, p.x1 - p.pad_x + tw)
        lo_y, hi_y = max(0, p.y1 - p.pad_y), min(p.rs_h, p.y1 - p.pad_y + th)
        kh, bh = bicubic_tables(w, p.rs_w, lo_x, max(lo_x, hi_x))
        kv, bv = bicubic_tables(h, p.rs_h, lo_y, max(lo_y, hi_y))
        nx = nearest_table(w, p.rs_w, lo_x, max(lo_x, hi_x))
        ny = nearest_table(h, p.rs_h, lo_y, max(lo_y, hi_y))
        return dict(kh=kh, bh=bh, kv=kv, bv=bv, nx=nx, ny=ny, lo_x=lo_x, lo_y=lo_y, n_x=max(0, hi_x - lo_x),
                    n_y=max(0, hi_y - lo_y), th=th, tw=tw)

    def __call__(self, image_u8, mask_u8, params=None, centroid=None, out_image=None, out_label=None):
        assert image_u8.is_cuda and image_u8.dtype == torch.uint8 and image_u8.dim() == 3 and image_u8.shape[2] == 3
        assert mask_u8.is_cuda and mask_u8.dtype == torch.uint8 and tuple(mask_u8.shape) == tuple(image_u8.shape[:2])
        h, w = image_u8.shape[:2]
        p = params if params is not None else self.draw(w, h, centroid)
        t = self.tables(p, w, h)
        dev = image_u8.device
        if self._lut is None or self._lut.device != dev:
            self._lut = self._lut_host.to(dev)
        img, lab, self.last_rgb_u8 = raw.augment(image_u8.contiguous(), mask_u8.contiguous(), p, t, self._lut,
                                                 self.ignore_label, self.mean, self.std, out_image, out_label)
        return img, lab


class DeviceAugmentedBatches:
    """Wraps an iterable of decoded batches - (images uint8 [N, H, W, 3], label ids uint8 [N, H, W]) host (pinned) or CUDA
    tensors, optionally a third item with one centroid (x, y) or None per sample (class-uniform sampling,
    datasets/uniform.py) - and yields {'images': fp32 [N, 3, th, tw], 'gts': int64 [N, th, tw]} on the device, the dict
    the reference's training loop feeds the network (train.py:485-488). The random decisions of sample i are drawn on
    the host in loader order, like the reference's dataset workers draw them per sample."""

    def __init__(self, batches, transform, device="cuda"):
        self.batches, self.t, self.device = batches, transform, torch.device(device)

    def __iter__(self):
        for batch in self.batches:
            imgs, masks = batch[0], batch[1]
            cents = batch[2] if len(batch) > 2 else [None] * imgs.shape[0]
            imgs = imgs.to(self.device, non_blocking=True)
            masks = masks.to(self.device, non_blocking=True)
            n, h, w = masks.shape
            th, tw = (h, w) if self.t.full_size else self.t.crop_hw
            out_i = torch.empty((n, 3, th, tw), dtype=torch.float32, device=self.device)
            out_l = torch.empty((n, th, tw), dtype=torch.int64, device=self.device)
            for i in range(n):
                self.t(imgs[i], masks[i], centroid=cents[i], out_image=out_i[i], out_label=out_l[i])
            yield {"images": out_i, "gts": out_l}
