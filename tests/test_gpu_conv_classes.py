"""Every tensor-core convolution configuration the W48 two-scale training step launches, checked against float64.

A launch of conv_igemm_kernel, conv3x3_halo_kernel or wgrad_igemm_kernel runs one of several configurations the host
planners pick per shape: the Cout tile BN (which decides the wgmma widths of the n64 groups and the n16/n32/n48 tail),
the co-resident (OCC 2, <= 128 accumulator columns) or full-SM (OCC 1) build, the channel chunk KC of the per-tap kernel,
resident or streamed weights and the ring depth of the halo kernel, and for the weight gradient the N tile, the taps per
group and a direct or pixel-split decomposition. CASES holds, for every configuration key of the traced step (both scale
passes, forward, stride-1 data gradient and weight gradient, without and with the SyncBN shared-memory reserve), the
smallest shape found that reaches it under the default planner settings. tests/test_conv_plans.py checks on the CPU that
every case still plans to its key and that the keys cover the step.

Every case is compared with F.conv2d and its autograd in float64 on the GPU, computed from exactly the bf16 inputs, with
bounds tied to fp32 accumulation (A = the same convolution of |inputs|):
  * bf16 outputs: |y - r| <= ulp_bf16(r) + ACC_REL * A elementwise, and at most MISMATCH_MAX of the elements differ
    from round_bf16(r) (a systematic error of ~1e-4 relative flips many roundings without breaking the first bound);
  * fp32 outputs: |y - r| <= ACC_REL * A;
  * weight gradients: the increment of a random non-zero accumulator within WGRAD_NORM of r normwise (a dropped pixel
    tile shows up there) and within WGRAD_ELEM * A elementwise;
  * statistics (per-CTA partials and the fp64 cells): within STATS_REL of the float64 sums of the stored outputs.
Outputs go into a slice of a NaN-filled wider buffer with a NaN guard behind it: every element outside the slice must
keep its NaN bits (edge-tile rows and column tails are masked), every element inside must be finite. Inputs carry NaN
in the channels past their extent, which the kernels must never read. Every launch runs twice and must give the same bits.
Forward cases run every epilogue: statistics partials, bias + fp64 cells, bias + addend + partials, BatchNorm affine,
and affine + addend + ReLU; data-gradient cases run with and without an addend.
"""
import contextlib
import ctypes
import zlib

import pytest

from b200seg import _lib

SYNCBN_RESERVE = 12288      # shared memory per SM the planners leave free in SyncBN mode (b200seg/p2p.py)

# Largest values observed over all cases on one H100 80GB HBM3 (700 W power limit); every bound keeps >= 4x headroom:
#   accumulation error / A, bf16 and fp32 outputs   6.9e-7 (igemm), 5.4e-7 (halo)     -> ACC_REL 2^-18 = 3.8e-6
#   share of bf16 outputs != round_bf16(reference)  0.38 % (halo, Cin 720)             -> MISMATCH_MAX 1.6 %
#   weight gradient normwise / elementwise / A      1.2e-6 / 1.9e-7                    -> 5e-6 / 2^-20 = 9.5e-7
#   statistics relative to sum |y| (or sum y^2)     1.3e-7                             -> 1e-6
# Scaling the output columns >= 192 by 1 + 2^-9 (an error tests/test_gpu_ops.py passes) makes 9-23 % of the outputs of
# every wide case differ from round_bf16(reference).
ACC_REL = 2.0 ** -18
MISMATCH_MAX = 0.016
WGRAD_NORM = 5e-6
WGRAD_ELEM = 2.0 ** -20
STATS_REL = 1e-6

# (entry point, (n, h, w, cin, cout, k, stride) of the forward convolution, smem reserve, configuration key)
#   fwd / dgrad key: (kernel, BN, CTAs per SM, KC (igemm) or 'res' / weight-ring slots (halo), more tiles than CTAs)
#   wgrad key:       (N tile, width of the last N tile mod 64, taps per group, direct / split, dy blocks of the last M tile)
# A data-gradient cout is the padded extent roundup8(cout) the step hands over.
CASES = [
    ('fwd', (1, 17, 421, 720, 512, 3, 1), 0, ('halo', 256, 1, 4, True)),
    ('fwd', (1, 49, 397, 256, 256, 3, 1), 0, ('halo', 256, 1, 5, True)),
    ('fwd', (1, 9, 9, 192, 192, 3, 1), 0, ('halo', 32, 2, 8, False)),
    ('fwd', (1, 33, 181, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', False)),
    ('fwd', (1, 69, 421, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', True)),
    ('fwd', (1, 17, 41, 384, 384, 3, 1), SYNCBN_RESERVE, ('halo', 48, 2, 5, False)),
    ('fwd', (1, 17, 41, 384, 384, 3, 1), 0, ('halo', 48, 2, 6, False)),
    ('fwd', (1, 33, 117, 96, 96, 3, 1), 0, ('halo', 48, 2, 8, False)),
    ('fwd', (1, 69, 421, 256, 48, 3, 1), 0, ('halo', 48, 2, 8, True)),
    ('fwd', (1, 33, 181, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, False)),
    ('fwd', (1, 69, 421, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, True)),
    ('fwd', (1, 33, 181, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, False)),
    ('fwd', (1, 69, 421, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, True)),
    ('fwd', (1, 33, 117, 192, 192, 3, 1), SYNCBN_RESERVE, ('halo', 96, 1, 8, False)),
    ('fwd', (1, 33, 237, 96, 96, 3, 1), 0, ('halo', 96, 2, 4, False)),
    ('fwd', (1, 49, 229, 64, 256, 1, 1), 0, ('igemm', 128, 1, 64, True)),
    ('fwd', (1, 9, 9, 96, 96, 3, 2), 0, ('igemm', 16, 2, 32, False)),
    ('fwd', (1, 9, 9, 256, 1, 1, 1), 0, ('igemm', 16, 2, 64, False)),
    ('fwd', (1, 237, 133, 256, 1, 1, 1), 0, ('igemm', 16, 2, 64, True)),
    ('fwd', (1, 181, 33, 720, 720, 1, 1), 0, ('igemm', 240, 1, 64, True)),
    ('fwd', (1, 229, 245, 64, 256, 1, 1), 0, ('igemm', 256, 1, 64, True)),
    ('fwd', (1, 9, 9, 96, 384, 3, 2), 0, ('igemm', 32, 2, 32, False)),
    ('fwd', (1, 9, 9, 48, 384, 3, 2), 0, ('igemm', 32, 2, 64, False)),
    ('fwd', (1, 237, 133, 256, 19, 1, 1), 0, ('igemm', 32, 2, 64, True)),
    ('fwd', (1, 33, 213, 96, 48, 1, 1), 0, ('igemm', 48, 2, 32, False)),
    ('fwd', (1, 41, 117, 192, 96, 1, 1), 0, ('igemm', 48, 2, 64, False)),
    ('fwd', (1, 837, 133, 16, 64, 3, 2), 0, ('igemm', 64, 2, 16, True)),
    ('fwd', (1, 33, 213, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, False)),
    ('fwd', (1, 237, 133, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, True)),
    ('fwd', (1, 117, 165, 96, 192, 3, 2), 0, ('igemm', 96, 2, 32, False)),
    ('fwd', (1, 213, 133, 48, 96, 3, 2), 0, ('igemm', 96, 2, 64, False)),
    ('dgrad', (1, 49, 197, 256, 48, 3, 1), 0, ('halo', 128, 1, 8, True)),
    ('dgrad', (1, 17, 317, 720, 512, 3, 1), 0, ('halo', 240, 1, 4, True)),
    ('dgrad', (1, 49, 213, 512, 256, 3, 1), 0, ('halo', 256, 1, 4, True)),
    ('dgrad', (1, 85, 445, 256, 48, 3, 1), 0, ('halo', 256, 1, 5, True)),
    ('dgrad', (1, 9, 9, 192, 192, 3, 1), 0, ('halo', 32, 2, 8, False)),
    ('dgrad', (1, 33, 181, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', False)),
    ('dgrad', (1, 69, 421, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', True)),
    ('dgrad', (1, 17, 41, 384, 384, 3, 1), SYNCBN_RESERVE, ('halo', 48, 2, 5, False)),
    ('dgrad', (1, 17, 41, 384, 384, 3, 1), 0, ('halo', 48, 2, 6, False)),
    ('dgrad', (1, 33, 117, 96, 96, 3, 1), 0, ('halo', 48, 2, 8, False)),
    ('dgrad', (1, 33, 181, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, False)),
    ('dgrad', (1, 69, 421, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, True)),
    ('dgrad', (1, 33, 181, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, False)),
    ('dgrad', (1, 69, 421, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, True)),
    ('dgrad', (1, 33, 117, 192, 192, 3, 1), SYNCBN_RESERVE, ('halo', 96, 1, 8, False)),
    ('dgrad', (1, 33, 237, 96, 96, 3, 1), 0, ('halo', 96, 2, 4, False)),
    ('dgrad', (1, 49, 229, 256, 8, 1, 1), 0, ('igemm', 128, 1, 64, True)),
    ('dgrad', (1, 41, 437, 720, 24, 1, 1), 0, ('igemm', 240, 1, 64, True)),
    ('dgrad', (1, 57, 453, 512, 24, 1, 1), 0, ('igemm', 256, 1, 64, True)),
    ('dgrad', (1, 9, 9, 192, 96, 1, 1), 0, ('igemm', 32, 2, 32, False)),
    ('dgrad', (1, 9, 9, 192, 48, 1, 1), 0, ('igemm', 32, 2, 64, False)),
    ('dgrad', (1, 9, 9, 384, 96, 1, 1), 0, ('igemm', 48, 2, 32, False)),
    ('dgrad', (1, 9, 9, 384, 48, 1, 1), 0, ('igemm', 48, 2, 64, False)),
    ('dgrad', (1, 33, 213, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, False)),
    ('dgrad', (1, 237, 133, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, True)),
    ('dgrad', (1, 41, 117, 192, 96, 1, 1), 0, ('igemm', 96, 2, 32, False)),
    ('dgrad', (1, 41, 117, 192, 48, 1, 1), 0, ('igemm', 96, 2, 64, False)),
    ('wgrad', (1, 49, 229, 256, 1, 1, 1), 0, ('wgrad', 128, 0, 1, 'split', 1)),
    ('wgrad', (1, 69, 133, 256, 96, 3, 2), 0, ('wgrad', 128, 0, 1, 'split', 2)),
    ('wgrad', (1, 9, 9, 720, 512, 3, 1), 0, ('wgrad', 128, 16, 2, 'direct', 2)),
    ('wgrad', (1, 33, 197, 96, 192, 3, 2), 0, ('wgrad', 128, 32, 1, 'split', 1)),
    ('wgrad', (1, 41, 85, 96, 96, 3, 1), 0, ('wgrad', 128, 32, 1, 'split', 2)),
    ('wgrad', (1, 125, 245, 96, 96, 3, 1), 0, ('wgrad', 128, 32, 2, 'split', 2)),
    ('wgrad', (1, 221, 197, 512, 19, 1, 1), 0, ('wgrad', 256, 0, 1, 'split', 1)),
    ('wgrad', (1, 17, 165, 512, 256, 3, 1), 0, ('wgrad', 256, 0, 1, 'split', 2)),
    ('wgrad', (1, 57, 485, 720, 19, 1, 1), 0, ('wgrad', 256, 16, 1, 'split', 1)),
    ('wgrad', (1, 221, 17, 720, 720, 1, 1), 0, ('wgrad', 256, 16, 1, 'split', 2)),
    ('wgrad', (1, 9, 9, 384, 48, 1, 1), 0, ('wgrad', 64, 0, 1, 'direct', 1)),
    ('wgrad', (1, 9, 9, 384, 96, 1, 1), 0, ('wgrad', 64, 0, 1, 'direct', 2)),
    ('wgrad', (1, 49, 17, 64, 64, 1, 1), 0, ('wgrad', 64, 0, 1, 'split', 1)),
    ('wgrad', (1, 33, 17, 64, 256, 1, 1), 0, ('wgrad', 64, 0, 1, 'split', 2)),
    ('wgrad', (1, 9, 9, 384, 384, 3, 1), 0, ('wgrad', 64, 0, 2, 'direct', 2)),
    ('wgrad', (1, 229, 453, 64, 64, 3, 2), 0, ('wgrad', 64, 0, 2, 'split', 1)),
    ('wgrad', (1, 25, 245, 256, 48, 3, 1), 0, ('wgrad', 64, 0, 3, 'split', 1)),
    ('wgrad', (1, 165, 229, 256, 96, 3, 2), 0, ('wgrad', 64, 0, 3, 'split', 2)),
    ('wgrad', (1, 981, 293, 16, 64, 3, 2), 0, ('wgrad', 64, 16, 9, 'split', 1)),
    ('wgrad', (1, 9, 9, 96, 192, 3, 2), 0, ('wgrad', 64, 32, 1, 'direct', 1)),
    ('wgrad', (1, 9, 9, 96, 384, 3, 2), 0, ('wgrad', 64, 32, 1, 'direct', 2)),
    ('wgrad', (1, 49, 17, 96, 48, 1, 1), 0, ('wgrad', 64, 32, 1, 'split', 1)),
    ('wgrad', (1, 49, 101, 96, 96, 3, 2), 0, ('wgrad', 64, 32, 1, 'split', 2)),
    ('wgrad', (1, 9, 9, 48, 384, 3, 2), 0, ('wgrad', 64, 48, 1, 'direct', 2)),
    ('wgrad', (1, 117, 33, 48, 48, 3, 2), 0, ('wgrad', 64, 48, 1, 'split', 1)),
    ('wgrad', (1, 17, 165, 48, 96, 3, 2), 0, ('wgrad', 64, 48, 1, 'split', 2)),
    ('wgrad', (1, 117, 229, 48, 192, 3, 2), 0, ('wgrad', 64, 48, 2, 'split', 1)),
    ('wgrad', (1, 41, 341, 48, 48, 3, 1), 0, ('wgrad', 64, 48, 3, 'split', 1)),
    ('wgrad', (1, 181, 325, 48, 96, 3, 2), 0, ('wgrad', 64, 48, 3, 'split', 2)),
]

# Launches no plan query reports: stride-2 data gradients run as four sub-lattice launches of conv_igemm_kernel (odd
# extents give sub-lattices of different sizes), and the fp32 logit head (512 -> 19, bias, out_ld 20 in the step).
EXTRA_CASES = [
    ("dgrad", (1, 69, 133, 48, 96, 3, 2), 0, None),
    ("dgrad", (1, 101, 205, 64, 64, 3, 2), 0, None),
    ("dgrad", (1, 37, 67, 256, 96, 3, 2), 0, None),
    ("fwd_fp32", (1, 33, 69, 512, 19, 1, 1), 0, None),
]


def _desc(n, h, w, cin, cout, k, s):
    d = _lib.ConvDesc()
    d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride, d.pad = n, h, w, cin, cout, k, s, (k - 1) // 2
    d.x_ld, d.y_ld = cin, (cout + 7) // 8 * 8
    return d


def config_key(entry, shape):
    """Configuration key of a launch under the current shared-memory reserve, from the host-only plan queries."""
    L = _lib.lib()
    d = _desc(*shape)
    cin, cout = shape[3], shape[4]
    if entry == "wgrad":
        out = (ctypes.c_int32 * 10)()
        assert L.b200seg_conv2d_wgrad_plan_info(ctypes.byref(d), out) == 0, shape
        ntile, n_tiles, tpg, _groups, splits, m_tiles = list(out)[:6]
        return ("wgrad", ntile, (cin - (n_tiles - 1) * ntile) % 64, tpg, "direct" if splits == 1 else "split",
                2 if cout - (m_tiles - 1) * 128 > 64 else 1)
    out = (ctypes.c_int32 * 12)()
    assert L.b200seg_conv2d_plan_info(ctypes.byref(d), 0 if entry == "fwd" else 1, out) == 0, (entry, shape)
    kern, bn, _nt, grid, _smem, _depth, occ, _acc, resident, b_slots, kc, tiles = list(out)
    return ("halo" if kern else "igemm", bn, occ, ("res" if resident else b_slots) if kern else kc, tiles > grid)


@contextlib.contextmanager
def smem_reserve(nbytes):
    """The reserve is process-global: set it for the block, back to the default (0) afterwards."""
    L = _lib.lib()
    assert L.b200seg_set_smem_reserve(nbytes) == 0
    try:
        yield
    finally:
        L.b200seg_set_smem_reserve(0)


def _case_id(case):
    entry, (n, h, w, cin, cout, k, s), res, _key = case
    return "%s-%dx%dx%d-c%d-%d-k%ds%d%s" % (entry, n, h, w, cin, cout, k, s, "-syncbn" if res else "")


# ------------------------------------------------------------------------------------------------------------ GPU part
def _torch():
    import torch
    import torch.nn.functional as F
    from b200seg import raw
    return torch, F, raw


def _seed(case):
    return zlib.crc32(_case_id(case).encode())


def _randn(shape, seed, scale=1.0):
    torch, _, _ = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) * scale


def _nan_bits(dtype):
    torch, _, _ = _torch()
    itype = torch.int16 if dtype == torch.bfloat16 else torch.int32
    return itype, torch.full((1,), float("nan"), dtype=dtype, device="cuda").view(itype)


class Canvas:
    """NaN-filled [n, h, w, ld] buffer (ld = roundup8(c) + 16) plus a NaN guard behind it; the tensor under test is the
    slice [..., 8:8 + c]. A masked tile can overrun the last image by at most 2 x 16 rows + 1 tile (stride-2 lattices)."""

    def __init__(self, n, h, w, c, dtype):
        torch, _, _ = _torch()
        self.ld = (c + 7) // 8 * 8 + 16
        self.c = c
        body = n * h * w * self.ld
        self.flat = torch.full((body + (34 * w + 64) * self.ld,), float("nan"), dtype=dtype, device="cuda")
        self.full = self.flat[:body].view(n, h, w, self.ld)
        self.y = self.full[..., 8:8 + c]

    def check(self, what):
        torch, _, _ = _torch()
        itype, nan = _nan_bits(self.flat.dtype)
        assert bool(torch.isfinite(self.y).all()), "%s: non-finite or unwritten output element" % what
        outside = torch.ones(self.flat.shape, dtype=torch.bool, device="cuda")
        outside[: self.full.numel()].view(self.full.shape)[..., 8:8 + self.c] = False
        bad = int((self.flat.view(itype)[outside] != nan).sum())
        assert bad == 0, "%s: %d elements outside the output slice were written" % (what, bad)


def _input(n, h, w, c, seed, pad_value=float("nan"), real=None):
    """bf16 [n, h, w, c] whose pixel pitch is roundup8(c) + 8; channels [real, c) are zero (the padded channels of a
    data-gradient operand) and the channels past c hold pad_value."""
    torch, _, _ = _torch()
    buf = torch.full((n, h, w, (c + 7) // 8 * 8 + 8), pad_value, dtype=torch.bfloat16, device="cuda")
    real = c if real is None else real
    buf[..., :real] = _randn((n, h, w, real), seed).to(torch.bfloat16)
    buf[..., real:c] = 0
    return buf[..., :c]


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _ulp_bf16(r):
    torch, _, _ = _torch()
    _m, e = torch.frexp(r)
    return torch.where(r == 0, torch.zeros_like(r), torch.ldexp(torch.ones_like(r), e - 8))


def _check_values(y, ref, A, other, what, bf16=True, pre=None):
    """y (bf16 or fp32) against the float64 reference ref; A bounds the accumulation error, other (|bias| + |shift| +
    |addend|) the fp32 epilogue arithmetic; pre = the reference before a ReLU (its ulp is the larger). Also prints the
    accumulation error alone: what is left of |y - r| after the rounding to bf16 (ulp(y) / 2), over A."""
    torch, _, _ = _torch()
    yd = y.double()
    err = (yd - ref).abs()
    bound = ACC_REL * A + 2.0 ** -20 * other
    acc = err
    if bf16:
        bound = bound + _ulp_bf16(ref if pre is None else pre)
        acc = (err - 0.5 * torch.maximum(_ulp_bf16(yd), _ulp_bf16(ref if pre is None else pre))).clamp_min(0)
    ratio = float((err / bound.clamp_min(1e-300)).max())
    acc_rel = float((acc / A.clamp_min(1e-300)).max())
    mism = float((y != ref.to(y.dtype)).double().mean()) if bf16 else 0.0
    print("%-50s max err/bound %.4f  accumulation err/A %.2e  rounding mismatches %.4f%%" %
          (what, ratio, acc_rel, 100 * mism))
    assert ratio <= 1.0, "%s: max err/bound %.3f" % (what, ratio)
    assert mism <= MISMATCH_MAX, "%s: %.3f%% of the elements differ from round_bf16(reference)" % (what, 100 * mism)


def _check_sums(got_sum, got_sq, y, what):
    """Channel sums / sums of squares against the float64 sums of the stored output y."""
    yd = y.double().reshape(-1, y.shape[-1])
    s1, s2, a1 = yd.sum(0), (yd * yd).sum(0), yd.abs().sum(0)
    e1 = float(((got_sum.double() - s1).abs() / a1.clamp_min(1e-30)).max())
    e2 = float(((got_sq.double() - s2).abs() / s2.clamp_min(1e-30)).max())
    print("%-50s statistics rel err %.2e / %.2e" % (what, e1, e2))
    assert e1 <= STATS_REL and e2 <= STATS_REL, "%s: statistics rel err %.2e (sum) %.2e (sum of squares)" % (what, e1, e2)


def _twice(run, make_out):
    """Runs a launch into two fresh outputs; both must agree bit for bit."""
    torch, _, _ = _torch()
    a, b = make_out(), make_out()
    ra, rb = run(a), run(b)
    torch.cuda.synchronize()
    assert torch.equal(a.flat.view(torch.uint8), b.flat.view(torch.uint8)), "run-to-run difference in the output"
    return a, ra, rb


def _run_fwd(case):
    torch, F, raw = _torch()
    entry, (n, h, w, cin, cout, k, s), _res, _key = case
    seed = _seed(case)
    tag = _case_id(case)
    x = _input(n, h, w, cin, seed)
    wt = (_randn((cout, cin, k, k), seed + 1) * (cin * k * k) ** -0.5).to(torch.bfloat16).float().contiguous()
    w_f, _ = raw.pack_weight(wt, want_dgrad=False)
    xd, wd = _nchw(x), wt.double()
    r = F.conv2d(xd, wd, stride=s, padding=(k - 1) // 2).permute(0, 2, 3, 1)
    A = F.conv2d(xd.abs(), wd.abs(), stride=s, padding=(k - 1) // 2).permute(0, 2, 3, 1)
    ho, wo = r.shape[1:3]
    bias = (0.5 * _randn((cout,), seed + 2)).float()
    b64 = bias.double()
    if entry == "fwd_fp32":
        out, _, _ = _twice(lambda o: raw.conv2d_fwd(x, w_f, bias, stride=s, out=o.y, out_fp32=True),
                           lambda: Canvas(n, ho, wo, cout, torch.float32))
        out.check(tag)
        _check_values(out.y, r + b64, A, b64.abs(), tag + " fp32+bias", bf16=False)
        return
    add = _input(n, ho, wo, cout, seed + 3)
    add64 = add.double()
    scale = (1.0 + 0.25 * _randn((cout,), seed + 4)).float()
    shift = (0.25 * _randn((cout,), seed + 5)).float()
    sc, sh = scale.double(), shift.double()
    cpad = (cout + 15) // 16 * 16
    make = lambda: Canvas(n, ho, wo, cout, torch.bfloat16)      # noqa: E731

    def partials(st):
        buf, grid, cp = st
        return buf[: grid * 2 * cp].view(grid, 2, cp).double().sum(0)[:, :cout]

    # statistics partials, no bias
    out, (s_a, g_a, _), (s_b, g_b, _) = _twice(lambda o: raw.conv2d_fwd(x, w_f, None, s, out=o.y, emit_stats=True)[1],
                                                make)
    out.check(tag + " stats")
    assert g_a == g_b and torch.equal(s_a[: g_a * 2 * cpad], s_b[: g_b * 2 * cpad]), "run-to-run difference in the partials"
    _check_values(out.y, r, A, torch.zeros_like(r), tag + " stats")
    p = partials((s_a, g_a, cpad))
    _check_sums(p[0], p[1], out.y, tag + " partials")
    # bias + fp64 statistics cells (deferred BatchNorm finalisation)
    cells = []

    def run_cells(o):
        c = torch.zeros(2 * cpad, dtype=torch.float64, device="cuda")
        cells.append(c)
        raw.conv2d_fwd_cells(x, w_f, bias, s, c, out=o.y)
    out, _, _ = _twice(run_cells, make)
    out.check(tag + " bias+cells")
    _check_values(out.y, r + b64, A, b64.abs(), tag + " bias+cells")
    _check_sums(cells[0][:cout], cells[0][cpad:cpad + cout], out.y, tag + " cells")
    # bias + residual addend + partials
    out, (s_a, g_a, _), _ = _twice(
        lambda o: raw.conv2d_fwd(x, w_f, bias, s, out=o.y, emit_stats=True, addend=add)[1], make)
    out.check(tag + " bias+add")
    _check_values(out.y, r + b64 + add64, A, b64.abs() + add64.abs(), tag + " bias+add")
    p = partials((s_a, g_a, cpad))
    _check_sums(p[0], p[1], out.y, tag + " add partials")
    # evaluation: BatchNorm affine, then affine + addend + ReLU
    out, _, _ = _twice(lambda o: raw.conv2d_fwd_affine(x, w_f, scale, shift, False, s, out=o.y), make)
    out.check(tag + " affine")
    _check_values(out.y, r * sc + sh, A * sc.abs(), sh.abs(), tag + " affine")
    out, _, _ = _twice(lambda o: raw.conv2d_fwd_affine(x, w_f, scale, shift, True, s, addend=add, out=o.y), make)
    out.check(tag + " affine+add+relu")
    pre = r * sc + sh + add64
    _check_values(out.y, pre.clamp_min(0), A * sc.abs(), sh.abs() + add64.abs(), tag + " affine+add+relu", pre=pre)


def _run_dgrad(case):
    torch, _, raw = _torch()
    _entry, (n, h, w, cin, cout, k, s), _res, _key = case
    seed = _seed(case)
    tag = _case_id(case)
    cout8 = (cout + 7) // 8 * 8
    wt = (_randn((cout, cin, k, k), seed + 1) * (cin * k * k) ** -0.5).to(torch.bfloat16).float().contiguous()
    _, w_d = raw.pack_weight(wt)
    ho, wo = raw.out_hw(h, w, k, s)
    dy = _input(n, ho, wo, cout8, seed + 2, real=cout)
    dyd, wd = _nchw(dy[..., :cout]), wt.double()
    grad_in = torch.nn.grad.conv2d_input
    r = grad_in((n, cin, h, w), wd, dyd, stride=s, padding=(k - 1) // 2).permute(0, 2, 3, 1)
    A = grad_in((n, cin, h, w), wd.abs(), dyd.abs(), stride=s, padding=(k - 1) // 2).permute(0, 2, 3, 1)
    make = lambda: Canvas(n, h, w, cin, torch.bfloat16)      # noqa: E731
    out, _, _ = _twice(lambda o: raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), k, s, out=o.y), make)
    out.check(tag)
    _check_values(out.y, r, A, torch.zeros_like(r), tag)
    add = _input(n, h, w, cin, seed + 3)
    out, _, _ = _twice(lambda o: raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), k, s, addend=add, out=o.y), make)
    out.check(tag + " addend")
    _check_values(out.y, r + add.double(), A, add.double().abs(), tag + " addend")


def _run_wgrad(case):
    torch, _, raw = _torch()
    _entry, (n, h, w, cin, cout, k, s), _res, _key = case
    seed = _seed(case)
    tag = _case_id(case)
    x = _input(n, h, w, cin, seed)
    ho, wo = raw.out_hw(h, w, k, s)
    dy = _input(n, ho, wo, cout, seed + 2)       # the channels past cout hold NaN (read only into masked rows)
    xd, dyd = _nchw(x), _nchw(dy)
    grad_w = torch.nn.grad.conv2d_weight
    ohwi = lambda t: t.permute(0, 2, 3, 1).reshape(cout, k * k, cin)      # noqa: E731
    r = ohwi(grad_w(xd, (cout, cin, k, k), dyd, stride=s, padding=(k - 1) // 2))
    A = ohwi(grad_w(xd.abs(), (cout, cin, k, k), dyd.abs(), stride=s, padding=(k - 1) // 2))
    rnorm = float(r.norm())
    dw0 = (_randn((cout, k * k, cin), seed + 3) * rnorm / r.numel() ** 0.5).float()
    runs = []
    for _ in range(2):
        dw = dw0.clone()
        raw.conv2d_wgrad(x, dy, dw, cout, k, s)
        runs.append(dw)
    torch.cuda.synchronize()
    assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), "run-to-run difference in the gradient"
    dw = runs[0]
    inc = dw.double() - dw0.double()
    norm_err = float((inc - r).norm()) / rnorm
    err = (inc - r).abs()
    ratio = float((err / (WGRAD_ELEM * A + 2.0 ** -23 * dw.double().abs()).clamp_min(1e-300)).max())
    acc_rel = float(((err - 2.0 ** -24 * dw.double().abs()).clamp_min(0) / A.clamp_min(1e-300)).max())
    print("%-50s normwise err %.2e  max err/bound %.4f  accumulation err/A %.2e" % (tag, norm_err, ratio, acc_rel))
    assert norm_err <= WGRAD_NORM, "%s: normwise error %.2e" % (tag, norm_err)
    assert ratio <= 1.0, "%s: max err/bound %.3f" % (tag, ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + EXTRA_CASES, ids=_case_id)
def test_convolution_configuration_against_float64(case):
    torch, _, _ = _torch()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    entry, _shape, res, _key = case
    with smem_reserve(res):
        if case[3] is not None:
            assert config_key(entry, case[1]) == case[3], "the planner no longer picks this case's configuration"
        {"fwd": _run_fwd, "fwd_fp32": _run_fwd, "dgrad": _run_dgrad, "wgrad": _run_wgrad}[entry](case)
