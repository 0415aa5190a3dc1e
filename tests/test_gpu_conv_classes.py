"""Every tensor-core convolution configuration the traced programs launch, checked against float64.

A launch of conv_igemm_kernel, conv3x3_halo_kernel or wgrad_igemm_kernel runs one of several configurations the host
planners pick per shape: the Cout tile BN (which decides the wgmma widths of the n64 groups and the n16/n32/n48 tail),
the co-resident (OCC 2, <= 128 accumulator columns) or full-SM (OCC 1) build, the channel chunk KC of the per-tap kernel,
resident or streamed weights and the ring depth of the halo kernel, and for the weight gradient the N tile, the taps per
group and a direct or pixel-split decomposition. The key also names the tap geometry (1x1, 1x1 stride 2, 3x3, 3x3
stride 2, dilated 3x3), the pixel tile width of the per-tap kernel (8 when the output is at most 8 wide, else 16) and
the statistics window (layers too wide for every channel's statistics in one CTA keep only their own N tile's columns).
CASES holds, for every configuration key of the traced programs (the training step of every architecture with and
without deferred BatchNorm cells, the attention-head variants, the evaluation forwards at 0.5x, 1.0x and 2.0x;
forward, stride-1 data gradient and weight gradient, without and with the SyncBN shared-memory reserve), the smallest
shape found that reaches it under the default planner settings: at least 9 x 9 (edge tiles in both directions), and for
dilated layers large enough that every tap reads image pixels, unless the key asks for a narrow map.
tests/test_conv_plans.py checks on the CPU that every case still plans to its key and that the keys cover the programs.

Every case is compared with F.conv2d and its autograd in float64 on the GPU, computed from exactly the bf16 inputs, with
bounds tied to fp32 accumulation (A = the same convolution of |inputs|):
  * bf16 outputs: |y - r| <= ulp_bf16(r) + ACC_REL * A elementwise, and at most a share _mismatch_limit of the
    elements differ from round_bf16(r) (a systematic error of ~1e-4 relative flips many roundings without breaking the
    first bound): MISMATCH_MAX up to a reduction depth of MISMATCH_DEPTH terms, growing with the square root of the
    depth beyond it like the fp32 accumulation error;
  * fp32 outputs: |y - r| <= ACC_REL * A;
  * weight gradients: the increment of a random non-zero accumulator within WGRAD_NORM of r normwise (a dropped pixel
    tile shows up there) and within WGRAD_ELEM * A elementwise;
  * statistics (per-CTA partials and the fp64 cells): within STATS_REL of the float64 sums of the stored outputs; with
    the statistics window, every partials row is exactly zero outside its CTA's own N tile.
Outputs go into a slice of a NaN-filled wider buffer with a NaN guard behind it: every element outside the slice must
keep its NaN bits (edge-tile rows and column tails are masked), every element inside must be finite. Inputs carry NaN
in the channels past their extent, which the kernels must never read. Every launch runs twice and must give the same bits.
Forward cases run every epilogue: statistics partials, bias + fp64 cells, bias + addend + partials, BatchNorm affine,
and affine + addend + ReLU; data-gradient cases run with and without an addend (the 1x1 stride-2 data gradient writes
only the even lattice, into a prefilled dx that is its own addend: the odd lattice must keep its bits).
"""
import contextlib
import ctypes
import zlib

import pytest

from b200seg import _lib

SYNCBN_RESERVE = 12288      # shared memory per SM the planners leave free in SyncBN mode (b200seg/p2p.py)

# Largest values observed on one H100 80GB HBM3 (700 W power limit), over the cases of the W48 step (reductions of at
# most 720 x 9 = 6480 terms) and over the rows the WideResNet-38, ASPP, attention-head and evaluation programs added
# (dilated 3x3 up to 4096 x 9 = 36 864 terms, 1x1 up to 4096 terms, weight gradients up to 4233 pixels per work unit):
#                                                   W48 step cases              added rows (headroom)
#   accumulation error / A, bf16 and fp32 outputs   6.9e-7 (igemm)              1.25e-6, 4096 -> 256 dilation 12 (3.0x)
#                                                                                 -> ACC_REL 2^-18 = 3.8e-6
#   share of bf16 outputs != round_bf16(reference)  0.38 % (halo, Cin 720)      1.43 % at 36 864 terms (2.7x), 4 of the
#                                                                                 256 outputs of the 1x1 map (1.02x)
#                                                                                 -> MISMATCH_MAX 1.6 % (scaled)
#   weight gradient normwise / elementwise / A      1.2e-6 / 1.9e-7             4.2e-6 / 5.4e-7, 720 -> 256 3x3 over
#                                                                                 17 x 249 (1.2x / 1.8x)
#                                                                                 -> 5e-6 / 2^-20 = 9.5e-7
#   statistics relative to sum |y| (or sum y^2)     1.3e-7                      1.7e-7 (5.9x) -> STATS_REL 1e-6
# The share of honest rounding mismatches grows like the fp32 accumulation error, with the square root of the reduction
# depth (0.38 % at 6480 terms, 1.43 % at 36 864): past MISMATCH_DEPTH the limit scales by sqrt(depth / MISMATCH_DEPTH),
# so no case of the W48 step gets a looser limit. The 1x1-map row has 256 outputs: one mismatch is 0.39 %.
# Scaling the output columns >= 192 by 1 + 2^-9 (an error tests/test_gpu_ops.py passes) makes 9-23 % of the outputs of
# every wide case differ from round_bf16(reference).
ACC_REL = 2.0 ** -18
MISMATCH_MAX = 0.016
MISMATCH_DEPTH = 6480
WGRAD_NORM = 5e-6
WGRAD_ELEM = 2.0 ** -20
STATS_REL = 1e-6


def _mismatch_limit(depth):
    """Largest share of the bf16 outputs of a reduction over depth terms allowed to differ from round_bf16(reference)."""
    return MISMATCH_MAX * max(1.0, depth / MISMATCH_DEPTH) ** 0.5


# (entry point, (n, h, w, cin, cout, k, stride[, dilation]) of the forward convolution, smem reserve, configuration key)
#   fwd / dgrad key: (kernel, BN, CTAs per SM, KC (igemm) or 'res' / weight-ring slots (halo), more tiles than CTAs,
#                     taps, pixel tile width, statistics window)
#   wgrad key:       (N tile, width of the last N tile mod 64, taps per group, direct / split, dy blocks of the last M tile,
#                     taps)
# A data-gradient cout is the padded extent roundup8(cout) the step hands over. A forward case's key is that of its
# launches with statistics (case_keys).
CASES = [
    ('fwd', (1, 17, 793, 64, 128, 3, 1), 0, ('halo', 128, 1, 'res', True, '3x3', 8, 0)),
    ('fwd', (1, 17, 793, 128, 128, 3, 1), 0, ('halo', 128, 1, 8, True, '3x3', 8, 0)),
    ('fwd', (1, 17, 209, 384, 384, 3, 1), SYNCBN_RESERVE, ('halo', 192, 1, 5, False, '3x3', 8, 0)),
    ('fwd', (1, 17, 209, 384, 384, 3, 1), 0, ('halo', 192, 1, 6, False, '3x3', 8, 0)),
    ('fwd', (1, 17, 881, 192, 192, 3, 1), 0, ('halo', 192, 1, 6, True, '3x3', 8, 0)),
    ('fwd', (1, 17, 209, 512, 512, 3, 1), 0, ('halo', 256, 1, 4, False, '3x3', 8, 0)),
    ('fwd', (1, 17, 421, 720, 512, 3, 1), 0, ('halo', 256, 1, 4, True, '3x3', 8, 0)),
    ('fwd', (1, 49, 397, 256, 256, 3, 1), 0, ('halo', 256, 1, 5, True, '3x3', 8, 0)),
    ('fwd', (1, 9, 9, 192, 192, 3, 1), 0, ('halo', 32, 2, 8, False, '3x3', 8, 0)),
    ('fwd', (1, 33, 181, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', False, '3x3', 8, 0)),
    ('fwd', (1, 69, 421, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', True, '3x3', 8, 0)),
    ('fwd', (1, 17, 41, 384, 384, 3, 1), SYNCBN_RESERVE, ('halo', 48, 2, 5, False, '3x3', 8, 0)),
    ('fwd', (1, 17, 41, 384, 384, 3, 1), 0, ('halo', 48, 2, 6, False, '3x3', 8, 0)),
    ('fwd', (1, 33, 117, 96, 96, 3, 1), 0, ('halo', 48, 2, 8, False, '3x3', 8, 0)),
    ('fwd', (1, 69, 421, 256, 48, 3, 1), 0, ('halo', 48, 2, 8, True, '3x3', 8, 0)),
    ('fwd', (1, 33, 181, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, False, '3x3', 8, 0)),
    ('fwd', (1, 69, 421, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, True, '3x3', 8, 0)),
    ('fwd', (1, 33, 181, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, False, '3x3', 8, 0)),
    ('fwd', (1, 69, 421, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, True, '3x3', 8, 0)),
    ('fwd', (1, 33, 117, 192, 192, 3, 1), SYNCBN_RESERVE, ('halo', 96, 1, 8, False, '3x3', 8, 0)),
    ('fwd', (1, 33, 237, 96, 96, 3, 1), 0, ('halo', 96, 2, 4, False, '3x3', 8, 0)),
    ('fwd', (1, 33, 881, 96, 96, 3, 1), 0, ('halo', 96, 2, 4, True, '3x3', 8, 0)),
    ('fwd', (1, 177, 17, 1280, 256, 1, 1), 0, ('igemm', 128, 1, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 113, 33, 4096, 256, 3, 1, 12), 0, ('igemm', 128, 1, 64, False, '3x3d', 16, 0)),
    ('fwd', (1, 49, 229, 64, 256, 1, 1), 0, ('igemm', 128, 1, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 881, 33, 64, 128, 1, 1), 0, ('igemm', 128, 2, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 9, 17, 96, 96, 3, 2), 0, ('igemm', 16, 2, 32, False, '3x3s2', 16, 0)),
    ('fwd', (1, 9, 9, 96, 96, 3, 2), 0, ('igemm', 16, 2, 32, False, '3x3s2', 8, 0)),
    ('fwd', (1, 9, 9, 256, 1, 1, 1), 0, ('igemm', 16, 2, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 1, 1, 4096, 256, 1, 1), 0, ('igemm', 16, 2, 64, False, '1x1', 8, 0)),
    ('fwd', (1, 9, 17, 48, 48, 3, 2), 0, ('igemm', 16, 2, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 237, 133, 256, 1, 1, 1), 0, ('igemm', 16, 2, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 353, 33, 96, 384, 3, 2), 0, ('igemm', 192, 1, 32, False, '3x3s2', 16, 0)),
    ('fwd', (1, 1057, 33, 96, 192, 3, 2), 0, ('igemm', 192, 1, 32, True, '3x3s2', 16, 0)),
    ('fwd', (1, 353, 33, 48, 384, 3, 2), 0, ('igemm', 192, 1, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 1057, 65, 48, 192, 3, 2), 0, ('igemm', 192, 1, 64, True, '3x3s2', 16, 0)),
    ('fwd', (1, 181, 33, 720, 720, 1, 1), 0, ('igemm', 240, 1, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 177, 17, 1024, 512, 1, 1), 0, ('igemm', 256, 1, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 417, 33, 256, 512, 1, 2), 0, ('igemm', 256, 1, 64, False, '1x1s2', 16, 0)),
    ('fwd', (1, 177, 17, 512, 512, 3, 1, 2), 0, ('igemm', 256, 1, 64, False, '3x3d', 16, 0)),
    ('fwd', (1, 353, 33, 256, 512, 3, 2), 0, ('igemm', 256, 1, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 229, 245, 64, 256, 1, 1), 0, ('igemm', 256, 1, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 17, 41, 2048, 4096, 1, 1), 0, ('igemm', 256, 1, 64, True, '1x1', 16, 1)),
    ('fwd', (1, 785, 33, 256, 512, 1, 2), 0, ('igemm', 256, 1, 64, True, '1x1s2', 16, 0)),
    ('fwd', (1, 393, 17, 512, 512, 3, 1, 2), 0, ('igemm', 256, 1, 64, True, '3x3d', 16, 0)),
    ('fwd', (1, 113, 17, 1024, 2048, 3, 1, 4), SYNCBN_RESERVE, ('igemm', 256, 1, 64, True, '3x3d', 16, 1)),
    ('fwd', (1, 785, 33, 256, 512, 3, 2), 0, ('igemm', 256, 1, 64, True, '3x3s2', 16, 0)),
    ('fwd', (1, 177, 17, 96, 48, 1, 1), 0, ('igemm', 32, 2, 32, False, '1x1', 16, 0)),
    ('fwd', (1, 9, 17, 96, 384, 3, 2), 0, ('igemm', 32, 2, 32, False, '3x3s2', 16, 0)),
    ('fwd', (1, 9, 9, 96, 384, 3, 2), 0, ('igemm', 32, 2, 32, False, '3x3s2', 8, 0)),
    ('fwd', (1, 9, 9, 384, 192, 1, 1), 0, ('igemm', 32, 2, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 1, 1, 256, 256, 1, 1), 0, ('igemm', 32, 2, 64, False, '1x1', 8, 0)),
    ('fwd', (1, 9, 17, 48, 384, 3, 2), 0, ('igemm', 32, 2, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 9, 9, 48, 384, 3, 2), 0, ('igemm', 32, 2, 64, False, '3x3s2', 8, 0)),
    ('fwd', (1, 237, 133, 256, 19, 1, 1), 0, ('igemm', 32, 2, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 33, 213, 96, 48, 1, 1), 0, ('igemm', 48, 2, 32, False, '1x1', 16, 0)),
    ('fwd', (1, 81, 33, 96, 384, 3, 2), 0, ('igemm', 48, 2, 32, False, '3x3s2', 16, 0)),
    ('fwd', (1, 1057, 17, 96, 48, 1, 1), 0, ('igemm', 48, 2, 32, True, '1x1', 16, 0)),
    ('fwd', (1, 41, 117, 192, 96, 1, 1), 0, ('igemm', 48, 2, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 529, 33, 48, 48, 3, 2), 0, ('igemm', 48, 2, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 1057, 17, 128, 48, 1, 1), 0, ('igemm', 48, 2, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 1057, 97, 48, 48, 3, 2), 0, ('igemm', 48, 2, 64, True, '3x3s2', 16, 0)),
    ('fwd', (1, 837, 133, 16, 64, 3, 2), 0, ('igemm', 64, 2, 16, True, '3x3s2', 16, 0)),
    ('fwd', (1, 33, 213, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 529, 33, 64, 64, 3, 2), 0, ('igemm', 64, 2, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 237, 133, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, True, '1x1', 16, 0)),
    ('fwd', (1, 1057, 97, 64, 64, 3, 2), 0, ('igemm', 64, 2, 64, True, '3x3s2', 16, 0)),
    ('fwd', (1, 117, 165, 96, 192, 3, 2), 0, ('igemm', 96, 2, 32, False, '3x3s2', 16, 0)),
    ('fwd', (1, 265, 17, 192, 96, 1, 1), 0, ('igemm', 96, 2, 64, False, '1x1', 16, 0)),
    ('fwd', (1, 213, 133, 48, 96, 3, 2), 0, ('igemm', 96, 2, 64, False, '3x3s2', 16, 0)),
    ('fwd', (1, 1057, 97, 48, 96, 3, 2), 0, ('igemm', 96, 2, 64, True, '3x3s2', 16, 0)),
    ('dgrad', (1, 49, 197, 256, 48, 3, 1), 0, ('halo', 128, 1, 8, True, '3x3', 8, 0)),
    ('dgrad', (1, 17, 417, 304, 256, 3, 1), 0, ('halo', 160, 1, 7, True, '3x3', 8, 0)),
    ('dgrad', (1, 17, 317, 720, 512, 3, 1), 0, ('halo', 240, 1, 4, True, '3x3', 8, 0)),
    ('dgrad', (1, 17, 209, 512, 512, 3, 1), 0, ('halo', 256, 1, 4, False, '3x3', 8, 0)),
    ('dgrad', (1, 49, 213, 512, 256, 3, 1), 0, ('halo', 256, 1, 4, True, '3x3', 8, 0)),
    ('dgrad', (1, 85, 445, 256, 48, 3, 1), 0, ('halo', 256, 1, 5, True, '3x3', 8, 0)),
    ('dgrad', (1, 9, 9, 192, 192, 3, 1), 0, ('halo', 32, 2, 8, False, '3x3', 8, 0)),
    ('dgrad', (1, 33, 181, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', False, '3x3', 8, 0)),
    ('dgrad', (1, 69, 421, 48, 48, 3, 1), 0, ('halo', 48, 2, 'res', True, '3x3', 8, 0)),
    ('dgrad', (1, 17, 41, 384, 384, 3, 1), SYNCBN_RESERVE, ('halo', 48, 2, 5, False, '3x3', 8, 0)),
    ('dgrad', (1, 17, 41, 384, 384, 3, 1), 0, ('halo', 48, 2, 6, False, '3x3', 8, 0)),
    ('dgrad', (1, 33, 117, 96, 96, 3, 1), 0, ('halo', 48, 2, 8, False, '3x3', 8, 0)),
    ('dgrad', (1, 33, 181, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, False, '3x3', 8, 0)),
    ('dgrad', (1, 69, 421, 64, 64, 3, 1), SYNCBN_RESERVE, ('halo', 64, 2, 6, True, '3x3', 8, 0)),
    ('dgrad', (1, 33, 181, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, False, '3x3', 8, 0)),
    ('dgrad', (1, 69, 421, 64, 64, 3, 1), 0, ('halo', 64, 2, 7, True, '3x3', 8, 0)),
    ('dgrad', (1, 33, 117, 192, 192, 3, 1), SYNCBN_RESERVE, ('halo', 96, 1, 8, False, '3x3', 8, 0)),
    ('dgrad', (1, 33, 237, 96, 96, 3, 1), 0, ('halo', 96, 2, 4, False, '3x3', 8, 0)),
    ('dgrad', (1, 49, 229, 256, 8, 1, 1), 0, ('igemm', 128, 1, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 265, 17, 128, 256, 1, 1), 0, ('igemm', 128, 2, 64, False, '1x1', 16, 0)),
    ('dgrad', (1, 881, 33, 128, 48, 1, 1), 0, ('igemm', 128, 2, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 145, 17, 1280, 256, 1, 1), 0, ('igemm', 224, 1, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 41, 437, 720, 24, 1, 1), 0, ('igemm', 240, 1, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 177, 33, 720, 256, 3, 1, 12), 0, ('igemm', 240, 1, 64, True, '3x3d', 16, 0)),
    ('dgrad', (1, 9, 17, 4096, 256, 1, 1), 0, ('igemm', 256, 1, 64, False, '1x1', 16, 0)),
    ('dgrad', (1, 1, 1, 4096, 256, 1, 1), 0, ('igemm', 256, 1, 64, False, '1x1', 8, 0)),
    ('dgrad', (1, 177, 17, 512, 512, 3, 1, 2), 0, ('igemm', 256, 1, 64, False, '3x3d', 16, 0)),
    ('dgrad', (1, 57, 453, 512, 24, 1, 1), 0, ('igemm', 256, 1, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 33, 33, 4096, 256, 3, 1, 12), 0, ('igemm', 256, 1, 64, True, '3x3d', 16, 0)),
    ('dgrad', (1, 9, 9, 192, 96, 1, 1), 0, ('igemm', 32, 2, 32, False, '1x1', 16, 0)),
    ('dgrad', (1, 9, 9, 192, 48, 1, 1), 0, ('igemm', 32, 2, 64, False, '1x1', 16, 0)),
    ('dgrad', (1, 1, 1, 256, 256, 1, 1), 0, ('igemm', 32, 2, 64, False, '1x1', 8, 0)),
    ('dgrad', (1, 1, 1, 720, 256, 1, 1), SYNCBN_RESERVE, ('igemm', 48, 1, 64, False, '1x1', 8, 0)),
    ('dgrad', (1, 9, 9, 384, 96, 1, 1), 0, ('igemm', 48, 2, 32, False, '1x1', 16, 0)),
    ('dgrad', (1, 9, 9, 384, 48, 1, 1), 0, ('igemm', 48, 2, 64, False, '1x1', 16, 0)),
    ('dgrad', (1, 1, 1, 512, 256, 1, 1), 0, ('igemm', 48, 2, 64, False, '1x1', 8, 0)),
    ('dgrad', (1, 33, 213, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, False, '1x1', 16, 0)),
    ('dgrad', (1, 237, 133, 64, 64, 1, 1), 0, ('igemm', 64, 2, 64, True, '1x1', 16, 0)),
    ('dgrad', (1, 41, 117, 192, 96, 1, 1), 0, ('igemm', 96, 2, 32, False, '1x1', 16, 0)),
    ('dgrad', (1, 41, 117, 192, 48, 1, 1), 0, ('igemm', 96, 2, 64, False, '1x1', 16, 0)),
    ('wgrad', (1, 9, 9, 1024, 2048, 1, 1), 0, ('wgrad', 128, 0, 1, 'direct', 2, '1x1')),
    ('wgrad', (1, 49, 229, 256, 1, 1, 1), 0, ('wgrad', 128, 0, 1, 'split', 1, '1x1')),
    ('wgrad', (1, 129, 17, 128, 256, 1, 1), 0, ('wgrad', 128, 0, 1, 'split', 2, '1x1')),
    ('wgrad', (1, 705, 33, 256, 512, 1, 2), 0, ('wgrad', 128, 0, 1, 'split', 2, '1x1s2')),
    ('wgrad', (1, 69, 133, 256, 96, 3, 2), 0, ('wgrad', 128, 0, 1, 'split', 2, '3x3s2')),
    ('wgrad', (1, 17, 17, 1024, 2048, 3, 1, 4), 0, ('wgrad', 128, 0, 2, 'direct', 2, '3x3d')),
    ('wgrad', (1, 241, 17, 720, 256, 1, 1), 0, ('wgrad', 128, 16, 1, 'split', 2, '1x1')),
    ('wgrad', (1, 9, 9, 720, 512, 3, 1), 0, ('wgrad', 128, 16, 2, 'direct', 2, '3x3')),
    ('wgrad', (1, 33, 197, 96, 192, 3, 2), 0, ('wgrad', 128, 32, 1, 'split', 1, '3x3s2')),
    ('wgrad', (1, 41, 85, 96, 96, 3, 1), 0, ('wgrad', 128, 32, 1, 'split', 2, '3x3')),
    ('wgrad', (1, 273, 33, 96, 96, 3, 2), 0, ('wgrad', 128, 32, 1, 'split', 2, '3x3s2')),
    ('wgrad', (1, 125, 245, 96, 96, 3, 1), 0, ('wgrad', 128, 32, 2, 'split', 2, '3x3')),
    ('wgrad', (1, 9, 9, 2048, 4096, 1, 1), 0, ('wgrad', 256, 0, 1, 'direct', 2, '1x1')),
    ('wgrad', (1, 221, 197, 512, 19, 1, 1), 0, ('wgrad', 256, 0, 1, 'split', 1, '1x1')),
    ('wgrad', (1, 833, 17, 256, 48, 3, 1), 0, ('wgrad', 256, 0, 1, 'split', 1, '3x3')),
    ('wgrad', (1, 457, 17, 1280, 256, 1, 1), 0, ('wgrad', 256, 0, 1, 'split', 2, '1x1')),
    ('wgrad', (1, 17, 165, 512, 256, 3, 1), 0, ('wgrad', 256, 0, 1, 'split', 2, '3x3')),
    ('wgrad', (1, 513, 17, 256, 512, 3, 2), 0, ('wgrad', 256, 0, 1, 'split', 2, '3x3s2')),
    ('wgrad', (1, 57, 485, 720, 19, 1, 1), 0, ('wgrad', 256, 16, 1, 'split', 1, '1x1')),
    ('wgrad', (1, 221, 17, 720, 720, 1, 1), 0, ('wgrad', 256, 16, 1, 'split', 2, '1x1')),
    ('wgrad', (1, 249, 17, 720, 256, 3, 1), 0, ('wgrad', 256, 16, 1, 'split', 2, '3x3')),
    ('wgrad', (1, 169, 33, 720, 256, 3, 1, 12), 0, ('wgrad', 256, 16, 1, 'split', 2, '3x3d')),
    ('wgrad', (1, 9, 9, 384, 48, 1, 1), 0, ('wgrad', 64, 0, 1, 'direct', 1, '1x1')),
    ('wgrad', (1, 9, 9, 192, 192, 3, 1), 0, ('wgrad', 64, 0, 1, 'direct', 1, '3x3')),
    ('wgrad', (1, 9, 9, 384, 96, 1, 1), 0, ('wgrad', 64, 0, 1, 'direct', 2, '1x1')),
    ('wgrad', (1, 9, 9, 192, 384, 3, 2), 0, ('wgrad', 64, 0, 1, 'direct', 2, '3x3s2')),
    ('wgrad', (1, 49, 17, 64, 64, 1, 1), 0, ('wgrad', 64, 0, 1, 'split', 1, '1x1')),
    ('wgrad', (1, 33, 17, 64, 256, 1, 1), 0, ('wgrad', 64, 0, 1, 'split', 2, '1x1')),
    ('wgrad', (1, 97, 33, 256, 512, 1, 2), 0, ('wgrad', 64, 0, 1, 'split', 2, '1x1s2')),
    ('wgrad', (1, 9, 9, 384, 384, 3, 1), 0, ('wgrad', 64, 0, 2, 'direct', 2, '3x3')),
    ('wgrad', (1, 897, 17, 64, 64, 3, 1), 0, ('wgrad', 64, 0, 2, 'split', 1, '3x3')),
    ('wgrad', (1, 229, 453, 64, 64, 3, 2), 0, ('wgrad', 64, 0, 2, 'split', 1, '3x3s2')),
    ('wgrad', (1, 9, 9, 512, 512, 3, 1), 0, ('wgrad', 64, 0, 3, 'direct', 2, '3x3')),
    ('wgrad', (1, 9, 9, 512, 512, 3, 1, 2), 0, ('wgrad', 64, 0, 3, 'direct', 2, '3x3d')),
    ('wgrad', (1, 25, 245, 256, 48, 3, 1), 0, ('wgrad', 64, 0, 3, 'split', 1, '3x3')),
    ('wgrad', (1, 1041, 97, 64, 64, 3, 2), 0, ('wgrad', 64, 0, 3, 'split', 1, '3x3s2')),
    ('wgrad', (1, 1041, 17, 64, 128, 3, 1), 0, ('wgrad', 64, 0, 3, 'split', 2, '3x3')),
    ('wgrad', (1, 165, 229, 256, 96, 3, 2), 0, ('wgrad', 64, 0, 3, 'split', 2, '3x3s2')),
    ('wgrad', (1, 9, 9, 720, 256, 1, 1), 0, ('wgrad', 64, 16, 1, 'direct', 2, '1x1')),
    ('wgrad', (1, 985, 65, 16, 64, 3, 1), 0, ('wgrad', 64, 16, 9, 'split', 1, '3x3')),
    ('wgrad', (1, 981, 293, 16, 64, 3, 2), 0, ('wgrad', 64, 16, 9, 'split', 1, '3x3s2')),
    ('wgrad', (1, 9, 9, 96, 192, 3, 2), 0, ('wgrad', 64, 32, 1, 'direct', 1, '3x3s2')),
    ('wgrad', (1, 9, 9, 96, 384, 3, 2), 0, ('wgrad', 64, 32, 1, 'direct', 2, '3x3s2')),
    ('wgrad', (1, 49, 17, 96, 48, 1, 1), 0, ('wgrad', 64, 32, 1, 'split', 1, '1x1')),
    ('wgrad', (1, 49, 101, 96, 96, 3, 2), 0, ('wgrad', 64, 32, 1, 'split', 2, '3x3s2')),
    ('wgrad', (1, 9, 9, 48, 384, 3, 2), 0, ('wgrad', 64, 48, 1, 'direct', 2, '3x3s2')),
    ('wgrad', (1, 117, 33, 48, 48, 3, 2), 0, ('wgrad', 64, 48, 1, 'split', 1, '3x3s2')),
    ('wgrad', (1, 17, 165, 48, 96, 3, 2), 0, ('wgrad', 64, 48, 1, 'split', 2, '3x3s2')),
    ('wgrad', (1, 117, 229, 48, 192, 3, 2), 0, ('wgrad', 64, 48, 2, 'split', 1, '3x3s2')),
    ('wgrad', (1, 41, 341, 48, 48, 3, 1), 0, ('wgrad', 64, 48, 3, 'split', 1, '3x3')),
    ('wgrad', (1, 1041, 33, 48, 48, 3, 2), 0, ('wgrad', 64, 48, 3, 'split', 1, '3x3s2')),
    ('wgrad', (1, 129, 17, 304, 256, 3, 1), 0, ('wgrad', 64, 48, 3, 'split', 2, '3x3')),
    ('wgrad', (1, 181, 325, 48, 96, 3, 2), 0, ('wgrad', 64, 48, 3, 'split', 2, '3x3s2')),
]

# Launches no plan query reports: 3x3 stride-2 data gradients run as four sub-lattice launches of conv_igemm_kernel (odd
# extents give sub-lattices of different sizes), the 1x1 stride-2 data gradient (WideResNet-38's 256 -> 512 projection)
# as one launch over the even lattice, and the fp32 logit head (512 -> 19, bias, out_ld 20 in the step). Also the
# statistics window with fewer tiles than CTAs (2048 -> 4096: every CTA one tile), which no traced program plans.
EXTRA_CASES = [
    ("dgrad", (1, 69, 133, 48, 96, 3, 2), 0, None),
    ("dgrad", (1, 101, 205, 64, 64, 3, 2), 0, None),
    ("dgrad", (1, 37, 67, 256, 96, 3, 2), 0, None),
    ("dgrad", (1, 37, 67, 256, 512, 1, 2), 0, None),
    ("fwd_fp32", (1, 33, 69, 512, 19, 1, 1), 0, None),
    ("fwd", (1, 9, 17, 2048, 4096, 1, 1), 0, None),
]


def _shape8(shape):
    """(n, h, w, cin, cout, k, stride, dilation): a table shape without a dilation is dense."""
    return tuple(shape) + (1,) * (8 - len(shape))


def _desc(shape, emit_stats=0, out_fp32=0, has_bias=0):
    n, h, w, cin, cout, k, s, dil = _shape8(shape)
    d = _lib.ConvDesc()
    d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride = n, h, w, cin, cout, k, s
    d.pad, d.dilation = (dil if k == 3 else 0), dil
    d.x_ld, d.y_ld = cin, (cout + 7) // 8 * 8
    d.emit_stats, d.out_fp32, d.has_bias = emit_stats, out_fp32, has_bias
    return d


def _taps(shape):
    _n, _h, _w, _cin, _cout, k, s, dil = _shape8(shape)
    return "3x3d" if dil > 1 else "%dx%d%s" % (k, k, "s2" if s == 2 else "")


def config_key(entry, shape, emit_stats=0, out_fp32=0, has_bias=0):
    """Configuration key of a launch with this descriptor under the current shared-memory reserve, from the host-only
    plan queries."""
    L = _lib.lib()
    d = _desc(shape, emit_stats, out_fp32, has_bias)
    _n, _h, w, cin, cout, _k, s, _dil = _shape8(shape)
    if entry == "wgrad":
        out = (ctypes.c_int32 * 10)()
        assert L.b200seg_conv2d_wgrad_plan_info(ctypes.byref(d), out) == 0, shape
        ntile, n_tiles, tpg, _groups, splits, m_tiles = list(out)[:6]
        return ("wgrad", ntile, (cin - (n_tiles - 1) * ntile) % 64, tpg, "direct" if splits == 1 else "split",
                2 if cout - (m_tiles - 1) * 128 > 64 else 1, _taps(shape))
    out = (ctypes.c_int32 * 13)()
    assert L.b200seg_conv2d_plan_info(ctypes.byref(d), (0 if entry == "fwd" else 1) | _lib.PLAN_WINDOW, out) == 0, \
        (entry, shape)
    kern, bn, _nt, grid, _smem, _depth, occ, _acc, resident, b_slots, kc, tiles, window = list(out)
    wo = (w - 1) // s + 1          # output width (a data gradient's output is the forward input, stride 1)
    return ("halo" if kern else "igemm", bn, occ, ("res" if resident else b_slots) if kern else kc, tiles > grid,
            _taps(shape), 8 if kern or wo <= 8 else 16, window)


def case_keys(entry, shape):
    """(declared key, every key the case runs). A forward case's declared key is that of its statistics launches; its
    affine launches run without statistics, which for the widest layers is a plan without the statistics window."""
    if entry != "fwd":
        key = config_key(entry, shape)
        return key, {key}
    key = config_key(entry, shape, emit_stats=1)
    return key, {key, config_key(entry, shape, emit_stats=0)}


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
    entry, shape, res, _key = case
    n, h, w, cin, cout, k, s, dil = _shape8(shape)
    return "%s-%dx%dx%d-c%d-%d-k%ds%d%s%s" % (entry, n, h, w, cin, cout, k, s, "d%d" % dil if dil > 1 else "",
                                             "-syncbn" if res else "")


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


def _check_values(y, ref, A, other, what, bf16=True, pre=None, depth=1):
    """y (bf16 or fp32) against the float64 reference ref; A bounds the accumulation error, other (|bias| + |shift| +
    |addend|) the fp32 epilogue arithmetic; pre = the reference before a ReLU (its ulp is the larger); depth = terms per
    output of the reduction. Also prints the accumulation error alone: what is left of |y - r| after the rounding to
    bf16 (ulp(y) / 2), over A."""
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
    limit = _mismatch_limit(depth)
    print("%-50s max err/bound %.4f  accumulation err/A %.2e  rounding mismatches %.4f%% (limit %.2f%%)" %
          (what, ratio, acc_rel, 100 * mism, 100 * limit))
    assert ratio <= 1.0, "%s: max err/bound %.3f" % (what, ratio)
    assert mism <= limit, "%s: %.3f%% of the elements differ from round_bf16(reference)" % (what, 100 * mism)


def _check_sums(got_sum, got_sq, y, what):
    """Channel sums / sums of squares against the float64 sums of the stored output y."""
    yd = y.double().reshape(-1, y.shape[-1])
    s1, s2, a1 = yd.sum(0), (yd * yd).sum(0), yd.abs().sum(0)
    e1 = float(((got_sum.double() - s1).abs() / a1.clamp_min(1e-30)).max())
    e2 = float(((got_sq.double() - s2).abs() / s2.clamp_min(1e-30)).max())
    print("%-50s statistics rel err %.2e / %.2e" % (what, e1, e2))
    assert e1 <= STATS_REL and e2 <= STATS_REL, "%s: statistics rel err %.2e (sum) %.2e (sum of squares)" % (what, e1, e2)


def _check_window(st, plan, what):
    """Windowed statistics: CTA b keeps only N tile b % n_tiles, so every partials row is exactly zero outside those BN
    columns, and the grid is the planned one (a multiple of n_tiles)."""
    torch, _, _ = _torch()
    buf, grid, cpad = st
    bn, n_tiles, planned = plan[1], plan[2], plan[3]
    assert grid == planned and grid % n_tiles == 0, "%s: grid %d, planned %d, %d N tiles" % (what, grid, planned, n_tiles)
    rows = buf[: grid * 2 * cpad].view(grid, 2, cpad)
    own = torch.arange(grid, device="cuda") % n_tiles
    foreign = (torch.arange(cpad, device="cuda") // bn)[None, :] != own[:, None]
    bad = int((rows.view(torch.int32) != 0).logical_and(foreign[:, None, :]).sum())
    assert bad == 0, "%s: %d partials outside their CTA's N tile are not zero" % (what, bad)


def _plan(entry, shape, emit_stats):
    L = _lib.lib()
    out = (ctypes.c_int32 * 13)()
    assert L.b200seg_conv2d_plan_info(ctypes.byref(_desc(shape, emit_stats)), (0 if entry == "fwd" else 1) |
                                      _lib.PLAN_WINDOW, out) == 0
    return list(out)


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
    entry, shape, _res, _key = case
    n, h, w, cin, cout, k, s, dil = _shape8(shape)
    pad = dil if k == 3 else 0
    depth = cin * k * k           # terms per output
    seed = _seed(case)
    tag = _case_id(case)
    x = _input(n, h, w, cin, seed)
    wt = (_randn((cout, cin, k, k), seed + 1) * (cin * k * k) ** -0.5).to(torch.bfloat16).float().contiguous()
    w_f, _ = raw.pack_weight(wt, want_dgrad=False)
    xd, wd = _nchw(x), wt.double()
    r = F.conv2d(xd, wd, stride=s, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    A = F.conv2d(xd.abs(), wd.abs(), stride=s, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    ho, wo = r.shape[1:3]
    bias = (0.5 * _randn((cout,), seed + 2)).float()
    b64 = bias.double()
    if entry == "fwd_fp32":
        out, _, _ = _twice(lambda o: raw.conv2d_fwd(x, w_f, bias, stride=s, out=o.y, out_fp32=True, dilation=dil),
                           lambda: Canvas(n, ho, wo, cout, torch.float32))
        out.check(tag)
        _check_values(out.y, r + b64, A, b64.abs(), tag + " fp32+bias", bf16=False, depth=depth)
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

    plan = _plan("fwd", shape, emit_stats=1)
    # statistics partials, no bias
    out, (s_a, g_a, _), (s_b, g_b, _) = _twice(
        lambda o: raw.conv2d_fwd(x, w_f, None, s, out=o.y, emit_stats=True, dilation=dil)[1], make)
    out.check(tag + " stats")
    assert g_a == g_b and torch.equal(s_a[: g_a * 2 * cpad], s_b[: g_b * 2 * cpad]), "run-to-run difference in the partials"
    _check_values(out.y, r, A, torch.zeros_like(r), tag + " stats", depth=depth)
    if plan[12]:
        _check_window((s_a, g_a, cpad), plan, tag + " stats")
    p = partials((s_a, g_a, cpad))
    _check_sums(p[0], p[1], out.y, tag + " partials")
    # bias + fp64 statistics cells (deferred BatchNorm finalisation)
    cells = []

    def run_cells(o):
        c = torch.zeros(2 * cpad, dtype=torch.float64, device="cuda")
        cells.append(c)
        raw.conv2d_fwd_cells(x, w_f, bias, s, c, out=o.y, dilation=dil)
    out, _, _ = _twice(run_cells, make)
    out.check(tag + " bias+cells")
    _check_values(out.y, r + b64, A, b64.abs(), tag + " bias+cells", depth=depth)
    _check_sums(cells[0][:cout], cells[0][cpad:cpad + cout], out.y, tag + " cells")
    # bias + residual addend + partials
    out, (s_a, g_a, _), _ = _twice(
        lambda o: raw.conv2d_fwd(x, w_f, bias, s, out=o.y, emit_stats=True, addend=add, dilation=dil)[1], make)
    out.check(tag + " bias+add")
    _check_values(out.y, r + b64 + add64, A, b64.abs() + add64.abs(), tag + " bias+add", depth=depth)
    if plan[12]:
        _check_window((s_a, g_a, cpad), plan, tag + " bias+add")
    p = partials((s_a, g_a, cpad))
    _check_sums(p[0], p[1], out.y, tag + " add partials")
    # evaluation: BatchNorm affine, then affine + addend + ReLU
    out, _, _ = _twice(lambda o: raw.conv2d_fwd_affine(x, w_f, scale, shift, False, s, out=o.y, dilation=dil), make)
    out.check(tag + " affine")
    _check_values(out.y, r * sc + sh, A * sc.abs(), sh.abs(), tag + " affine", depth=depth)
    out, _, _ = _twice(lambda o: raw.conv2d_fwd_affine(x, w_f, scale, shift, True, s, addend=add, out=o.y,
                                                       dilation=dil), make)
    out.check(tag + " affine+add+relu")
    pre = r * sc + sh + add64
    _check_values(out.y, pre.clamp_min(0), A * sc.abs(), sh.abs() + add64.abs(), tag + " affine+add+relu", pre=pre,
                  depth=depth)


def _run_dgrad(case):
    torch, _, raw = _torch()
    _entry, shape, _res, _key = case
    n, h, w, cin, cout, k, s, dil = _shape8(shape)
    pad = dil if k == 3 else 0
    depth = cout * k * k          # terms per output (at most: a stride-2 sub-lattice takes fewer taps)
    seed = _seed(case)
    tag = _case_id(case)
    cout8 = (cout + 7) // 8 * 8
    wt = (_randn((cout, cin, k, k), seed + 1) * (cin * k * k) ** -0.5).to(torch.bfloat16).float().contiguous()
    _, w_d = raw.pack_weight(wt)
    ho, wo = raw.out_hw(h, w, k, s, dil)
    dy = _input(n, ho, wo, cout8, seed + 2, real=cout)
    dyd, wd = _nchw(dy[..., :cout]), wt.double()
    grad_in = torch.nn.grad.conv2d_input
    r = grad_in((n, cin, h, w), wd, dyd, stride=s, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    A = grad_in((n, cin, h, w), wd.abs(), dyd.abs(), stride=s, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    if k == 1 and s == 2:
        # only the even lattice receives a gradient: dx is accumulated in place (addend == dx) or zero-filled
        even = torch.zeros((h, w), dtype=torch.bool, device="cuda")
        even[::2, ::2] = True
        for name, fill in (("zero-filled", torch.zeros((n, h, w, cin), dtype=torch.bfloat16, device="cuda")),
                           ("in place", _input(n, h, w, cin, seed + 3).contiguous())):
            def run(o):
                o.y.copy_(fill)
                raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), k, s, addend=o.y if name == "in place" else None, out=o.y)
            out, _, _ = _twice(run, lambda: Canvas(n, h, w, cin, torch.bfloat16))
            out.check(tag + " " + name)
            keep = int((out.y.view(torch.int16) != fill.view(torch.int16))[:, ~even].sum())
            assert keep == 0, "%s %s: %d odd-lattice elements changed" % (tag, name, keep)
            f64 = fill.double()
            _check_values(out.y[:, even], (r + f64)[:, even], A[:, even], f64.abs()[:, even], tag + " " + name,
                          depth=depth)
        return
    make = lambda: Canvas(n, h, w, cin, torch.bfloat16)      # noqa: E731
    out, _, _ = _twice(lambda o: raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), k, s, out=o.y, dilation=dil), make)
    out.check(tag)
    _check_values(out.y, r, A, torch.zeros_like(r), tag, depth=depth)
    add = _input(n, h, w, cin, seed + 3)
    out, _, _ = _twice(lambda o: raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), k, s, addend=add, out=o.y, dilation=dil),
                       make)
    out.check(tag + " addend")
    _check_values(out.y, r + add.double(), A, add.double().abs(), tag + " addend", depth=depth)


def _run_wgrad(case):
    torch, _, raw = _torch()
    _entry, shape, _res, _key = case
    n, h, w, cin, cout, k, s, dil = _shape8(shape)
    pad = dil if k == 3 else 0
    seed = _seed(case)
    tag = _case_id(case)
    x = _input(n, h, w, cin, seed)
    ho, wo = raw.out_hw(h, w, k, s, dil)
    dy = _input(n, ho, wo, cout, seed + 2)       # the channels past cout hold NaN (read only into masked rows)
    xd, dyd = _nchw(x), _nchw(dy)
    grad_w = torch.nn.grad.conv2d_weight
    ohwi = lambda t: t.permute(0, 2, 3, 1).reshape(cout, k * k, cin)      # noqa: E731
    r = ohwi(grad_w(xd, (cout, cin, k, k), dyd, stride=s, padding=pad, dilation=dil))
    A = ohwi(grad_w(xd.abs(), (cout, cin, k, k), dyd.abs(), stride=s, padding=pad, dilation=dil))
    rnorm = float(r.norm())
    dw0 = (_randn((cout, k * k, cin), seed + 3) * rnorm / r.numel() ** 0.5).float()
    runs = []
    for _ in range(2):
        dw = dw0.clone()
        raw.conv2d_wgrad(x, dy, dw, cout, k, s, dilation=dil)
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
            assert case_keys(entry, case[1])[0] == case[3], "the planner no longer picks this case's configuration"
        {"fwd": _run_fwd, "fwd_fp32": _run_fwd, "dgrad": _run_dgrad, "wgrad": _run_wgrad}[entry](case)
