"""Every configuration of the launches that are not tensor-core convolutions (BatchNorm, resampling, pooling, softmax,
sums, layout helpers and the evaluation assembly) that the traced programs make, checked against float64.

ROWS holds, per configuration key of tools/ew_classes.py that the traced programs reach (the training step of every
architecture with and without deferred BatchNorm cells, the attention-head variants, the evaluation with its output
assembly and scoring tail), the smallest shape found that reaches it: a launch of one C ABI entry point with its
arguments in ABI order, PTR marking the operands that are present; an optional third element is the |mean| / std ratio
of the BatchNorm input. tests/test_ew_plans.py checks on the CPU that the rows cover every key of the programs. Edge
rows no traced program reaches follow: npix 1, 2 and 19, |mean| / std of 0, 16 and 64 (the E[y^2] - mean^2
cancellation), non-integer resampling ratios, broadcast_pixels at 2^-13, a spatial softmax of less than one block.

Every row is compared with a float64 reference computed from exactly the bf16 / fp32 inputs the kernel saw
(A = the same operation on |inputs|):
  * BatchNorm forward: mean and biased variance folded in float64 from the fp64 cells or the fp32 partials the kernel
    read, unbiased variance for the running and batch statistics;
  * BatchNorm backward: gamma * invstd * (g - mean g - xhat * mean(g * xhat)), g = dz with post_scale, dropout and the
    ReLU mask applied first;
  * resampling (fuse_fwd, image_prep, resize_to_nchw, resize_nchw) and its adjoint: the float64 interpolation matrix
    built with PyTorch's align_corners=False source-index rule (fp32 scale in / out) and its border clamp, or its
    transpose;
  * softmaxes, pooling (float64 max_pool2d and its autograd), sums, blends and the scoring tail directly in float64.
Bounds:
  * bf16 outputs: |out - r| <= ulp_bf16(r) + EW_REL * A elementwise (STAT_REL * A for spatial_sum's long sums), and at
    most MISMATCH_MAX of them differ from round_bf16(r); fp32 outputs: |out - r| <= EW_REL * A;
  * outputs that are one rounding of an exact value are compared bit for bit: masked_accum without accumulate,
    broadcast_pixels at scale 1, maxpool forward, transpose_pad, cast_rows without accumulate, accum_pred, and
    argmax_hist's class map and histogram;
  * per-channel statistics (mean, invstd, scale, shift, running and batch statistics): within PAR_REL, the fp32
    rounding of fp64 arithmetic, at every |mean| / std; sums (dgamma, dbeta, the backward and channel partial sums,
    bias_grad): within STAT_REL of the sum of magnitudes; num_batches_tracked exactly.
Outputs go into a slice of a NaN-filled wider buffer with a NaN guard behind it: nothing outside the slice may change and
everything inside must be finite. Inputs with ld > C hold NaN in the columns past C. Every launch runs twice and must
give the same bits.

Largest values observed on one H100 80GB HBM3 (700 W power limit) over the 177 rows (headroom = bound / observed):
  |out - r| / (ulp_bf16(r) + EW_REL * A), every bf16 output   0.4998 (2x: the bf16 rounding itself)
  fp32 arithmetic error / A (EW_REL 2^-18 = 3.8e-6)          softmaxes 8.5e-7 (4.5x), argmax_hist max probability
                                                              4.2e-7 (9x), resizes 2.5e-7 (15x), blend 1.7e-7, BatchNorm
                                                              dy 1.6e-7, bn_apply 9.8e-8, fuse_fwd 8.9e-8 (43x and more)
  share of bf16 outputs != round_bf16(r)                      0.21 % (bn_apply at |mean| / std 64, 4.8x; rows of fewer
                                                              than 1024 outputs not counted)
  sums / sum of magnitudes (STAT_REL 1e-5)                    1.8e-6 (backward, 5.6x), 5.2e-8 (channel_stats)
  statistics and parameters (PAR_REL 2^-21 = 4.8e-7)          1.5e-7 (3.2x), the same at |mean| / std 0, 16 and 64
Substituted errors that fail rows: bn_bwd_reduce_kernel dropping the last of 264 blocks (34 rows, every capped
reduction); masked_accum addressing its source with pitch C instead of src_ld (the 720-wide row); upsample_adjoint's
lane butterfly stopping one step early (16 of 17 adjoint rows, all but ratio 1). Removing upsample_adjoint_kernel's
+-1 window margin changes no output: the margin only guards the fp32 window bounds, and the fine pixels it adds carry
zero weight.
"""
import ctypes
import zlib

import pytest

from b200seg import _lib

PTR = "ptr"
EW_REL = 2.0 ** -18
MISMATCH_MAX = 0.01
MISMATCH_FEW = 16         # ... plus 16 outputs: the one- and two-pixel rows, where y - mean cancels in fp32
STAT_REL = 1e-5
PAR_REL = 2.0 ** -21

ROWS = [
    ('bn_apply', ('ptr', 256, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 256, 1, 1, 256, None, 0, 0)),
    ('bn_apply', ('ptr', 720, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 720, 33014, 33014, 720, None, 0, 0)),
    ('bn_apply', ('ptr', 64, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 64, 38, 38, 64, None, 0, 0)),
    ('bn_apply', ('ptr', 256, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 256, 131102, 131102, 256, 'ptr', 1, 0)),
    ('bn_apply', ('ptr', 256, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 256, 19, 19, 256, 'ptr', 0, 0)),
    ('bn_apply', ('ptr', 512, 'ptr', 'ptr', None, 0, 'ptr', 1, 'ptr', 512, 66104, 33052, 512, None, 0, 0)),
    ('bn_apply', ('ptr', 512, 'ptr', 'ptr', None, 0, 'ptr', 1, 'ptr', 512, 19, 19, 512, None, 0, 0)),
    ('bn_apply', ('ptr', 512, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 1024, 66104, 66104, 512, None, 0, 0)),
    ('bn_apply', ('ptr', 512, 'ptr', 'ptr', None, 0, None, 1, 'ptr', 1024, 19, 19, 512, None, 0, 0)),
    ('bn_apply', ('ptr', 256, 'ptr', 'ptr', 'ptr', 256, None, 1, 'ptr', 256, 131102, 131102, 256, None, 0, 0)),
    ('bn_apply', ('ptr', 256, 'ptr', 'ptr', 'ptr', 256, None, 1, 'ptr', 256, 19, 19, 256, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 256, ('fold', 256, 1.0, True, True, False), None, 0, None, 1, 'ptr', 256, 1, 1, 256, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 720, ('fold', 720, 33014.0, True, True, False), None, 0, None, 1, 'ptr', 720, 33014, 33014, 720, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 64, ('fold', 64, 38.0, True, True, False), None, 0, None, 1, 'ptr', 64, 38, 38, 64, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 256, ('fold', 256, 131102.0, True, True, False), None, 0, None, 1, 'ptr', 256, 131102, 131102, 256, 'ptr', 1, 0)),
    ('bn_apply_cells', ('ptr', 256, ('fold', 256, 19.0, True, True, False), None, 0, None, 1, 'ptr', 256, 19, 19, 256, 'ptr', 0, 0)),
    ('bn_apply_cells', ('ptr', 512, ('fold', 512, 66104.0, True, True, False), None, 0, 'ptr', 1, 'ptr', 512, 66104, 33052, 512, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 512, ('fold', 512, 19.0, True, True, False), None, 0, 'ptr', 1, 'ptr', 512, 19, 19, 512, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 512, ('fold', 512, 66104.0, True, True, False), None, 0, None, 1, 'ptr', 1024, 66104, 66104, 512, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 512, ('fold', 512, 19.0, True, True, False), None, 0, None, 1, 'ptr', 1024, 19, 19, 512, None, 0, 0)),
    ('bn_apply_cells', ('ptr', 48, ('fold', 48, 98.0, True, True, False), 'ptr', 48, None, 1, 'ptr', 48, 98, 98, 48, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 192, None, 0, None, 'ptr', 192, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 192, None, 0, 0, 19, 19, 192, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 1, 1, 256, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 131102, 131102, 256, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 19, 19, 256, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 19, 19, 256, 'ptr', 0, 0)),
    ('bn_bwd_apply', ('ptr', 512, 'ptr', 512, 'ptr', 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 66104, 33052, 512, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 512, 'ptr', 512, 'ptr', 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 19, 19, 512, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, 'ptr', 256, 0, 131102, 131102, 256, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 384, 'ptr', 384, None, 'ptr', 384, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 384, 'ptr', 384, 0, 19, 19, 384, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 66104, 66104, 512, None, 0, 0)),
    ('bn_bwd_apply', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 19, 19, 512, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 2048, 'ptr', 2048, None, 'ptr', 2048, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 2048, None, 0, 0, 16410, 16410, 2048, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 2048, 'ptr', 2048, None, 'ptr', 2048, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 2048, None, 0, 0, 8210, 8210, 2048, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 2048, 'ptr', 2048, 'ptr', 'ptr', 2048, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 2048, None, 0, 0, 16410, 8205, 2048, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 2048, 'ptr', 2048, 'ptr', 'ptr', 2048, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 2048, None, 0, 0, 8210, 4105, 2048, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 720, 'ptr', 720, None, 'ptr', 720, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 720, None, 0, 0, 33014, 33014, 720, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 1024, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 1024, None, 0, 0, 33014, 33014, 1024, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 1024, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 1024, None, 0, 0, 8210, 8210, 1024, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, 'ptr', 'ptr', 1024, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 1024, None, 0, 0, 33014, 16507, 1024, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, 'ptr', 'ptr', 1024, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 1024, None, 0, 0, 8210, 4105, 1024, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 48, 'ptr', 48, None, 'ptr', 48, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 48, None, 0, 0, 131102, 131102, 48, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 48, 'ptr', 48, None, 'ptr', 48, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 48, 'ptr', 48, 0, 131102, 131102, 48, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 192, None, 0, None, 'ptr', 192, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 192, None, 0, 0, 19, 19, 192, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 384, 'ptr', 384, None, 'ptr', 384, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 384, None, 0, 0, 19, 19, 384, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 384, 'ptr', 384, None, 'ptr', 384, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 384, 'ptr', 384, 0, 19, 19, 384, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 1, 1, 256, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 131102, 131102, 256, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 64, 'ptr', 64, None, 'ptr', 64, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 64, None, 0, 0, 131102, 131102, 64, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 33014, 33014, 256, 'ptr', 0, 0)),
    ('bn_bwd_cells', ('ptr', 512, 'ptr', 512, 'ptr', 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 66104, 33052, 512, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 512, 'ptr', 512, 'ptr', 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 16410, 8205, 512, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, 'ptr', 256, 0, 131102, 131102, 256, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, 'ptr', 256, 0, 33014, 33014, 256, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 66104, 66104, 512, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 512, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 512, None, 0, 0, 16410, 16410, 512, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 19, 19, 256, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 1280, 'ptr', 1280, None, 'ptr', 256, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 256, None, 0, 0, 19, 19, 256, None, 0, 0)),
    ('bn_bwd_finalize', ('ptr', 7, 48, 2048.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_finalize', ('ptr', 25, 48, 8192.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_finalize', ('ptr', 264, 720, 131072.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_finalize', ('ptr', 1, 256, 19.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_finalize', ('ptr', 26, 192, 2048.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_finalize', ('ptr', 264, 512, 131072.0, 'ptr', 'ptr', 'ptr', 'ptr', None, 0)),
    ('bn_bwd_reduce', ('ptr', 2048, 'ptr', 2048, None, 'ptr', 2048, 'ptr', 'ptr', 8210, 8210, 2048, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 2048, 'ptr', 2048, 'ptr', 'ptr', 2048, 'ptr', 'ptr', 8210, 4105, 2048, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 720, 'ptr', 720, None, 'ptr', 720, 'ptr', 'ptr', 8210, 8210, 720, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 1024, 'ptr', 'ptr', 8210, 8210, 1024, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 1024, 'ptr', 1024, 'ptr', 'ptr', 1024, 'ptr', 'ptr', 8210, 4105, 1024, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 48, 'ptr', 48, None, 'ptr', 48, 'ptr', 'ptr', 131102, 131102, 48, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 192, None, 0, None, 'ptr', 192, 'ptr', 'ptr', 19, 19, 192, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 384, 'ptr', 384, None, 'ptr', 384, 'ptr', 'ptr', 19, 19, 384, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 1, 1, 256, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 33014, 33014, 256, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 33014, 33014, 256, 'ptr', 'ptr', 0, 0)),
    ('bn_bwd_reduce', ('ptr', 512, 'ptr', 512, 'ptr', 'ptr', 512, 'ptr', 'ptr', 16410, 8205, 512, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 1024, 'ptr', 1024, None, 'ptr', 512, 'ptr', 'ptr', 16410, 16410, 512, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 256, 'ptr', 256, None, 'ptr', 256, 'ptr', 'ptr', 19, 19, 256, 'ptr', None, 0, 0)),
    ('bn_bwd_reduce', ('ptr', 1280, 'ptr', 1280, None, 'ptr', 256, 'ptr', 'ptr', 19, 19, 256, 'ptr', None, 0, 0)),
    ('bn_finalize', ('ptr', 148, 48, 48, 4096.0, 'ptr', 'ptr', 1e-05, 0.1, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', None, None, 0)),
    ('bn_finalize', ('ptr', 148, 64, 64, 4096.0, 'ptr', 'ptr', 1e-05, 0.1, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', None, None, 0)),
    ('masked_accum', ('ptr', 4096, None, 0, 'ptr', 4096, 0, 8210, 4096, 0)),
    ('masked_accum', ('ptr', 512, None, 0, 'ptr', 512, 0, 19, 512, 0)),
    ('masked_accum', ('ptr', 1024, None, 0, 'ptr', 1024, 1, 33014, 1024, 0)),
    ('masked_accum', ('ptr', 512, None, 0, 'ptr', 512, 1, 19, 512, 0)),
    ('masked_accum', ('ptr', 384, 'ptr', 384, 'ptr', 384, 0, 19, 384, 0)),
    ('masked_accum', ('ptr', 192, 'ptr', 192, 'ptr', 192, 1, 19, 192, 0)),
    ('masked_accum', ('ptr', 720, 'ptr', 720, 'ptr', 48, 1, 98, 48, 0)),
    ('upsample_adjoint', ('ptr', 96, 'ptr', 96, 1, 132, 268, 96, 'ptr', 96, 33, 67, 0, 0)),
    ('upsample_adjoint', ('ptr', 96, 'ptr', 96, 1, 12, 28, 96, 'ptr', 96, 3, 7, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, None, 0, 1, 132, 268, 192, 'ptr', 192, 33, 67, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 260, 524, 48, 'ptr', 48, 65, 131, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 12, 28, 48, 'ptr', 48, 3, 7, 0, 0)),
    ('upsample_adjoint', ('ptr', 48, 'ptr', 48, 1, 264, 536, 48, 'ptr', 48, 33, 67, 0, 0)),
    ('upsample_adjoint', ('ptr', 48, 'ptr', 48, 1, 24, 56, 48, 'ptr', 48, 3, 7, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, None, 0, 1, 136, 280, 384, 'ptr', 384, 17, 35, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 264, 536, 48, 'ptr', 48, 33, 67, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 24, 56, 48, 'ptr', 48, 3, 7, 0, 0)),
    ('upsample_adjoint', ('ptr', 96, 'ptr', 96, 1, 130, 262, 96, 'ptr', 96, 65, 131, 0, 0)),
    ('upsample_adjoint', ('ptr', 192, 'ptr', 192, 1, 6, 14, 192, 'ptr', 192, 3, 7, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, None, 0, 1, 130, 262, 96, 'ptr', 96, 65, 131, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 258, 518, 48, 'ptr', 48, 129, 259, 0, 0)),
    ('upsample_adjoint', ('ptr', 720, 'ptr', 720, 1, 6, 14, 48, 'ptr', 48, 3, 7, 0, 0)),
    ('accum_pred', ('ptr', 'ptr', 1, 19, 129, 257, 0, 1, 0)),
    ('accum_pred', ('ptr', 'ptr', 1, 3, 513, 1025, 1, 0, 0)),
    ('accum_pred', ('ptr', 'ptr', 1, 19, 129, 257, 1, 1, 0)),
    ('argmax_hist', ('ptr', 1, 19, 1048577, 0.5, 'ptr', 'ptr', 'ptr', 'ptr', 0)),
    ('bias_grad', ('ptr', 32, 513, 19, 'ptr', 0)),
    ('blend', ('ptr', 'ptr', 'ptr', 'ptr', 1, 19, 32769, 0, 0)),
    ('blend', ('ptr', 'ptr', 'ptr', 'ptr', 1, 19, 32769, 1, 0)),
    ('blend', ('ptr', 'ptr', None, 'ptr', 1, 19, 32769, 2, 0)),
    ('broadcast_pixels', ('ptr', 4096, 1, 1025, 4096, 3.0517578125e-05, 'ptr', 4096, 1, 0)),
    ('broadcast_pixels', ('ptr', 256, 1, 16385, 256, 1.0, 'ptr', 1280, 0, 0)),
    ('broadcast_pixels', ('ptr', 256, 1, 33, 256, 1.0, 'ptr', 1280, 0, 0)),
    ('cast_rows', ('ptr', 512, 'ptr', 512, 2, 512, 0, 0)),
    ('cast_rows', ('ptr', 256, 'ptr', 256, 2, 256, 1, 0)),
    ('channel_stats', ('ptr', 64, 8193, 64, 'ptr', 0)),
    ('class_softmax_bwd', ('ptr', 20, 'ptr', 513, 19, 0.0625, 'ptr', 0)),
    ('class_softmax_fwd', ('ptr', 20, 524289, 19, 0.0625, 'ptr', 0)),
    ('class_softmax_fwd', ('ptr', 20, 257, 19, 0.0625, 'ptr', 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 96, 1, ((129, 257, 96, True), (129, 257, 96, False))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 5, 9, 96, 1, ((5, 9, 96, True), (5, 9, 96, False))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 192, 1, ((129, 257, 192, True), (129, 257, 192, True), (129, 257, 192, False))), 'ptr', 192, 0)),
    ('fuse_fwd', (('fuse', 1, 3, 5, 192, 1, ((3, 5, 192, True), (3, 5, 192, True), (3, 5, 192, False))), 'ptr', 192, 0)),
    ('fuse_fwd', (('fuse', 1, 65, 129, 384, 1, ((65, 129, 384, True), (65, 129, 384, True), (65, 129, 384, True), (65, 129, 384, False))), 'ptr', 384, 0)),
    ('fuse_fwd', (('fuse', 1, 2, 3, 384, 1, ((2, 3, 384, True), (2, 3, 384, True), (2, 3, 384, True), (2, 3, 384, False))), 'ptr', 384, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 192, 1, ((129, 257, 192, True), (129, 257, 192, True), (129, 257, 192, False), (64, 128, 192, True))), 'ptr', 192, 0)),
    ('fuse_fwd', (('fuse', 1, 3, 5, 192, 1, ((3, 5, 192, True), (3, 5, 192, True), (3, 5, 192, False), (1, 2, 192, True))), 'ptr', 192, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 96, 1, ((129, 257, 96, True), (129, 257, 96, False), (64, 128, 96, True))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 5, 9, 96, 1, ((5, 9, 96, True), (5, 9, 96, False), (2, 4, 96, True))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 96, 1, ((129, 257, 96, True), (129, 257, 96, False), (64, 128, 96, True), (32, 64, 96, True))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 5, 9, 96, 1, ((5, 9, 96, True), (5, 9, 96, False), (2, 4, 96, True), (1, 2, 96, True))), 'ptr', 96, 0)),
    ('fuse_fwd', (('fuse', 1, 257, 513, 48, 1, ((257, 513, 48, False), (128, 256, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 5, 9, 48, 1, ((5, 9, 48, False), (2, 4, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 257, 513, 48, 1, ((257, 513, 48, False), (128, 256, 48, True), (64, 128, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 5, 9, 48, 1, ((5, 9, 48, False), (2, 4, 48, True), (1, 2, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 257, 513, 48, 1, ((257, 513, 48, False), (128, 256, 48, True), (64, 128, 48, True), (32, 64, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 9, 17, 48, 1, ((9, 17, 48, False), (4, 8, 48, True), (2, 4, 48, True), (1, 2, 48, True))), 'ptr', 48, 0)),
    ('fuse_fwd', (('fuse', 1, 257, 513, 48, 1, ((257, 513, 48, False), (128, 256, 48, True), (64, 128, 48, True), (32, 64, 48, True))), 'ptr', 720, 0)),
    ('fuse_fwd', (('fuse', 1, 9, 17, 48, 1, ((9, 17, 48, False), (4, 8, 48, True), (2, 4, 48, True), (1, 2, 48, True))), 'ptr', 720, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 256, 1, ((129, 257, 256, True), (129, 257, 256, True))), 'ptr', 256, 0)),
    ('fuse_fwd', (('fuse', 1, 129, 257, 96, 0, ((64, 128, 96, False),)), 'ptr', 720, 0)),
    ('image_prep', ('ptr', 1, 1025, 2049, 'ptr', 513, 1025, 0)),
    ('image_prep', ('ptr', 1, 33, 65, 'ptr', 17, 33, 0)),
    ('image_prep', ('ptr', 1, 513, 1025, 'ptr', 513, 1025, 0)),
    ('maxpool3x3s2_bwd', ('ptr', 64, 'ptr', 64, 1, 256, 512, 64, 'ptr', 64, 0, 0)),
    ('maxpool3x3s2_bwd', ('ptr', 128, 'ptr', 128, 1, 128, 256, 128, 'ptr', 128, 1, 0)),
    ('maxpool3x3s2_fwd', ('ptr', 64, 1, 512, 1024, 64, 'ptr', 64, 0)),
    ('maxpool3x3s2_fwd', ('ptr', 64, 1, 8, 16, 64, 'ptr', 64, 0)),
    ('resize_nchw', ('ptr', 19, 257, 513, 'ptr', 129, 257, 0)),
    ('resize_nchw', ('ptr', 19, 65, 129, 'ptr', 129, 257, 0)),
    ('resize_nchw', ('ptr', 1, 9, 17, 'ptr', 17, 33, 0)),
    ('resize_to_nchw', ('ptr', 1, 1, 257, 513, 1, 1, 'ptr', 1025, 2049, 0)),
    ('resize_to_nchw', ('ptr', 1, 1, 5, 9, 1, 1, 'ptr', 17, 33, 0)),
    ('resize_to_nchw', ('ptr', 20, 1, 33, 65, 19, 0, 'ptr', 129, 257, 0)),
    ('spatial_softmax_bwd', ('ptr', 20, 'ptr', 1, 131073, 19, 'ptr', 'ptr', 1, 0)),
    ('spatial_softmax_bwd', ('ptr', 20, 'ptr', 1, 257, 19, 'ptr', 'ptr', 1, 0)),
    ('spatial_softmax_fwd', ('ptr', 20, 1, 131073, 19, 'ptr', 'ptr', None, 0)),
    ('spatial_softmax_fwd', ('ptr', 20, 1, 257, 19, 'ptr', 'ptr', None, 0)),
    ('spatial_sum', ('ptr', 4096, 1, 9, 4096, 0.00048828125, 'ptr', 'ptr', 4096, 0, 0)),
    ('spatial_sum', ('ptr', 720, 1, 4097, 720, 7.62939453125e-06, 'ptr', 'ptr', 720, 0, 0)),
    ('spatial_sum', ('ptr', 4096, 1, 4097, 4096, 3.0517578125e-05, 'ptr', 'ptr', 4096, 0, 0)),
    ('spatial_sum', ('ptr', 1280, 1, 4097, 256, 1.0, 'ptr', 'ptr', 256, 0, 0)),
    ('transpose_pad', ('ptr', 0, 19, 256, 256, 'ptr', 24, 0)),
    # edge rows no traced program reaches: npix 2 (and 1, 19 above), |mean| / std of 0, 16 and 64, a non-integer
    # resampling ratio (33 -> 17) and ratio 1 of the adjoint, accumulating, a non-integer fuse_fwd term (17 -> 33),
    # broadcast_pixels accumulating at scale 2^-13, a spatial softmax of less than one block over two images
    ('fuse_fwd', (('fuse', 1, 33, 35, 48, 1, ((33, 35, 48, False), (17, 18, 48, True))), 'ptr', 48, 0)),
    ('broadcast_pixels', ('ptr', 4096, 1, 1025, 4096, 2.0 ** -13, 'ptr', 4096, 1, 0)),
    ('spatial_softmax_fwd', ('ptr', 20, 2, 200, 19, 'ptr', 'ptr', None, 0)),
    ('bn_apply_cells', ('ptr', 64, ('fold', 64, 2.0, True, True, False), None, 0, None, 1, 'ptr', 64, 2, 2, 64, None, 0, 0)),
    ('bn_bwd_cells', ('ptr', 64, 'ptr', 64, None, 'ptr', 64, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 64, None, 0, 0, 2, 2, 64, None, 0, 0)),
    ('bn_finalize', ('ptr', 148, 64, 64, 33014.0, 'ptr', 'ptr', 1e-05, 0.1, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', None, None, 0), 0),
    ('bn_finalize', ('ptr', 148, 64, 64, 33014.0, 'ptr', 'ptr', 1e-05, 0.1, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', None, None, 0), 16),
    ('bn_finalize', ('ptr', 148, 64, 64, 33014.0, 'ptr', 'ptr', 1e-05, 0.1, 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', 'ptr', None, None, 0), 64),
    ('bn_apply_cells', ('ptr', 64, ('fold', 64, 33014.0, True, True, False), None, 0, None, 0, 'ptr', 64, 33014, 33014, 64, None, 0, 0), 0),
    ('bn_apply_cells', ('ptr', 64, ('fold', 64, 33014.0, True, False, True), None, 0, None, 0, 'ptr', 64, 33014, 33014, 64, None, 0, 0), 16),
    ('bn_apply_cells', ('ptr', 64, ('fold', 64, 33014.0, True, True, False), None, 0, None, 0, 'ptr', 64, 33014, 33014, 64, None, 0, 0), 64),
    ('upsample_adjoint', ('ptr', 48, None, 0, 1, 33, 67, 48, 'ptr', 48, 17, 31, 1, 0)),
    ('upsample_adjoint', ('ptr', 64, 'ptr', 64, 2, 9, 13, 64, 'ptr', 72, 9, 13, 0, 0)),
]


def row_id(row):
    name, a = row[0], row[1]
    return "%s-%08x%s" % (name, zlib.crc32(repr(a).encode()), "-ratio%d" % row[2] if len(row) > 2 else "")


# ------------------------------------------------------------------------------------------------------------ GPU part
def _torch():
    import torch
    from b200seg import raw
    return torch, raw


def _ulp_bf16(r):
    torch, _ = _torch()
    _m, e = torch.frexp(r)
    return torch.where(r == 0, torch.zeros_like(r), torch.ldexp(torch.ones_like(r), e - 8))


class Buf:
    """NaN-filled [rows, ld] buffer plus a NaN guard behind it; the operand is the slice [:, :c] (optionally filled)."""

    def __init__(self, rows, c, ld, dtype, fill=None):
        torch, _ = _torch()
        self.flat = torch.full((rows * ld + 4096,), float("nan"), dtype=dtype, device="cuda")
        self.v = self.flat[: rows * ld].view(rows, ld)[:, :c]
        self.c = c
        if fill is not None:
            self.v.copy_(fill)

    def data_ptr(self):
        return self.v.data_ptr()

    def check(self, what):
        torch, _ = _torch()
        itype = torch.int16 if self.flat.dtype == torch.bfloat16 else torch.int32
        nan = torch.full((1,), float("nan"), dtype=self.flat.dtype, device="cuda").view(itype)
        assert bool(torch.isfinite(self.v).all()), "%s: non-finite or unwritten output element" % what
        outside = torch.ones(self.flat.shape, dtype=torch.bool, device="cuda")
        rows, ld = self.v.shape[0], self.v.stride(0)
        outside[: rows * ld].view(rows, ld)[:, : self.c] = False
        bad = int((self.flat.view(itype)[outside] != nan).sum())
        assert bad == 0, "%s: %d elements outside the output slice were written" % (what, bad)

    def bits(self):
        torch, _ = _torch()
        return self.flat.view(torch.uint8).clone()


def _call(name, a, ops):
    """Launches entry point `name` with the row's arguments, operands from ops {argument index: tensor, Buf or
    ctypes structure}, on the current stream."""
    from b200seg import raw
    args = []
    for i, x in enumerate(a):
        if x == PTR:
            args.append(ops[i].data_ptr())
        elif isinstance(x, tuple):
            args.append(ctypes.byref(ops[i]))
        else:
            args.append(x)
    args[-1] = raw.stream_ptr()
    assert getattr(_lib.lib(), "b200seg_" + name)(*args) == 0, name


def _twice(name, a, inputs, make_outputs):
    """Runs the launch with two fresh sets of outputs ({index: Buf}, plus named extra state); both must agree bit for
    bit. Returns the first set."""
    torch, _ = _torch()
    runs = []
    for _ in range(2):
        outs, extra = make_outputs()
        _call(name, a, {**inputs, **outs})
        runs.append((outs, extra))
    torch.cuda.synchronize()
    (o1, e1), (o2, e2) = runs
    for k in o1:
        if isinstance(o1[k], Buf):
            assert torch.equal(o1[k].bits(), o2[k].bits()), "run-to-run difference in argument %d" % k
    for k in e1:
        assert torch.equal(e1[k].view(torch.uint8), e2[k].view(torch.uint8)), "run-to-run difference in %s" % k
    return o1, e1


MEASURED = {}


def _note(kind, value, what=""):
    MEASURED[kind] = max(MEASURED.get(kind, 0.0), value)
    print("\nMEASURE %-36s %.3e  %s" % (kind.replace(" ", "_"), value, what))


def _check_bf16(out, r, A, what, kind, exact=False, rel=EW_REL):
    """bf16 out against the float64 reference r; A bounds the fp32 arithmetic error."""
    torch, _ = _torch()
    y = out.double()
    if exact:
        bad = int((out.view(torch.int16) != r.to(torch.bfloat16).view(torch.int16)).sum())
        assert bad == 0, "%s: %d outputs differ from round_bf16(reference)" % (what, bad)
        return
    err = (y - r).abs()
    acc = (err - 0.5 * torch.maximum(_ulp_bf16(y), _ulp_bf16(r))).clamp_min(0)
    _note(kind + " err/A", float((acc / A.clamp_min(1e-300)).max()), what)
    ratio = float((err / (_ulp_bf16(r) + rel * A).clamp_min(1e-300)).max())
    mism = float((out != r.to(torch.bfloat16)).double().mean())
    _note(kind + " mismatch", mism if out.numel() >= 1024 else 0.0, what)
    _note(kind + " err/bound", ratio, what)
    assert ratio <= 1.0, "%s: max err/bound %.3f" % (what, ratio)
    limit = MISMATCH_MAX + MISMATCH_FEW / out.numel()
    assert mism <= limit, "%s: %.3f%% of the outputs differ from round_bf16(reference)" % (what, 100 * mism)


def _check_rel(got, r, scale, bound, what, kind):
    """Per-channel statistic got (fp32) against r (float64): |got - r| <= bound * scale."""
    e = float(((got.double() - r).abs() / scale.clamp_min(1e-300)).max())
    _note(kind, e, what)
    assert e <= bound, "%s: error %.3e of the scale, bound %.1e" % (what, e, bound)


def _rng(row):
    torch, _ = _torch()
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(row_id(row).encode()))


def _randn(g, *shape):
    torch, _ = _torch()
    return torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)


def _bf16(t):
    torch, _ = _torch()
    return t.to(torch.bfloat16)


def _f32(t):
    torch, _ = _torch()
    return t.float().contiguous()


def _bn_input(g, npix, c, ratio=None):
    """bf16 [npix, c] with per-channel spread around 1 and mean ratio x std (or about half a std)."""
    torch, _ = _torch()
    std = torch.exp(0.3 * _randn(g, c))
    mean = (ratio * std * torch.sign(_randn(g, c))) if ratio is not None else 0.5 * _randn(g, c)
    return _bf16(mean + std * _randn(g, npix, c))


def _keep(raw, seed, pass_idx, npix, c):
    """Element-wise dropout of the BatchNorm passes: factor 2 where kept, 0 where dropped."""
    return 2.0 * raw.dropout_keep_mask(seed, pass_idx, npix, c).view(npix, c).double()


def _post(g, n, c, hw):
    torch, _ = _torch()
    ps = _f32(torch.exp(0.5 * _randn(g, n, c)))
    return ps, ps.double().repeat_interleave(hw, 0)


def _seed(g):
    torch, _ = _torch()
    return torch.randint(0, 2 ** 62, (1,), generator=g, device="cuda", dtype=torch.int64)


def _bn_stats_ref(yd, count):
    mean = yd.mean(0)
    var = ((yd - mean) ** 2).mean(0)
    unb = var * count / (count - 1) if count > 1 else var
    return mean, var, unb


# ------------------------------------------------------------------------------------------------- BatchNorm forward
def _run_bn_apply(row):
    torch, raw = _torch()
    name, a = row[0], row[1]
    cells = name == "bn_apply_cells"
    o = 1 if cells else 0
    y_ld, res, res_ld, post, relu, z_ld, npix, hw, c, seed, pidx = (a[1], a[4 - o], a[5 - o], a[6 - o], a[7 - o],
                                                                     a[9 - o], a[10 - o], a[11 - o], a[12 - o],
                                                                     a[13 - o], a[14 - o])
    g = _rng(row)
    tag = row_id(row)
    y = _bn_input(g, npix, c, row[2] if len(row) > 2 else None)
    yd = y.double()
    ins = {0: Buf(npix, c, y_ld, torch.bfloat16, y)}
    gamma, beta = _f32(1.0 + 0.25 * _randn(g, c)), _f32(0.25 * _randn(g, c))
    if cells:
        fold = a[2]
        cpad = (c + 15) // 16 * 16
        acc = torch.zeros(2 * cpad, dtype=torch.float64, device="cuda")
        acc[:c], acc[cpad:cpad + c] = yd.sum(0), (yd * yd).sum(0)
        mean, var, unb = _bn_stats_ref(yd, npix)
        inv = 1.0 / torch.sqrt(var + 1e-5)
        sc, sh = gamma.double() * inv, beta.double() - mean * gamma.double() * inv
        rm0, rv0 = _f32(_randn(g, c)), _f32(torch.exp(_randn(g, c)))
    else:
        scale, shift = _f32(1.0 + 0.25 * _randn(g, c)), _f32(0.25 * _randn(g, c))
        ins[2], ins[3] = scale, shift
        sc, sh = scale.double(), shift.double()
    pre = yd * sc + sh
    A = (yd * sc).abs() + sh.abs()
    if cells:       # the kernel forms shift = beta - mean * gamma * invstd in fp32: its error follows the two terms
        A = (yd * sc).abs() + beta.double().abs() + (mean * sc).abs()
    if res is not None:
        rb = _bf16(_randn(g, npix, c))
        ins[4 - o] = Buf(npix, c, res_ld, torch.bfloat16, rb)
        pre, A = pre + rb.double(), A + rb.double().abs()
    r = pre.clamp_min(0) if relu else pre
    if post is not None:
        ps, psd = _post(g, npix // hw, c, hw)
        ins[6 - o] = ps
        r, A = r * psd, A * psd
    if seed is not None:
        sd = _seed(g)
        ins[13 - o] = sd
        k = _keep(raw, sd, pidx, npix, c)
        r, A = r * k, A * k

    def outputs():
        outs = {8 - o: Buf(npix, c, z_ld, torch.bfloat16)}
        extra = {}
        if cells:
            f = _lib.BnFold()
            extra["par"] = torch.full((4, c), float("nan"), dtype=torch.float32, device="cuda")
            extra["cells"] = acc
            f.accum, f.c, f.count, f.eps, f.momentum = acc.data_ptr(), c, float(npix), 1e-5, 0.1
            f.gamma, f.beta = gamma.data_ptr(), beta.data_ptr()
            f.scale, f.shift, f.mean, f.invstd = [extra["par"][i].data_ptr() for i in range(4)]
            if fold[4]:
                extra["rm"], extra["rv"] = rm0.clone(), rv0.clone()
                extra["nbt"] = torch.full((1,), 7, dtype=torch.int64, device="cuda")
                f.running_mean, f.running_var = extra["rm"].data_ptr(), extra["rv"].data_ptr()
                f.num_batches_tracked = extra["nbt"].data_ptr()
            if fold[5]:
                extra["batch"] = torch.full((2 * c,), float("nan"), dtype=torch.float32, device="cuda")
                f.batch_stats_out = extra["batch"].data_ptr()
            outs[2] = f
        return outs, extra
    outs, extra = _twice(name, a, ins, outputs)
    z = outs[8 - o]
    z.check(tag)
    _check_bf16(z.v, r, A, tag, "bn_apply")
    if cells:
        par = extra["par"]
        std = torch.sqrt(var + 1e-5)
        _check_rel(par[0], sc, sc.abs(), PAR_REL, tag + " scale", "bn params")
        _check_rel(par[1], sh, beta.double().abs() + (mean * sc).abs(), PAR_REL, tag + " shift", "bn params")
        _check_rel(par[2], mean, mean.abs() + 2.0 ** -40 * std, PAR_REL, tag + " mean", "bn params")
        _check_rel(par[3], inv, inv, PAR_REL, tag + " invstd", "bn params")
        if fold[4]:
            _check_rel(extra["rm"], 0.9 * rm0.double() + 0.1 * mean, 0.9 * rm0.double().abs() + 0.1 * mean.abs(),
                       PAR_REL, tag + " running mean", "bn params")
            _check_rel(extra["rv"], 0.9 * rv0.double() + 0.1 * unb, 0.9 * rv0.double() + 0.1 * unb, PAR_REL,
                       tag + " running var", "bn params")
            assert int(extra["nbt"]) == 8, "num_batches_tracked %d, want 8" % int(extra["nbt"])
        if fold[5]:
            b = extra["batch"]
            _check_rel(b[:c], mean, mean.abs() + 2.0 ** -40 * std, PAR_REL, tag + " batch mean", "bn params")
            _check_rel(b[c:], unb, unb.clamp_min(1e-30), PAR_REL, tag + " batch var", "bn params")


def _run_bn_finalize(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    G, c, cpad, count = a[1], a[2], a[3], int(a[4])
    g = _rng(row)
    tag = row_id(row)
    ratio = row[2] if len(row) > 2 else None
    yd = _bn_input(g, count, c, ratio).double()
    # fp32 partials of G pixel ranges, as a convolution epilogue or channel_stats emits them
    bounds = [count * i // G for i in range(G + 1)]
    part = torch.zeros((G, 2, cpad), dtype=torch.float32, device="cuda")
    for i in range(G):
        blk = yd[bounds[i]:bounds[i + 1]]
        part[i, 0, :c], part[i, 1, :c] = blk.sum(0).float(), (blk * blk).sum(0).float()
    gamma, beta = _f32(1.0 + 0.25 * _randn(g, c)), _f32(0.25 * _randn(g, c))
    rm0, rv0 = _f32(_randn(g, c)), _f32(torch.exp(_randn(g, c)))
    ins = {0: part, 5: gamma, 6: beta}

    def outputs():
        extra = dict(par=torch.full((4, c), float("nan"), dtype=torch.float32, device="cuda"), rm=rm0.clone(),
                     rv=rv0.clone(), nbt=torch.full((1,), 7, dtype=torch.int64, device="cuda"))
        outs = {9: extra["rm"], 10: extra["rv"], 11: extra["nbt"]}
        outs.update({12 + i: extra["par"][i] for i in range(4)})
        return outs, extra
    _outs, extra = _twice(name, a, ins, outputs)
    # the reference takes the fp32 partials the kernel saw and folds them in float64, like the kernel
    s1, s2 = part[:, 0, :c].double().sum(0), part[:, 1, :c].double().sum(0)
    mean = s1 / count
    var = (s2 / count - mean * mean).clamp_min(0)
    unb = var * count / (count - 1)
    inv = 1.0 / torch.sqrt(var + 1e-5)
    par = extra["par"]
    assert bool(torch.isfinite(par).all()), tag
    sc = gamma.double() * inv
    _check_rel(par[3], inv, inv, PAR_REL, tag + " invstd", "bn params")
    _check_rel(par[2], mean, mean.abs(), PAR_REL, tag + " mean", "bn params")
    _check_rel(par[0], sc, sc.abs(), PAR_REL, tag + " scale", "bn params")
    _check_rel(par[1], beta.double() - mean * sc, beta.double().abs() + (mean * sc).abs(), PAR_REL, tag + " shift",
               "bn params")
    _check_rel(extra["rm"], 0.9 * rm0.double() + 0.1 * mean, 0.9 * rm0.double().abs() + 0.1 * mean.abs(), PAR_REL,
               tag + " running mean", "bn params")
    _check_rel(extra["rv"], 0.9 * rv0.double() + 0.1 * unb, 0.9 * rv0.double() + 0.1 * unb, PAR_REL,
               tag + " running var", "bn params")
    assert int(extra["nbt"]) == 8, "num_batches_tracked %d, want 8" % int(extra["nbt"])


# ------------------------------------------------------------------------------------------------ BatchNorm backward
def _bn_bwd_data(row, npix, c, dz_ld, mask, mask_ld, post, y_ld, hw, seed, pidx, ins, idx):
    """Inputs of the backward passes (idx: argument indices of dz, mask, post, y, mean, invstd, seed) and the float64
    g, xhat of the reference."""
    torch, raw = _torch()
    g = _rng(row)
    dz = _bf16(_randn(g, npix, c))
    y = _bn_input(g, npix, c)
    yd = y.double()
    mean = _f32(yd.mean(0) + 0.01 * _randn(g, c))
    invstd = _f32(1.0 / (((yd - yd.mean(0)) ** 2).mean(0) + 1e-5).sqrt())
    ins.update({idx[0]: Buf(npix, c, dz_ld, torch.bfloat16, dz), idx[3]: Buf(npix, c, y_ld, torch.bfloat16, y),
                idx[4]: mean, idx[5]: invstd})
    gd = dz.double()
    if post is not None:
        ps, psd = _post(g, npix // hw, c, hw)
        ins[idx[2]] = ps
        gd = gd * psd
    if seed is not None:
        sd = _seed(g)
        ins[idx[6]] = sd
        gd = gd * _keep(raw, sd, pidx, npix, c)
    if mask is not None:
        mk = _bf16(_randn(g, npix, c))
        ins[idx[1]] = Buf(npix, c, mask_ld, torch.bfloat16, mk)
        gd = torch.where(mk.double() > 0, gd, torch.zeros_like(gd))
    xhat = (yd - mean.double()) * invstd.double()
    return g, gd, xhat, invstd.double()


def _check_stat_sums(got, want, mag, what, acc=None):
    """Sums of the backward pass within STAT_REL of the sum of magnitudes mag, plus the rounding of the fp32 parameter
    gradient acc they are added to."""
    scale = mag if acc is None else mag + (2.0 ** -23 / STAT_REL) * acc.abs()
    _check_rel(got, want, scale, STAT_REL, what, "bn_bwd sums")


def _run_bn_bwd(row):
    torch, raw = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    cells = name == "bn_bwd_cells"
    if cells:
        (dz_ld, mask, mask_ld, post, y_ld, dy_ld, g_out, g_ld, g_acc, npix, hw, c, seed, pidx) = (
            a[1], a[2], a[3], a[4], a[6], a[14], a[15], a[16], a[17], a[18], a[19], a[20], a[21], a[22])
        idx = (0, 2, 4, 5, 7, 8, 21)
        gam_i, dy_i, g_i = 9, 13, 15
    else:
        (dz_ld, mask, mask_ld, post, y_ld, dy_ld, g_out, g_ld, g_acc, npix, hw, c, seed, pidx) = (
            a[1], a[2], a[3], a[4], a[6], a[13], a[14], a[15], a[16], a[17], a[18], a[19], a[20], a[21])
        idx = (0, 2, 4, 5, 7, 8, 20)
        gam_i, dy_i, g_i = 9, 12, 14
    ins = {}
    g, gd, xhat, inv = _bn_bwd_data(row, npix, c, dz_ld, mask, mask_ld, post, y_ld, hw, seed, pidx, ins, idx)
    gamma = _f32(1.0 + 0.25 * _randn(g, c))
    ins[gam_i] = gamma
    s1, s2 = gd.sum(0), (gd * xhat).sum(0)
    m1, m2 = gd.abs().sum(0), (gd * xhat).abs().sum(0)
    if cells:
        c1, c2 = s1 / npix, s2 / npix
        A1, A2 = m1 / npix, m2 / npix
        d0 = _f32(_randn(g, 2, c))
    else:
        c1f, c2f = _f32(s1 / npix), _f32(s2 / npix)
        ins[10], ins[11] = c1f, c2f
        c1, c2 = c1f.double(), c2f.double()
        A1, A2 = c1.abs(), c2.abs()
    gi = gamma.double() * inv
    r = gi * (gd - c1 - xhat * c2)
    A = gi.abs() * (gd.abs() + A1 + xhat.abs() * A2)
    old = _bf16(_randn(g, npix, c)) if g_acc else None

    def outputs():
        outs = {dy_i: Buf(npix, c, dy_ld, torch.bfloat16)}
        extra = {}
        if g_out is not None:
            outs[g_i] = Buf(npix, c, g_ld, torch.bfloat16, old)
        if cells:
            extra["dgb"] = d0.clone()
            extra["cells"] = torch.zeros(2 * c, dtype=torch.float64, device="cuda")
            outs[10], outs[11], outs[12] = extra["dgb"][0], extra["dgb"][1], extra["cells"]
        return outs, extra
    outs, extra = _twice(name, a, ins, outputs)
    outs[dy_i].check(tag + " dy")
    _check_bf16(outs[dy_i].v, r, A, tag + " dy", "bn_bwd dy")
    if g_out is not None:
        outs[g_i].check(tag + " g_out")
        rg, Ag = gd, gd.abs()
        if g_acc:
            rg, Ag = rg + old.double(), Ag + old.double().abs()
        _check_bf16(outs[g_i].v, rg, Ag, tag + " g_out", "bn_bwd g_out")
    if cells:
        dgamma, dbeta = extra["dgb"][0].double(), extra["dgb"][1].double()
        _check_stat_sums(dbeta, d0[1].double() + s1, m1, tag + " dbeta", dbeta)
        _check_stat_sums(dgamma, d0[0].double() + s2, m2, tag + " dgamma", dgamma)
        _check_stat_sums(extra["cells"][:c], s1, m1, tag + " cells sum g")
        _check_stat_sums(extra["cells"][c:], s2, m2, tag + " cells sum g xhat")


def _run_bn_bwd_reduce(row):
    torch, raw = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    dz_ld, mask, mask_ld, post, y_ld, npix, hw, c, seed, pidx = (a[1], a[2], a[3], a[4], a[6], a[9], a[10], a[11],
                                                                  a[13], a[14])
    ins = {}
    _g, gd, xhat, _inv = _bn_bwd_data(row, npix, c, dz_ld, mask, mask_ld, post, y_ld, hw, seed, pidx, ins,
                                      (0, 2, 4, 5, 7, 8, 13))
    grid = _lib.lib().b200seg_bn_bwd_grid(npix, c)
    outs, _ = _twice(name, a, ins, lambda: ({12: Buf(grid, 2 * c, 2 * c, torch.float32)}, {}))
    outs[12].check(tag + " partials")
    part = outs[12].v.double().view(grid, 2, c).sum(0)
    _check_stat_sums(part[0], gd.sum(0), gd.abs().sum(0), tag + " sum g")
    _check_stat_sums(part[1], (gd * xhat).sum(0), (gd * xhat).abs().sum(0), tag + " sum g xhat")


def _run_bn_bwd_finalize(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    G, c, count = a[1], a[2], a[3]
    g = _rng(row)
    part = _f32(_randn(g, G, 2, c) * 30.0)
    d0 = _f32(_randn(g, 2, c))

    def outputs():
        extra = dict(dgb=d0.clone(), cc=torch.full((2, c), float("nan"), dtype=torch.float32, device="cuda"))
        return {4: extra["dgb"][0], 5: extra["dgb"][1], 6: extra["cc"][0], 7: extra["cc"][1]}, extra
    _outs, extra = _twice(name, a, {0: part}, outputs)
    s = part.double().sum(0)
    m = part.double().abs().sum(0)
    dg = extra["dgb"].double()
    _check_stat_sums(dg[1], d0[1].double() + s[0], m[0], tag + " dbeta", dg[1])
    _check_stat_sums(dg[0], d0[0].double() + s[1], m[1], tag + " dgamma", dg[0])
    _check_stat_sums(extra["cc"][0], s[0] / count, m[0] / count, tag + " c1")
    _check_stat_sums(extra["cc"][1], s[1] / count, m[1] / count, tag + " c2")


# ------------------------------------------------------------------------------------- masked accumulate, resampling
def _run_masked_accum(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    src_ld, mask, mask_ld, dst_ld, acc, npix, c = a[1], a[2], a[3], a[5], a[6], a[7], a[8]
    g = _rng(row)
    src = _bf16(_randn(g, npix, c))
    ins = {0: Buf(npix, c, src_ld, torch.bfloat16, src)}
    r = src.double()
    if mask is not None:
        mk = _bf16(_randn(g, npix, c))
        ins[2] = Buf(npix, c, mask_ld, torch.bfloat16, mk)
        r = torch.where(mk.double() > 0, r, torch.zeros_like(r))
    A = r.abs()
    old = _bf16(_randn(g, npix, c)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    outs, _ = _twice(name, a, ins, lambda: ({4: Buf(npix, c, dst_ld, torch.bfloat16, old)}, {}))
    outs[4].check(tag)
    _check_bf16(outs[4].v, r, A, tag, "masked_accum", exact=not acc)


def _interp(out_size, in_size):
    """[out_size, in_size] float64 bilinear weights, PyTorch's align_corners=False rule: fp32 scale in / out, source
    index scale * (dst + 0.5) - 0.5 rounded once to fp32, clamped at 0; i1 = min(i0 + 1, in - 1)."""
    import numpy as np
    torch, _ = _torch()
    sc = float(np.float32(in_size) / np.float32(out_size))
    m = np.zeros((out_size, in_size))
    for d in range(out_size):
        src = max(0.0, float(np.float32(sc * (d + 0.5) - 0.5)))
        i0 = min(int(src), in_size - 1)
        i1 = i0 + (1 if i0 < in_size - 1 else 0)
        lam = src - i0
        m[d, i0] += 1.0 - lam
        m[d, i1] += lam
    return torch.from_numpy(m).cuda()


def _run_upsample_adjoint(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    g_ld, mask, mask_ld, n, H, W, c, out_ld, h, w, acc = a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[9], a[10], a[11], \
        a[12]
    rg = _rng(row)
    gr = _bf16(_randn(rg, n * H * W, c))
    ins = {0: Buf(n * H * W, c, g_ld, torch.bfloat16, gr)}
    gd = gr.double()
    if mask is not None:
        mk = _bf16(_randn(rg, n * H * W, c))
        ins[2] = Buf(n * H * W, c, mask_ld, torch.bfloat16, mk)
        gd = torch.where(mk.double() > 0, gd, torch.zeros_like(gd))
    Uy, Ux = _interp(H, h), _interp(W, w)
    gd = gd.view(n, H, W, c)
    adj = lambda t: torch.einsum("Xx,nyXc->nyxc", Ux, torch.einsum("Yy,nYXc->nyXc", Uy, t))      # noqa: E731
    r = adj(gd).reshape(n * h * w, c)
    A = adj(gd.abs()).reshape(n * h * w, c)
    old = _bf16(_randn(rg, n * h * w, c)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    outs, _ = _twice(name, a, ins, lambda: ({8: Buf(n * h * w, c, out_ld, torch.bfloat16, old)}, {}))
    outs[8].check(tag)
    _check_bf16(outs[8].v, r, A, tag, "upsample_adjoint")


# --------------------------------------------------------------------------- fusion, softmaxes, pooling, sums, layout
def _check_f32(out, r, A, what, kind, rel=None):
    """fp32 out against the float64 reference r: |out - r| <= rel * A (EW_REL by default)."""
    rel = EW_REL if rel is None else rel
    e = float(((out.double() - r).abs() / A.clamp_min(1e-300)).max())
    _note(kind + " err/A", e, what)
    assert bool(torch_isfinite(out)), "%s: non-finite output" % what
    assert e <= rel, "%s: error %.3e of A, bound %.1e" % (what, e, rel)


def torch_isfinite(t):
    torch, _ = _torch()
    return torch.isfinite(t).all()


def _resample(x, n, h, w, H, W):
    """x [n * h * w, c] float64 -> [n * H * W, c] bilinear (align_corners=False), and the weights' |.| form."""
    torch, _ = _torch()
    Uy, Ux = _interp(H, h), _interp(W, w)
    c = x.shape[1]
    t = torch.einsum("Yy,nyxc->nYxc", Uy, x.reshape(n, h, w, c))       # one axis at a time: no 4-index intermediate
    return torch.einsum("Xx,nYxc->nYXc", Ux, t).reshape(n * H * W, c)


def _run_fuse_fwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    _f, n, h, w, c, relu, terms = a[0]
    g = _rng(row)
    d = _lib.FuseDesc()
    d.nterms, d.n, d.h, d.w, d.c, d.relu = len(terms), n, h, w, c, relu
    keep = []
    r = torch.zeros((n * h * w, c), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    for i, (th, tw, ld, aff) in enumerate(terms):
        x = _bf16(_randn(g, n * th * tw, c))
        b = Buf(n * th * tw, c, ld, torch.bfloat16, x)
        t = d.term[i]
        t.x, t.ld, t.h, t.w = b.data_ptr(), ld, th, tw
        keep.append(b)
        v, va = _resample(x.double(), n, th, tw, h, w), _resample(x.double().abs(), n, th, tw, h, w)
        if aff:
            sc, sh = _f32(1.0 + 0.25 * _randn(g, c)), _f32(0.25 * _randn(g, c))
            keep += [sc, sh]
            t.scale, t.shift = sc.data_ptr(), sh.data_ptr()
            v, va = v * sc.double() + sh.double(), va * sc.double().abs() + sh.double().abs()
        r, A = r + v, A + va
    if relu:
        r = r.clamp_min(0)
    outs, _ = _twice(name, a, {}, lambda: ({0: d, 1: Buf(n * h * w, c, a[2], torch.bfloat16)}, {}))
    outs[1].check(tag)
    _check_bf16(outs[1].v, r, A, tag, "fuse_fwd")


def _run_spatial_softmax_fwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ld, n, P, K = a[1], a[2], a[3], a[4]
    g = _rng(row)
    x = _f32(2.0 * _randn(g, n * P, K))
    B = _lib.lib().b200seg_spatial_softmax_blocks(P)
    xs = x.double().view(n, P, K)
    r = torch.zeros((n, P, 32), dtype=torch.float64, device="cuda")
    r[..., :K] = torch.softmax(xs, dim=1)
    r = r.view(n * P, 32)
    ins = {0: Buf(n * P, K, ld, torch.float32, x), 5: torch.empty(n * B * 64, dtype=torch.float32, device="cuda")}
    outs, _ = _twice(name, a, ins, lambda: ({6: Buf(n * P, 32, 32, torch.bfloat16)}, {}))
    outs[6].check(tag)
    _check_bf16(outs[6].v, r, r, tag, "softmax")


def _run_spatial_softmax_bwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ldd, n, P, K, acc = a[1], a[3], a[4], a[5], a[8]
    g = _rng(row)
    p = torch.zeros((n * P, 32), dtype=torch.float64, device="cuda")
    p[:, :K] = torch.softmax(2.0 * _randn(g, n, P, K), dim=1).view(n * P, K)
    p = _bf16(p)
    d = _f32(_randn(g, n * P, K))
    B = _lib.lib().b200seg_spatial_softmax_blocks(P)
    pd, dd = p.double()[:, :K].view(n, P, K), d.double().view(n, P, K)
    S = (pd * dd).sum(1, keepdim=True)
    Sa = (pd * dd.abs()).sum(1, keepdim=True)
    r = torch.zeros((n * P, 32), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    r[:, :K] = (pd * (dd - S)).view(n * P, K)
    A[:, :K] = (pd * (dd.abs() + Sa)).view(n * P, K)
    old = _bf16(_randn(g, n * P, 32)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    ins = {0: Buf(n * P, K, ldd, torch.float32, d), 2: p, 6: torch.empty(n * B * 32, dtype=torch.float32, device="cuda")}
    outs, _ = _twice(name, a, ins, lambda: ({7: Buf(n * P, 32, 32, torch.bfloat16, old)}, {}))
    outs[7].check(tag)
    _check_bf16(outs[7].v, r, A, tag, "softmax")


def _run_class_softmax_fwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ld, P, K, scale = a[1], a[2], a[3], a[4]
    g = _rng(row)
    x = _f32(8.0 * _randn(g, P, K))
    r = torch.zeros((P, 32), dtype=torch.float64, device="cuda")
    r[:, :K] = torch.softmax(x.double() * scale, dim=1)
    outs, _ = _twice(name, a, {0: Buf(P, K, ld, torch.float32, x)},
                     lambda: ({5: Buf(P, 32, 32, torch.bfloat16)}, {}))
    outs[5].check(tag)
    _check_bf16(outs[5].v, r, r, tag, "softmax")


def _run_class_softmax_bwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ld, P, K, scale = a[1], a[3], a[4], a[5]
    g = _rng(row)
    s = torch.zeros((P, 32), dtype=torch.float64, device="cuda")
    s[:, :K] = torch.softmax(2.0 * _randn(g, P, K), dim=1)
    s = _bf16(s)
    dg = _f32(_randn(g, P, K))
    sd, gd = s.double()[:, :K], dg.double()
    r = torch.zeros((P, 32), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    r[:, :K] = scale * sd * (gd - (sd * gd).sum(1, keepdim=True))
    A[:, :K] = abs(scale) * sd * (gd.abs() + (sd * gd.abs()).sum(1, keepdim=True))
    outs, _ = _twice(name, a, {0: Buf(P, K, ld, torch.float32, dg), 2: s},
                     lambda: ({6: Buf(P, 32, 32, torch.bfloat16)}, {}))
    outs[6].check(tag)
    _check_bf16(outs[6].v, r, A, tag, "softmax")


def _nchw4(t, n, h, w, c):
    return t.reshape(n, h, w, c).permute(0, 3, 1, 2)


def _nhwc2(t):
    n, c, h, w = t.shape
    return t.permute(0, 2, 3, 1).reshape(n * h * w, c)


def _run_maxpool_fwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    x_ld, n, h, w, c, y_ld = a[1], a[2], a[3], a[4], a[5], a[7]
    g = _rng(row)
    x = _bf16(_randn(g, n * h * w, c))
    r = _nhwc2(torch.nn.functional.max_pool2d(_nchw4(x.double(), n, h, w, c), 3, 2, 1))
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    outs, _ = _twice(name, a, {0: Buf(n * h * w, c, x_ld, torch.bfloat16, x)},
                     lambda: ({6: Buf(n * ho * wo, c, y_ld, torch.bfloat16)}, {}))
    outs[6].check(tag)
    _check_bf16(outs[6].v, r, r.abs(), tag, "maxpool", exact=True)


def _run_maxpool_bwd(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    x_ld, dy_ld, n, h, w, c, dx_ld, acc = a[1], a[3], a[4], a[5], a[6], a[7], a[9], a[10]
    g = _rng(row)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = _bf16(_randn(g, n * h * w, c))
    dy = _bf16(_randn(g, n * ho * wo, c))
    xd = _nchw4(x.double(), n, h, w, c).contiguous().requires_grad_()
    torch.nn.functional.max_pool2d(xd, 3, 2, 1).backward(_nchw4(dy.double(), n, ho, wo, c))
    r = _nhwc2(xd.grad)
    xa = _nchw4(x.double(), n, h, w, c).contiguous().requires_grad_()
    torch.nn.functional.max_pool2d(xa, 3, 2, 1).backward(_nchw4(dy.double().abs(), n, ho, wo, c))
    A = _nhwc2(xa.grad)
    old = _bf16(_randn(g, n * h * w, c)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    ins = {0: Buf(n * h * w, c, x_ld, torch.bfloat16, x), 2: Buf(n * ho * wo, c, dy_ld, torch.bfloat16, dy)}
    outs, _ = _twice(name, a, ins, lambda: ({8: Buf(n * h * w, c, dx_ld, torch.bfloat16, old)}, {}))
    outs[8].check(tag)
    _check_bf16(outs[8].v, r, A, tag, "maxpool")


def _run_channel_stats(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    x_ld, npix, c = a[1], a[2], a[3]
    g = _rng(row)
    x = _bn_input(g, npix, c)
    grid = _lib.lib().b200seg_channel_stats_grid(npix, c)
    outs, _ = _twice(name, a, {0: Buf(npix, c, x_ld, torch.bfloat16, x)},
                     lambda: ({4: Buf(grid, 2 * c, 2 * c, torch.float32)}, {}))
    outs[4].check(tag)
    p = outs[4].v.double().view(grid, 2, c).sum(0)
    xd = x.double()
    _check_rel(p[0], xd.sum(0), xd.abs().sum(0), STAT_REL, tag + " sum", "channel sums")
    _check_rel(p[1], (xd * xd).sum(0), (xd * xd).sum(0), STAT_REL, tag + " sum of squares", "channel sums")


def _run_spatial_sum(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    x_ld, n, p, c, scale, out_ld, acc = a[1], a[2], a[3], a[4], a[5], a[8], a[9]
    g = _rng(row)
    x = _bf16(_randn(g, n * p, c))
    splits = _lib.lib().b200seg_spatial_sum_splits(p)
    xd = x.double().view(n, p, c)
    r, A = scale * xd.sum(1), abs(scale) * xd.abs().sum(1)
    old = _bf16(_randn(g, n, c)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    ins = {0: Buf(n * p, c, x_ld, torch.bfloat16, x), 6: torch.empty(n * splits * c, dtype=torch.float32, device="cuda")}
    outs, _ = _twice(name, a, ins, lambda: ({7: Buf(n, c, out_ld, torch.bfloat16, old)}, {}))
    outs[7].check(tag)
    _check_bf16(outs[7].v, r, A, tag, "spatial_sum", rel=STAT_REL)


def _run_broadcast_pixels(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    v_ld, n, p, c, scale, out_ld, acc = a[1], a[2], a[3], a[4], a[5], a[7], a[8]
    g = _rng(row)
    v = _bf16(_randn(g, n, c))
    r = (scale * v.double()).repeat_interleave(p, 0)
    A = r.abs()
    old = _bf16(_randn(g, n * p, c)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    outs, _ = _twice(name, a, {0: Buf(n, c, v_ld, torch.bfloat16, v)},
                     lambda: ({6: Buf(n * p, c, out_ld, torch.bfloat16, old)}, {}))
    outs[6].check(tag)
    _check_bf16(outs[6].v, r, A, tag, "broadcast_pixels", exact=scale == 1.0 and not acc)


def _run_transpose_pad(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    fp32, R, C, ld, rpad = a[1], a[2], a[3], a[4], a[6]
    g = _rng(row)
    src = _randn(g, R, C).to(torch.float32 if fp32 else torch.bfloat16)
    r = torch.zeros((C, rpad), dtype=torch.float64, device="cuda")
    r[:, :R] = src.double().t()
    outs, _ = _twice(name, a, {0: Buf(R, C, ld, src.dtype, src)}, lambda: ({5: Buf(C, rpad, rpad, torch.bfloat16)}, {}))
    outs[5].check(tag)
    _check_bf16(outs[5].v, r, r.abs(), tag, "transpose_pad", exact=True)


def _run_cast_rows(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    src_ld, dst_ld, rows, C, acc = a[1], a[3], a[4], a[5], a[6]
    g = _rng(row)
    src = _f32(_randn(g, rows, C))
    r, A = src.double(), src.double().abs()
    old = _bf16(_randn(g, rows, C)) if acc else None
    if acc:
        r, A = r + old.double(), A + old.double().abs()
    outs, _ = _twice(name, a, {0: Buf(rows, C, src_ld, torch.float32, src)},
                     lambda: ({2: Buf(rows, C, dst_ld, torch.bfloat16, old)}, {}))
    outs[2].check(tag)
    _check_bf16(outs[2].v, r, A, tag, "cast_rows", exact=not acc)


def _run_bias_grad(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ld, rows, C = a[1], a[2], a[3]
    g = _rng(row)
    dy = _bf16(_randn(g, rows, C))
    d0 = _f32(_randn(g, C))
    _outs, extra = _twice(name, a, {0: Buf(rows, C, ld, torch.bfloat16, dy)},
                          lambda: ((lambda db: ({4: db}, {"db": db}))(d0.clone())))
    db = extra["db"].double()
    _check_stat_sums(db, d0.double() + dy.double().sum(0), dy.double().abs().sum(0), tag + " db", db)


def _run_image_prep(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    n, H, W, h, w = a[1], a[2], a[3], a[5], a[6]
    g = _rng(row)
    img = _f32(_randn(g, n, 3, H, W))
    src = img.double().permute(0, 2, 3, 1).reshape(n * H * W, 3)
    r = torch.zeros((n * h * w, 16), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    r[:, :3], A[:, :3] = _resample(src, n, H, W, h, w), _resample(src.abs(), n, H, W, h, w)
    outs, _ = _twice(name, a, {0: img}, lambda: ({4: Buf(n * h * w, 16, 16, torch.bfloat16)}, {}))
    outs[4].check(tag)
    _check_bf16(outs[4].v, r, A, tag, "image_prep")


def _run_resize_to_nchw(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    ld, n, h, w, C, sig, H, W = a[1], a[2], a[3], a[4], a[5], a[6], a[8], a[9]
    g = _rng(row)
    src = _f32(2.0 * _randn(g, n * h * w, C))
    s = torch.sigmoid(src.double()) if sig else src.double()
    r = _nchw4(_resample(s, n, h, w, H, W), n, H, W, C).reshape(-1)
    A = _nchw4(_resample(s.abs(), n, h, w, H, W), n, H, W, C).reshape(-1)
    outs, _ = _twice(name, a, {0: Buf(n * h * w, C, ld, torch.float32, src)},
                     lambda: ({7: Buf(1, n * C * H * W, n * C * H * W, torch.float32)}, {}))
    outs[7].check(tag)
    _check_f32(outs[7].v[0], r, A, tag, "resize fp32")


def _run_resize_nchw(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    planes, h, w, H, W = a[1], a[2], a[3], a[5], a[6]
    g = _rng(row)
    src = _f32(_randn(g, planes, h, w))
    Uy, Ux = _interp(H, h), _interp(W, w)
    r = (Uy @ src.double() @ Ux.t()).reshape(-1)
    A = (Uy @ src.double().abs() @ Ux.t()).reshape(-1)
    outs, _ = _twice(name, a, {0: src}, lambda: ({4: Buf(1, planes * H * W, planes * H * W, torch.float32)}, {}))
    outs[4].check(tag)
    _check_f32(outs[4].v[0], r, A, tag, "resize fp32")


def _run_blend(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    n, c, hw, mode = a[4], a[5], a[6], a[7]
    g = _rng(row)
    al = _f32(torch.sigmoid(_randn(g, n, 1, hw)))
    x, y = _f32(_randn(g, n, c, hw)), _f32(_randn(g, n, c, hw))
    ad, xd, yd = al.double(), x.double(), y.double()
    if mode == 0:
        r, A = ad * xd + (1 - ad) * yd, ad * xd.abs() + (1 - ad) * yd.abs()
    elif mode == 1:
        r, A = xd + (1 - ad) * yd, xd.abs() + (1 - ad) * yd.abs()
    else:
        r, A = ad * xd, ad * xd.abs()
    ins = {0: al, 1: x}
    if a[2] is not None:
        ins[2] = y
    outs, _ = _twice(name, a, ins, lambda: ({3: Buf(1, n * c * hw, n * c * hw, torch.float32)}, {}))
    outs[3].check(tag)
    _check_f32(outs[3].v[0], r.reshape(-1), A.reshape(-1), tag, "blend")


def _run_accum_pred(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    n, c, h, w, flip, acc = a[2], a[3], a[4], a[5], a[6], a[7]
    g = _rng(row)
    pred = _f32(_randn(g, n, c, h, w))
    r = (pred.flip(3) if flip else pred).double().reshape(-1)
    old = _f32(_randn(g, n * c * h * w)) if acc else None
    if acc:
        r = r + old.double()
    outs, _ = _twice(name, a, {0: pred}, lambda: ({1: Buf(1, n * c * h * w, n * c * h * w, torch.float32, old)}, {}))
    outs[1].check(tag)
    bad = int((outs[1].v[0] != r.float()).sum())
    assert bad == 0, "%s: %d outputs differ from round_fp32(reference)" % (tag, bad)


def _run_argmax_hist(row):
    torch, _ = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    n, c, hw, scale = a[1], a[2], a[3], a[4]
    g = _rng(row)
    pred = _f32(3.0 * _randn(g, n, c, hw))
    v = (pred * scale).permute(0, 2, 1).reshape(n * hw, c)        # the kernel's fp32 products
    arg = torch.argmax(v, dim=1)                                    # first maximum
    vd = v.double()
    mp = 1.0 / torch.exp(vd - vd.max(1, keepdim=True).values).sum(1)
    labels = torch.randint(0, c + 2, (n * hw,), generator=g, device="cuda", dtype=torch.int64)
    labels[labels == c + 1] = 255
    ins = {0: pred}
    if a[5] is not None:
        ins[5] = labels
    h0 = torch.randint(0, 1000, (c, c), generator=g, device="cuda", dtype=torch.int64)
    ok = labels < c
    want = h0 + torch.bincount(labels[ok] * c + arg[ok], minlength=c * c).view(c, c)

    def outputs():
        extra = dict(pm=torch.full((n * hw,), -1, dtype=torch.int64, device="cuda"),
                     mp=torch.full((n * hw,), float("nan"), dtype=torch.float32, device="cuda"))
        outs = {6: extra["pm"], 7: extra["mp"]}
        if a[8] is not None:
            extra["hist"] = h0.clone()
            outs[8] = extra["hist"]
        return outs, extra
    _outs, extra = _twice(name, a, ins, outputs)
    assert torch.equal(extra["pm"], arg), "%s: class map differs" % tag
    _check_f32(extra["mp"], mp, mp, tag + " max probability", "argmax_hist")
    if a[8] is not None:
        assert torch.equal(extra["hist"], want), "%s: histogram differs" % tag


RUNNERS = {"bn_apply": _run_bn_apply, "bn_apply_cells": _run_bn_apply, "bn_finalize": _run_bn_finalize,
           "bn_bwd_cells": _run_bn_bwd, "bn_bwd_apply": _run_bn_bwd, "bn_bwd_reduce": _run_bn_bwd_reduce,
           "bn_bwd_finalize": _run_bn_bwd_finalize, "masked_accum": _run_masked_accum,
           "upsample_adjoint": _run_upsample_adjoint, "fuse_fwd": _run_fuse_fwd,
           "spatial_softmax_fwd": _run_spatial_softmax_fwd, "spatial_softmax_bwd": _run_spatial_softmax_bwd,
           "class_softmax_fwd": _run_class_softmax_fwd, "class_softmax_bwd": _run_class_softmax_bwd,
           "maxpool3x3s2_fwd": _run_maxpool_fwd, "maxpool3x3s2_bwd": _run_maxpool_bwd,
           "channel_stats": _run_channel_stats, "spatial_sum": _run_spatial_sum,
           "broadcast_pixels": _run_broadcast_pixels, "transpose_pad": _run_transpose_pad,
           "cast_rows": _run_cast_rows, "bias_grad": _run_bias_grad, "image_prep": _run_image_prep,
           "resize_to_nchw": _run_resize_to_nchw, "resize_nchw": _run_resize_nchw, "blend": _run_blend,
           "accum_pred": _run_accum_pred, "argmax_hist": _run_argmax_hist}


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_ew_configuration_against_float64(row):
    RUNNERS[row[0]](row)
