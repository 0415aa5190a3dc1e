"""Configuration keys of the launches that are not tensor-core convolutions: BatchNorm passes, resampling, pooling,
softmaxes, layout helpers and the evaluation assembly. A key holds what selects a different code path or grid shape of
the entry point's kernels: the channel class of the per-block reductions, which operands sit in wider buffers (ld != C),
the optional operands and modes, and how the element count relates to the launch grid (less than one block, one pass of
an uncapped grid, or a capped grid whose threads loop). tests/test_gpu_ew_classes.py holds one row per key, and
tests/test_ew_plans.py checks that the rows cover every key of the traced programs (tools/trace_step.py LAUNCH_ARGS).

Arguments are the C ABI's, in its order (include/b200seg.h), with pointers as PTR (present) or None (absent), a fuse
descriptor as ("fuse", n, h, w, c, relu, ((h, w, ld, affine) per term)) and a BatchNorm fold as
("fold", c, count, gamma, running, batch). The grid rules mirror the launchers at their default tuning
(csrc/conv_igemm.cu tune(): 8 items per thread and 8 CTAs per SM for the BatchNorm passes, 8 pixel rows per thread and
2 CTAs per SM for the backward reduction, 1 item per thread for the resampling passes)."""
PTR = "ptr"
SMS = 132                 # B200SEG_MAX_CTAS
MAX_GRID = 264            # B200SEG_MAX_GRID

# Entry points outside this table: convolutions (tools/conv_classes.py, tests/test_gpu_conv_classes.py), the losses
# (tools/loss_classes.py, tests/test_gpu_loss_classes.py), the optimizer, gradient bookkeeping and weight packing
# (tests/test_gpu_bookkeeping.py) and the input pipeline (tests/test_gpu_augment.py).
OUT_OF_SCOPE = frozenset([
    "conv2d_fwd", "conv2d_fwd_add", "conv2d_fwd_bn", "conv2d_fwd_affine", "conv2d_dgrad", "conv2d_wgrad",
    "pack_weight", "pack_weights", "grad_fold", "publish_grads", "sgd_step", "accum_f32", "bn_running_update",
    "count_valid", "label_class_weights", "rmi_pool", "rmi_pool_aux", "rmi_solve_grad", "mscale_mid_fwd",
    "mscale_loss_fwd", "mscale_loss_fwd_ex", "mscale_hi_bwd", "mscale_lo_bwd", "aug_resize_crop", "aug_color_normalize",
    "spatial_softmax_blocks", "mscale_loss_blocks",        # host queries (the trace records them like launches)
])


def grid_class(total, per=256, cap=SMS * 8):
    """'block': fewer items than one 256-thread block; 'grid': one pass of an uncapped grid of ceil(total / per)
    blocks; 'capped': the grid is capped and its threads loop."""
    if total < 256:
        return "block"
    return "capped" if -(-total // per) > cap else "grid"


def reduce_rows(c):
    """Pixel rows per block of bn_bwd_reduce_kernel (csrc/bn_kernels.cu reduce_shape) and whether rows x C/8 fills the
    256 threads: ('rows1' | 'rows2' | 'rowsN', full)."""
    groups = c // 8
    rows = max(1, 256 // groups)
    return ("rows1" if rows == 1 else "rows2" if rows == 2 else "rowsN", rows * groups == 256)


def _reduce_grid(npix, c):
    rows = max(1, 256 // (c // 8))
    if npix < rows:
        return "block"
    return "capped" if -(-npix // (rows * 8)) > SMS * 2 else "grid"


def _fold_rows(g):
    """Partial rows per channel of the finalisers (16 slices, four rows per step while 4 x 16 remain): 'few' (< 16:
    some slices idle), 'mid', 'unrolled' (> 48: the four-row loop runs)."""
    return "few" if g < 16 else "mid" if g <= 48 else "unrolled"


def _opt(p, ld, c):
    """Optional operand: 0 absent, 1 present with pitch C, 2 present in a wider buffer."""
    return 0 if p is None else (2 if ld != c else 1)


def _ratio_lanes(big, small):
    r = -(-big // small)
    return 32 if r >= 8 else 16 if r >= 4 else 4 if r >= 2 else 1


def launch_key(name, a):
    """Key of one launch (entry point name without the b200seg_ prefix, its recorded arguments), or None when the
    entry point is OUT_OF_SCOPE."""
    if name in OUT_OF_SCOPE:
        return None
    if name == "bn_finalize":
        # partials, grid, c, cpad, count, gamma, beta, eps, momentum, running_mean, running_var, nbt, scale, shift,
        # mean, invstd, batch_out, sync, stream
        return (name, a[2] % 32 == 0, _fold_rows(a[1]), a[9] is not None, a[16] is not None)
    if name in ("bn_apply", "bn_apply_cells"):
        # y, y_ld, scale|fold, shift, res, res_ld, post_scale, relu, z, z_ld, npix, hw, c, seed, pass, stream
        # (the cells form has no shift argument: every later index is one less)
        o = 1 if name == "bn_apply_cells" else 0
        y_ld, res, res_ld, post, relu, z_ld, npix, c, seed = (a[1], a[4 - o], a[5 - o], a[6 - o], a[7 - o], a[9 - o],
                                                              a[10 - o], a[12 - o], a[13 - o])
        fold = a[2]
        extra = (fold[4], fold[5], npix == 1) if o else ()
        return (name, y_ld != c, _opt(res, res_ld, c), z_ld != c, post is not None, bool(relu), seed is not None,
                grid_class(npix * (c // 8), 2048)) + extra
    if name in ("bn_bwd_cells", "bn_bwd_apply", "bn_bwd_reduce"):
        dz_ld, mask, mask_ld, post, y_ld = a[1], a[2], a[3], a[4], a[6]
        if name == "bn_bwd_reduce":
            # dz, dz_ld, mask, mask_ld, post, y, y_ld, mean, invstd, npix, hw, c, partials, seed, pass, stream
            npix, c, seed = a[9], a[11], a[13]
            return (name,) + reduce_rows(c) + (_reduce_grid(npix, c), dz_ld != c, _opt(mask, mask_ld, c), y_ld != c,
                                               post is not None, seed is not None)
        if name == "bn_bwd_cells":
            # dz, dz_ld, mask, mask_ld, post, y, y_ld, mean, invstd, gamma, dgamma, dbeta, cells, dy, dy_ld, g_out,
            # g_ld, g_acc, npix, hw, c, seed, pass, stream
            dy_ld, g_out, g_ld, g_acc, npix, c, seed = a[14], a[15], a[16], a[17], a[18], a[20], a[21]
            red = reduce_rows(c) + (_reduce_grid(npix, c),)
        else:
            # dz, dz_ld, mask, mask_ld, post, y, y_ld, mean, invstd, gamma, c1, c2, dy, dy_ld, g_out, g_ld, g_acc,
            # npix, hw, c, seed, pass, stream
            dy_ld, g_out, g_ld, g_acc, npix, c, seed = a[13], a[14], a[15], a[16], a[17], a[19], a[20]
            red = ()
        g = 0 if g_out is None else (2 if g_acc else 1) + (2 if g_ld != c else 0)
        return (name,) + red + (dz_ld != c, _opt(mask, mask_ld, c), y_ld != c, dy_ld != c, g, post is not None,
                                seed is not None, grid_class(npix * (c // 8), 2048), npix == 1)
    if name == "bn_bwd_finalize":
        # partials, grid, c, count, dgamma, dbeta, c1, c2, sync, stream
        return (name, a[2] % 32 == 0, _fold_rows(a[1]))
    if name == "masked_accum":
        # src, src_ld, mask, mask_ld, dst, dst_ld, accumulate, npix, c, stream
        return (name, a[1] != a[8], _opt(a[2], a[3], a[8]), a[5] != a[8], bool(a[6]), grid_class(a[7] * (a[8] // 8), 2048))
    if name == "fuse_fwd":
        # desc, out, out_ld, stream
        _f, n, h, w, c, relu, terms = a[0]
        kinds = tuple(sorted(("same" if (th, tw) == (h, w) else "up",
                              ld != c, aff) for th, tw, ld, aff in terms))
        return (name, kinds, a[2] != c, bool(relu), grid_class(n * h * w * (c // 8)))
    if name == "upsample_adjoint":
        # g, g_ld, mask, mask_ld, n, H, W, c, out, out_ld, h, w, accumulate, stream
        n, H, W, c, h, w = a[4], a[5], a[6], a[7], a[10], a[11]
        lanes = _ratio_lanes(H, h)
        return (name, lanes, a[1] != c, _opt(a[2], a[3], c), a[9] != c, bool(a[12]),
                grid_class(n * h * w * (c // 8) * lanes))
    if name == "image_prep":
        # img, n, H, W, out, h, w, stream
        return (name, (a[2], a[3]) == (a[5], a[6]), grid_class(a[1] * a[5] * a[6]))
    if name in ("spatial_softmax_fwd", "spatial_softmax_bwd"):
        # fwd: logits, ld, n, P, K, ws, probs, stat_out, stream; bwd: dprobs, ldd, probs, n, P, K, ws, dlogit, acc, stream
        P = a[3] if name.endswith("fwd") else a[4]
        blocks = -(-P // 256)
        extra = (a[7] is not None,) if name.endswith("fwd") else (bool(a[8]),)
        return (name, "capped" if blocks > MAX_GRID else "one" if blocks == 1 else "grid") + extra
    if name in ("class_softmax_fwd", "class_softmax_bwd"):
        # fwd: x, ld, P, K, scale, sim, stream; bwd: dsim, ld, sim, P, K, scale, ds, stream
        P = a[2] if name.endswith("fwd") else a[3]
        return (name, grid_class(P, 256, MAX_GRID * 4))
    if name == "transpose_pad":
        # src, src_fp32, R, C, ld, dst, rpad, stream
        return (name, bool(a[1]), a[4] != a[3], a[6] > a[2])
    if name == "cast_rows":
        # src, src_ld, dst, dst_ld, rows, C, accumulate, stream
        return (name, a[1] != a[5], a[3] != a[5], bool(a[6]), grid_class(a[4] * a[5]))
    if name == "bias_grad":
        # dy, ld, rows, C, db, stream
        return (name, a[1] != a[3], a[2] < 32)
    if name == "resize_to_nchw":
        # src, ld, n, h, w, C, sigmoid, dst, H, W, stream
        return (name, a[1] != a[5], bool(a[6]), "up" if a[8] >= a[3] else "down", grid_class(a[2] * a[5] * a[8] * a[9],
                                                                                              256, SMS * 16))
    if name == "resize_nchw":
        # src, planes, h, w, dst, H, W, stream
        return (name, "up" if a[5] >= a[2] else "down", grid_class(a[1] * a[5] * a[6], 256, SMS * 16))
    if name == "blend":
        # a, x, y, out, n, c, hw, mode, stream
        return (name, a[7], grid_class(a[4] * a[5] * a[6], 256, SMS * 16))
    if name == "accum_pred":
        # pred, out, n, c, h, w, flip, accumulate, stream
        return (name, bool(a[6]), bool(a[7]), grid_class(a[2] * a[3] * a[4] * a[5], 256, SMS * 16))
    if name == "argmax_hist":
        # pred, n, c, hw, scale, labels, pred_out, maxprob_out, hist, stream
        return (name, a[4] != 1.0, a[8] is not None, grid_class(a[1] * a[3], 256, SMS * 16))
    if name in ("maxpool3x3s2_fwd", "maxpool3x3s2_bwd"):
        # fwd: x, x_ld, n, h, w, c, y, y_ld, stream; bwd: x, x_ld, dy, dy_ld, n, h, w, c, dx, dx_ld, acc, stream
        if name.endswith("fwd"):
            n, h, w, c = a[2:6]
            ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            return (name, a[1] != c, a[7] != c, h % 2, w % 2, grid_class(n * ho * wo * (c // 8)))
        n, h, w, c = a[4:8]
        return (name, a[1] != c, a[3] != c, a[9] != c, bool(a[10]), h % 2, w % 2, grid_class(n * h * w * (c // 8)))
    if name == "channel_stats":
        # x, x_ld, npix, c, partials, stream
        rows = min(32, max(1, 256 // (a[3] // 8)))
        return (name, a[1] != a[3], rows * (a[3] // 8) >= 32, "capped" if -(-a[2] // rows) > SMS else "grid")
    if name == "spatial_sum":
        # x, x_ld, n, p, c, scale, ws, out, out_ld, accumulate, stream
        return (name, a[1] != a[4], a[8] != a[4], bool(a[9]), a[5] == 1.0, "split" if a[3] >= 4096 else "one",
                a[4] % 64 == 0)
    if name == "broadcast_pixels":
        # v, v_ld, n, p, c, scale, out, out_ld, accumulate, stream
        return (name, a[1] != a[4], a[7] != a[4], bool(a[8]), a[5] == 1.0, grid_class(a[2] * a[3] * (a[4] // 8)))
    raise KeyError("no configuration key for entry point %r: key it here or list it in OUT_OF_SCOPE" % name)
