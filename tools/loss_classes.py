"""Configuration keys of the loss launches of the training step: the multi-scale blend with its cross-entropy, BCE and
image-weighted forms (csrc/mscale_loss.cu), the label counts feeding them, and the RMI terms (csrc/rmi_loss.cu). A key
holds what selects a different code path or grid shape of the entry point's kernels: the ratio of each resampling the
launch does (hi H / hq, mid H / hm, lo hm / hl: 1, 2, 4 or "frac" for a non-integer ratio), the number of heads, one
scale or two, supervision, the criterion, which loss_fwd_kernel instantiation runs, whether RMI terms arrive, the binary16
rounding of the class weights, the grid of each kernel against its own cap, and for RMI the padded last pooling row and
column (H % 4, W % 4) and whether the (Hp - 2)(Wp - 2) positions fill the 48 moment chunks. tests/test_gpu_loss_classes.py
holds one row per key, and tests/test_loss_plans.py checks that the rows cover every key of the traced programs
(tools/trace_step.py LAUNCH_ARGS).

Arguments are the C ABI's, in its order (include/b200seg.h), with pointers as PTR (present) or None (absent) and the loss
descriptor as ("ms", n, h, w, hq, wq, hm, wm, hl, wl, nheads, sup_wt, ignore_index, loss_kind). The grid rules mirror
the launchers: blocks_for (csrc/mscale_loss.cu, capped at 132 x 16 blocks), blocks_for_total (csrc/mscale_common.cuh,
148 x 16) and the label histogram's (blocks, n) grid of at most 528 / n blocks per image."""
PTR = "ptr"
BLOCKS_FOR_CAP = 132 * 16       # B200SEG_MAX_CTAS * 16
BLOCKS_TOTAL_CAP = 148 * 16
RMI_CHUNKS = 48                 # rmi_moments_kernel: position chunks per (image, class)

LOSS_ENTRY_POINTS = frozenset(["count_valid", "label_class_weights", "mscale_mid_fwd", "mscale_loss_fwd",
                               "mscale_loss_fwd_ex", "mscale_hi_bwd", "mscale_lo_bwd", "rmi_pool", "rmi_pool_aux",
                               "rmi_solve_grad"])


def grid(total, threads, cap):
    """'one': a single block; 'grid': one pass of an uncapped grid; 'capped': the grid is capped and its threads loop."""
    blocks = -(-total // threads)
    return "one" if blocks <= 1 else "capped" if blocks > cap else "grid"


def ratio(big, small):
    """Interpolation ratio of one axis: 1, 2, 4 or 'frac'."""
    for r in (1, 2, 4):
        if big == r * small:
            return r
    return "frac"


def ratio2(bh, bw, sh, sw):
    """Ratio of both axes, one value when they agree."""
    ry, rx = ratio(bh, sh), ratio(bw, sw)
    return ry if ry == rx else (ry, rx)


def _desc(d):
    _ms, n, h, w, hq, wq, hm, wm, hl, wl, nheads, sup_wt, ignore_index, loss_kind = d
    return dict(n=n, h=h, w=w, hq=hq, wq=wq, hm=hm, wm=wm, hl=hl, wl=wl, nheads=nheads, sup=sup_wt != 0.0,
                kind=loss_kind)


def _mid(g):
    """Mid ratio H / hm, or None for the one-scale step."""
    return ratio2(g["h"], g["w"], g["hm"], g["wm"]) if g["hm"] > 0 else None


def hist_grid(n, per_image):
    """label_hist_kernel: (blocks, n) with blocks = max(1, min(ceil(per_image / 2048), 528 // n))."""
    want = -(-per_image // 2048)
    return "one" if min(want, 528 // n) <= 1 else "capped" if want > 528 // n else "grid"


def launch_key(name, a):
    """Key of one launch (entry point name without the b200seg_ prefix, its recorded arguments), or None for an entry
    point outside this table."""
    if name not in LOSS_ENTRY_POINTS:
        return None
    if name == "count_valid":
        # labels, total, ignore_index, plus_one, counter_ws, inv_count, stream
        return (name, bool(a[3]), grid(a[1], 256, BLOCKS_FOR_CAP))
    if name == "label_class_weights":
        # labels, n, per_image, upper_bound, round_half, counts, weights, coef, loss_scale, stream
        return (name, bool(a[4]), hist_grid(a[1], a[2]))
    if name == "rmi_solve_grad":
        # n, h, w, pr_pool, la_pool, scale, ws, ws_bytes, G, rmi_terms, dpr, stream
        h, w = a[1], a[2]
        hp, wp = h // 4 + 1, w // 4 + 1
        return (name, h % 4, w % 4, (hp - 2) * (wp - 2) >= RMI_CHUNKS, grid(hp * wp * 20, 256, BLOCKS_TOTAL_CAP))
    g = _desc(a[0])
    n, h, w = g["n"], g["h"], g["w"]
    hi = ratio2(h, w, g["hq"], g["wq"])
    if name == "mscale_mid_fwd":
        # desc, lo_cls, lo_aux, lo_attn, mid, mid_sup, stream
        return (name, ratio2(g["hm"], g["wm"], g["hl"], g["wl"]), g["nheads"], a[5] is not None,
                grid(n * g["hm"] * g["wm"], 256, BLOCKS_FOR_CAP))
    if name in ("mscale_loss_fwd", "mscale_loss_fwd_ex"):
        # plain: desc, labels, inv_count, hi_cls, hi_aux, mid, mid_sup, g_hi, g_lo, g_sup, partial_ws, loss_out,
        #        rmi_dpr, rmi_terms, n_rmi_terms, stream
        # _ex:   desc, labels, inv_count, class_coef, hi_cls, hi_aux, mid, mid_sup, g_hi, g_lo, g_sup, partial_ws,
        #        loss_out, rmi_dpr, rmi_terms, n_rmi_terms, rmi_dpr_aux, rmi_terms_aux, n_rmi_terms_aux, stream
        if name == "mscale_loss_fwd":
            variant, dpr = "plain", a[12]
        else:
            variant, dpr = "wt" if a[3] is not None else "aux_rmi" if a[16] is not None else "plain", a[13]
        return (name, variant, hi, _mid(g), g["nheads"], g["sup"], g["kind"], dpr is not None,
                grid(n * h * w, 128, BLOCKS_FOR_CAP))
    if name == "mscale_hi_bwd":
        # desc, g_hi, d_cls, d_aux, stream
        return (name, hi, g["nheads"], grid(n * g["hq"] * g["wq"] * g["nheads"], 128, BLOCKS_FOR_CAP))
    if name == "mscale_lo_bwd":
        # desc, g_lo, g_sup, lo_cls, lo_aux, lo_attn, mid, dmid_ws, d_cls, d_aux, d_attn, stream
        return (name, _mid(g), ratio2(g["hm"], g["wm"], g["hl"], g["wl"]), g["nheads"], g["sup"],
                grid(n * g["hm"] * g["wm"], 128, BLOCKS_FOR_CAP), grid(n * g["hl"] * g["wl"], 128, BLOCKS_FOR_CAP))
    if name in ("rmi_pool", "rmi_pool_aux"):
        # desc, labels, hi, mid, pr_pool, [la_pool,] stream
        hp, wp = h // 4 + 1, w // 4 + 1
        return (name, hi, _mid(g), h % 4, w % 4, grid(n * hp * wp, 128, BLOCKS_TOTAL_CAP))
    raise KeyError(name)
