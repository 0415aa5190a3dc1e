"""Host-only sweep of the convolution launch planner (b200seg_conv2d_plan_info) over every convolution shape of the
W48 two-scale step (both passes) and of the reduced test networks: shared memory within the per-SM limits for the chosen
occupancy, accumulators that fit the register budget of that occupancy, rings deep enough to pipeline, grids within the slot count."""
import ctypes

import pytest

from b200seg import _lib

SM_SMEM = 233472          # 228 KB per SM
CTA_SMEM = 232448         # 227 KB opt-in maximum per CTA


def _desc(n, h, w, cin, cout, k, stride=1, emit_stats=1):
    d = _lib.ConvDesc()
    d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride, d.pad = n, h, w, cin, cout, k, stride, (k - 1) // 2
    d.x_ld, d.y_ld, d.emit_stats = cin, (cout + 7) // 8 * 8, emit_stats
    return d


def _hrnet_shapes(H, W, widths=(48, 96, 192, 384), n=1):
    """(h, w, cin, cout, k, stride) of the convolutions of one scale pass at input H x W (network/hrnetv2.py, ocrnet.py)."""
    out = [(H, W, 16, 64, 3, 2), (H // 2, W // 2, 64, 64, 3, 2)]
    q = (H // 4, W // 4)
    for cin in (64, 256):                                    # layer1 bottlenecks
        out += [(q[0], q[1], cin, 64, 1, 1), (q[0], q[1], 64, 64, 3, 1), (q[0], q[1], 64, 256, 1, 1)]
    out.append((q[0], q[1], 64, 256, 1, 1))                  # downsample
    res = [(H // (4 << i), W // (4 << i)) for i in range(4)]
    out.append((q[0], q[1], 256, widths[0], 3, 1))           # transition1
    out.append((q[0], q[1], 256, widths[1], 3, 2))
    for i, c in enumerate(widths):                           # branch BasicBlocks
        out.append((res[i][0], res[i][1], c, c, 3, 1))
    for i in range(4):                                       # fuse layers
        for j in range(4):
            if j > i:
                out.append((res[j][0], res[j][1], widths[j], widths[i], 1, 1))
            elif j < i:
                for k in range(i - j):
                    co = widths[i] if k == i - j - 1 else widths[j]
                    out.append((res[j + k][0], res[j + k][1], widths[j], co, 3, 2))
    for i in range(1, 3):                                    # transitions 2, 3
        out.append((res[i][0], res[i][1], widths[i], widths[i + 1], 3, 2))
    hl = sum(widths)
    out += [(q[0], q[1], hl, 512, 3, 1), (q[0], q[1], hl, hl, 1, 1), (q[0], q[1], 512, 256, 1, 1),
            (q[0], q[1], 256, 256, 1, 1), (q[0], q[1], 256, 512, 1, 1), (q[0], q[1], 1024, 512, 1, 1),
            (q[0], q[1], 512, 256, 3, 1), (q[0], q[1], 256, 256, 3, 1)]
    return [(n,) + s for s in out]


CASES = (_hrnet_shapes(1024, 2048) + _hrnet_shapes(512, 1024) + _hrnet_shapes(64, 128, (16, 32, 64, 128), n=2) +
         _hrnet_shapes(32, 64, (16, 32, 64, 128), n=2))


@pytest.mark.parametrize("which", [0, 1])
def test_every_model_convolution_has_a_valid_plan(which):
    L = _lib.lib()
    out = (ctypes.c_int32 * 10)()
    seen = set()
    for (n, h, w, cin, cout, k, stride) in CASES:
        if which == 1 and (stride != 1 or cin == 16):
            continue
        d = _desc(n, h, w, cin, cout, k, stride, emit_stats=1 if which == 0 else 0)
        rc = L.b200seg_conv2d_plan_info(ctypes.byref(d), which, out)
        assert rc == 0, (n, h, w, cin, cout, k, stride, rc)
        kern, bn, nt, grid, smem, depth, occ, acc_regs, resident, bslots = list(out)
        key = (n, h, w, cin, cout, k, stride)
        seen.add((kern, occ))
        assert occ in (1, 2) and 1 <= grid <= 132 * occ, key
        # fp32 accumulators per consumer thread: 64 rows x BN columns over 128 threads; two CTAs per SM hold <= 64 each
        assert acc_regs == bn // 2 and occ * acc_regs <= 128, (key, acc_regs, bn)
        assert smem <= CTA_SMEM and occ * (smem + 1024) <= SM_SMEM, (key, smem, occ)
        if occ == 1:
            assert 2 * (smem + 1024) > SM_SMEM, (key, smem)      # a second CTA can never slip in next to a full-SM one
        assert bn % 16 == 0 and bn <= 256 and nt * bn >= (cout if which == 0 else cin), key
        if kern == 1:
            assert depth >= 2 and (resident == 1 or bslots >= 2), key
            assert not (occ == 2 and resident == 0 and bslots < 4), key
        else:
            assert depth >= (3 if occ == 2 else 2), key
    assert (1, 2) in seen and (1, 1) in seen      # both the co-resident and the full-SM configuration are exercised
