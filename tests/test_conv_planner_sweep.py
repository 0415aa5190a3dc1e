"""Host-only sweep of the launch planners over every convolution shape of the W48 two-scale step (both passes) and of the
reduced test networks: the forward / data-gradient planner accepts the shape (statistics buffer size query) and the
weight-gradient planner returns a decomposition (workspace and launch-count queries). No kernel is launched."""
import ctypes

import pytest

from b200seg import _lib


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


def test_every_model_convolution_is_accepted_by_the_planners():
    L = _lib.lib()
    for (n, h, w, cin, cout, k, stride) in CASES:
        key = (n, h, w, cin, cout, k, stride)
        d = _desc(n, h, w, cin, cout, k, stride, emit_stats=1)
        assert L.b200seg_conv2d_stats_elems(ctypes.byref(d)) == 264 * 2 * ((cout + 15) // 16 * 16), key
        if cin % 16 == 0:                                   # the stem's 3 -> 16 padded input needs no weight-gradient GEMM
            ws = L.b200seg_conv2d_wgrad_ws_bytes(ctypes.byref(d))
            nl = L.b200seg_conv2d_wgrad_launches(ctypes.byref(d))
            assert ws > 0 and nl in (1, 2), (key, ws, nl)
            assert ws < (8 << 30), (key, ws)               # split-over-pixels slabs stay far below the activation memory
