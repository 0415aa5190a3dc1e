"""Per-layer kernel timings (CUDA-graph replay of 20 launches, CUDA events) for representative HRNet shapes."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
import torch
from b200seg import raw

def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1000.0   # us

shapes = [(16, 8, 48), (256, 512, 48), (128, 256, 48), (128, 256, 96), (64, 128, 96), (64, 128, 192), (32, 64, 192),
          (32, 64, 384), (16, 32, 384), (256, 512, 64), (256, 512, 256), (128, 256, 256)]
print("%-22s %10s %10s %10s %10s %10s %10s" % ("shape", "fwd3x3", "fwd_generic", "dgrad3x3", "wgrad", "bn_apply", "fwd1x1"))
for (h, w, c) in shapes:
    x = torch.randn((1, h, w, c), device="cuda").to(torch.bfloat16)
    dy = torch.randn((1, h, w, c), device="cuda").to(torch.bfloat16)
    wt = torch.randn((c, c, 3, 3), device="cuda") * 0.05
    w_f, w_d = raw.pack_weight(wt)
    w1 = torch.randn((c, c, 1, 1), device="cuda") * 0.05
    w1f, _ = raw.pack_weight(w1)
    dw = torch.zeros_like(wt)
    y = torch.empty_like(x)
    stats = torch.empty(264 * 2 * 1024, device="cuda")
    scale = torch.ones(c, device="cuda"); shift = torch.zeros(c, device="cuda")
    import ctypes
    from b200seg._lib import lib, ptr, stream_ptr
    from b200seg.raw import conv_desc
    L = lib()
    def fwd(kc=0):
        d = conv_desc(1, h, w, c, c, 3, 1, c, c, False, False, True, kc)
        g = ctypes.c_int32(0)
        rc = L.b200seg_conv2d_fwd(ctypes.byref(d), ptr(x), ptr(w_f), None, ptr(y), ptr(stats), ctypes.byref(g), stream_ptr())
        assert rc == 0, rc
    def fwd1():
        d = conv_desc(1, h, w, c, c, 1, 1, c, c, False, False, True, 0)
        g = ctypes.c_int32(0)
        rc = L.b200seg_conv2d_fwd(ctypes.byref(d), ptr(x), ptr(w1f), None, ptr(y), ptr(stats), ctypes.byref(g), stream_ptr())
        assert rc == 0, rc
    dx = torch.empty_like(x)
    def dgrad():
        raw.conv2d_dgrad(dy, w_d, (1, h, w, c), 3, 1, out=dx)
    d_w = conv_desc(1, h, w, c, c, 3, 1, c, c)
    nbytes = L.b200seg_conv2d_wgrad_ws_bytes(ctypes.byref(d_w))
    ws = torch.empty(nbytes // 4, device="cuda")
    def wgrad():
        rc = L.b200seg_conv2d_wgrad(ctypes.byref(d_w), ptr(x), ptr(dy), c, ptr(dw), ptr(ws), nbytes, stream_ptr())
        assert rc == 0, rc
    def bnapply():
        raw.bn_apply(x, scale, shift, None, None, True, out=y)
    r = [timeit(lambda: fwd(0)), timeit(lambda: fwd(64)), timeit(dgrad), timeit(wgrad), timeit(bnapply), timeit(fwd1)]
    print("%-22s %10.1f %10.1f %10.1f %10.1f %10.1f %10.1f" % ("%dx%dx%d" % (h, w, c), *r), flush=True)
