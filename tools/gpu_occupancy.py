"""Prints the CTAs per SM the runtime grants the convolution kernels for the shared-memory sizes the planner picks
(wip/coresident: 2 expected for every Cout tile <= 128). usage: python tools/gpu_occupancy.py"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from b200seg import _lib  # noqa: E402
import test_conv_plans as T  # noqa: E402

torch.zeros(1, device="cuda")
L = _lib.lib()
out = (ctypes.c_int32 * 12)()
seen = set()
for case in T._hrnet_shapes(1024, 2048) + T._hrnet_shapes(512, 1024):
    d = T._desc(*case)
    if L.b200seg_conv2d_plan_info(ctypes.byref(d), 0, out) != 0:
        continue
    kern, bn, nt, grid, smem, depth, occ = list(out)[:7]
    key = (kern, occ, smem)
    if key in seen:
        continue
    seen.add(key)
    got = L.b200seg_debug_occupancy(kern, occ, smem)
    print("%-5s planned occ %d  smem %6d B  BN %3d  -> runtime grants %d CTA/SM %s" %
          ("halo" if kern else "igemm", occ, smem, bn, got, "" if got >= occ else "  <-- LESS THAN PLANNED"))
L.b200seg_debug_occupancy_report()
