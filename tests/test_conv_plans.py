"""Host-only sweep of the convolution launch planners (b200seg_conv2d_plan_info, b200seg_conv2d_wgrad_plan_info) over
every convolution shape of the W48 two-scale step (both passes) and of the reduced test networks: shared memory within the
per-SM limits for the chosen occupancy, accumulators that fit the register budget of that occupancy, rings deep enough to
pipeline, grids within the slot count. Also checks that the plan query reports the kernel every traced launch runs, and
that the GPU configuration table of tests/test_gpu_conv_classes.py still reaches its configurations and covers every
configuration the traced programs launch: the training step of every architecture, its attention-head variants, with
and without deferred BatchNorm cells, and the evaluation forwards."""
import ctypes
import functools
import json
import os
import re
import subprocess
import sys

import pytest

from b200seg import _lib, arch as A
import _attn_head_oracle as AH
import test_gpu_conv_classes as classes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

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
    out = (ctypes.c_int32 * 13)()
    seen = set()
    for (n, h, w, cin, cout, k, stride) in CASES:
        if which == 1 and (stride != 1 or cin == 16):
            continue
        d = _desc(n, h, w, cin, cout, k, stride, emit_stats=1 if which == 0 else 0)
        rc = L.b200seg_conv2d_plan_info(ctypes.byref(d), which | _lib.PLAN_WINDOW, out)
        assert rc == 0, (n, h, w, cin, cout, k, stride, rc)
        kern, bn, nt, grid, smem, depth, occ, acc_regs, resident, bslots, kc, tiles, window = list(out)
        key = (n, h, w, cin, cout, k, stride)
        seen.add((kern, occ))
        assert occ in (1, 2) and 1 <= grid <= 132 * occ, key
        # fp32 accumulators per consumer thread: 64 rows x BN columns over 128 threads; two CTAs per SM hold <= 64 each
        assert acc_regs == bn // 2 and occ * acc_regs <= 128, (key, acc_regs, bn)
        assert smem <= CTA_SMEM and occ * (smem + 1024) <= SM_SMEM, (key, smem, occ)
        if occ == 1:
            assert 2 * (smem + 1024) > SM_SMEM, (key, smem)      # a second CTA can never slip in next to a full-SM one
        assert bn % 16 == 0 and bn <= 256 and nt * bn >= (cout if which == 0 else cin), key
        assert kc in (16, 32, 64) and tiles % nt == 0 and grid <= tiles, key
        assert window == 0 or (kern == 0 and which == 0 and grid % nt == 0), key
        if kern == 1:
            assert depth >= 2 and (resident == 1 or bslots >= 2), key
            assert not (occ == 2 and resident == 0 and bslots < 4), key
        else:
            assert depth >= (3 if occ == 2 else 2), key
    assert (1, 2) in seen and (1, 1) in seen      # both the co-resident and the full-SM configuration are exercised


@pytest.mark.parametrize("reserve", [0, classes.SYNCBN_RESERVE])
def test_every_model_weight_gradient_has_a_valid_plan(reserve):
    L = _lib.lib()
    out = (ctypes.c_int32 * 10)()
    seen = set()
    with classes.smem_reserve(reserve):
        for (n, h, w, cin, cout, k, stride) in CASES:
            key = (n, h, w, cin, cout, k, stride)
            d = _desc(n, h, w, cin, cout, k, stride)
            assert L.b200seg_conv2d_wgrad_plan_info(ctypes.byref(d), out) == 0, key
            ntile, n_tiles, tpg, groups, splits, m_tiles, units, grid, b_slots, smem = list(out)
            seen.add((ntile, splits == 1))
            assert ntile in (64, 128, 256) and (n_tiles - 1) * ntile < cin <= n_tiles * ntile, key
            assert tpg * min(cin, ntile) <= 256 and groups * tpg >= k * k > (groups - 1) * tpg, key
            assert m_tiles == (cout + 127) // 128 and units == m_tiles * n_tiles * groups * splits, key
            assert 1 <= grid <= 132 and grid == min(units, 132), key
            assert 2 <= b_slots <= 6 and smem <= CTA_SMEM - reserve, (key, smem)
            ws = L.b200seg_conv2d_wgrad_ws_bytes(ctypes.byref(d))
            assert L.b200seg_conv2d_wgrad_launches(ctypes.byref(d)) == (1 if splits == 1 else 2), key
            assert (ws == 16) == (splits == 1), key
    assert {(64, True), (64, False), (128, True), (128, False), (256, False)} <= seen


def test_conv_classes_table_plans_to_its_declared_keys():
    wrong = []
    for case in classes.CASES:
        entry, shape, reserve, key = case
        with classes.smem_reserve(reserve):
            got = classes.case_keys(entry, shape)[0]
        if got != key:
            wrong.append("%s declares %s, plans to %s" % (classes._case_id(case), key, got))
    assert not wrong, "\n".join(wrong)


def _programs():
    """tools/trace_step.py arguments of every program whose convolutions the table must cover: the training step of
    every architecture with and without deferred BatchNorm cells, the attention-head variants of the multi-scale
    architectures, and the evaluation forwards (0.5x, 1.0x, 2.0x) of all of these."""
    progs = []
    for arch in A.ARCHS:
        heads = ["default"] + [v for v in ("no3x3", "dropout", "oldarch", "no3x3_dropout")
                               if arch in AH.ARCHS and AH.supported(arch, v)]
        for head in heads:
            base = ["--arch", arch, "--attn-head", head]
            progs += [base, base + ["--bn-cells"], base + ["--eval"]]
    return progs


_TRACE = """import json, sys
sys.path.insert(0, %r)
import conv_classes
launches = conv_classes.load_trace(sys.argv[1:], descriptors=True)
print(json.dumps(sorted(set((kern, kind, desc) for kern, kind, _d, _f, _b, desc in launches))))
""" % os.path.join(ROOT, "tools")


@functools.lru_cache(maxsize=None)
def _step_convolutions():
    """{(kernel, entry, (n, h, w, cin, cout, k, stride, dilation), emit_stats, out_fp32, has_bias)} of every
    tensor-core launch of every program of _programs() (tools/trace_step.py through tools/conv_classes.py::load_trace,
    run with -O as the trace requires, one process per program, as many at once as there are CPUs: about 95 s for the
    60 programs on 8 cores). Computed once per session."""
    progs, running, convs = _programs(), [], set()

    def reap(proc, prog):
        out, err = proc.communicate(timeout=900)
        assert proc.returncode == 0, (prog, err[-2000:])
        for kern, kind, (shape, st, f32, bias) in json.loads(out.strip().splitlines()[-1]):
            convs.add((kern, kind, tuple(shape), st, f32, bias))
    for prog in progs:
        if len(running) >= (os.cpu_count() or 4):
            reap(*running.pop(0))
        running.append((subprocess.Popen([sys.executable, "-O", "-c", _TRACE] + prog, stdout=subprocess.PIPE,
                                         stderr=subprocess.PIPE, text=True), prog))
    while running:
        reap(*running.pop(0))
    return frozenset(convs)


def test_plan_query_reports_the_kernel_every_traced_launch_runs():
    """The kernel b200seg_conv2d_plan_info reports is the one the launch entry points run (conv_igemm.cu
    halo_eligible; tools/conv_classes.py mirrors the rule): every dilated 3x3 of the traced programs plans as the
    per-tap kernel, like every launch the trace attributes to it."""
    L = _lib.lib()
    out = (ctypes.c_int32 * 13)()
    out[12] = -7          # sentinel: without PLAN_WINDOW the query fills the 12 entries older callers allocate
    convs = _step_convolutions()
    dilated = 0
    for kern, kind, shape, st, f32, bias in sorted(convs):
        if kind == "wgrad" or (kind == "dgrad" and shape[6] != 1):
            continue
        d = classes._desc(shape, st, f32, bias)
        assert L.b200seg_conv2d_plan_info(ctypes.byref(d), 0 if kind == "fwd" else 1, out) == 0, (kind, shape)
        assert out[12] == -7, "the 12-entry form of the plan query wrote a 13th entry"
        if shape[7] > 1:
            dilated += 1
            assert out[0] == 0, ("dilated 3x3 planned on the halo kernel", kind, shape)
        assert out[0] == (kern == "conv3x3_halo_kernel"), (kern, kind, shape, st, f32)
    assert dilated > 10, dilated


def test_conv_classes_table_covers_every_configuration_of_the_step():
    convs = _step_convolutions()
    assert len(convs) > 150 and {kind for _, kind, *_ in convs} == {"fwd", "dgrad", "wgrad"}
    table = set()
    for entry, shape, reserve, _key in classes.CASES:
        with classes.smem_reserve(reserve):
            table |= {(entry, key) for key in classes.case_keys(entry, shape)[1]}
    # stride-2 data gradients run as sub-lattice launches no plan query reports: EXTRA_CASES holds one per tap geometry
    strided = {classes._taps(shape) for entry, shape, _res, _key in classes.EXTRA_CASES
               if entry == "dgrad" and shape[6] == 2}
    missing = []
    for reserve in (0, classes.SYNCBN_RESERVE):
        with classes.smem_reserve(reserve):
            for _kern, kind, shape, st, f32, bias in sorted(convs):
                if kind == "dgrad" and shape[6] != 1:
                    if classes._taps(shape) not in strided:
                        missing.append("stride-2 data gradient %s (step layer %s)" % (classes._taps(shape), shape))
                        strided.add(classes._taps(shape))
                    continue
                key = (kind, classes.config_key(kind, shape, st, f32, bias))
                if key not in table:
                    missing.append("reserve %d: %s %s (step layer %s, emit_stats %d)" %
                                   (reserve, kind, key[1], shape, st))
                    table.add(key)
    assert not missing, "configurations of the step without a case in tests/test_gpu_conv_classes.py:\n" + \
        "\n".join(missing)
