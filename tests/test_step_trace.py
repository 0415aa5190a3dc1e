"""The real step program (b200seg.model / engine / raw) traced on `meta` tensors without a GPU (tools/trace_step.py):
every convolution of the W48 two-scale training step is issued with the right shape, once forward and - except for the
dead 1.0x attention head - twice backward. SURVEY.md §8(d) gives the algorithmic FLOPs this must add up to."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _trace(*args):
    out = subprocess.run([sys.executable, "-O", os.path.join(ROOT, "tools", "trace_step.py")] + list(args),
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"^(\w+)\s+(\d+)\s+([\d.]+)\s+([\d.]+)\s+([\d.]+)$", line.strip())
        if m:
            rows[m.group(1)] = (int(m.group(2)), float(m.group(3)), float(m.group(4)), float(m.group(5)))
    return rows


def test_two_scale_step_flops_and_launch_structure():
    r = _trace("--arch", "ocrnet.HRNet_Mscale")
    total = r["total"]
    assert abs(total[1] - 10.53) <= 0.01 * 10.53 + 0.05, total           # TFLOP per 1024x2048 crop (SURVEY §8d)
    fwd, dgrad, wgrad = r["conv2d_fwd"], r["conv2d_dgrad"], r["conv2d_wgrad"]
    assert fwd[0] == 2 * 322                                             # 322 convolutions per scale pass
    # the 1.0x attention head (3 convolutions) has no backward; the two stem convolutions need no data gradient
    assert wgrad[0] == fwd[0] - 3 and dgrad[0] == fwd[0] - 3 - 2
    assert abs(fwd[1] - 1.25 * 3.0546) <= 0.02                           # 1.25 x one full-resolution _fwd
    assert r["bn_finalize"][0] == 2 * 316 and r["bn_bwd_finalize"][0] == r["bn_bwd_reduce"][0] == r["bn_bwd_apply"][0]
    # default training program with per-GPU statistics: deferred finalisation - a bn_finalize launch
    # remains only in front of the fuse layers (their consumers read scale / shift), no bn_bwd_finalize at all
    c = _trace("--arch", "ocrnet.HRNet_Mscale", "--bn-cells")
    assert c["bn_apply_cells"][0] + c["bn_finalize"][0] == 2 * 316 and "bn_bwd_finalize" not in c
    assert c["bn_bwd_cells"][0] == r["bn_bwd_reduce"][0] and "bn_bwd_reduce" not in c
    assert c["bn_apply_cells"][0] + c.get("bn_apply", (0,))[0] == r["bn_apply"][0]
    assert c["conv2d_fwd_bn"][0] == c["bn_apply_cells"][0]
    assert abs(c["total"][1] - total[1]) < 1e-6
    assert 60.0 < total[2] < 90.0                                        # GB of tensors handed to kernels per crop


def test_single_scale_architectures_trace():
    r = _trace("--arch", "ocrnet.HRNet")
    assert abs(r["total"][1] - 7.77) <= 0.08, r["total"]                 # 3 x 2.5907 TFLOP (SURVEY §8d, cfg2)
    r = _trace("--arch", "basic.HRNet", "--height", "256", "--width", "512")
    assert abs(r["total"][1] - 0.365) <= 0.01, r["total"]                # cfg1


def test_mscale_basic_architecture_traces():
    """arch 'mscale.HRNet' (MscaleBasic, network/mscale.py:450-475): per 1x forward the trunk (678.3 GMAC) plus two
    3x3-3x3-1x1 heads on the 720-channel features (295.3 + 294.7 GMAC) = 2.536 TFLOP; train step = 1.25 x forward +
    2 x (1.25 x forward - the dead 1.0x attention head 0.589 TFLOP)."""
    r = _trace("--arch", "mscale.HRNet")
    fwd1 = 2.0 * (678.3 + 295.3 + 294.7) * 1e-3
    want = 1.25 * fwd1 + 2.0 * (1.25 * fwd1 - 2.0 * 294.7e-3)
    assert abs(r["total"][1] - want) <= 0.01 * want, (r["total"], want)
    assert r["conv2d_wgrad"][0] == r["conv2d_fwd"][0] - 3


def test_deepv3_wrn38_program_traces():
    r = _trace("--arch", "deepv3.DeepV3PlusW38")
    assert abs(r["total"][1] - 34.95) <= 0.35, r["total"]                # 3 x 11.65 TFLOP (SURVEY §8d, cfg4)
    assert r["maxpool3x3s2_fwd"][0] == 2 and r["maxpool3x3s2_bwd"][0] == 2
    assert r["conv2d_fwd"][0] + r.get("conv2d_fwd_bn", (0,))[0] + r["conv2d_fwd_add"][0] == r["conv2d_wgrad"][0]
