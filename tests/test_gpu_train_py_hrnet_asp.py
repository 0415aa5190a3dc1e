"""The UNMODIFIED reference train.py on the overlay with --arch basic.HRNet_ASP and --arch mscale.HRNet_ASP (the ASPP
models over the full-width HRNet-W48 trunk), the mscale one with three-scale evaluation (--n_scales 0.5,1.0,2.0):
training and validate() run, the losses are finite and do not increase on the constant nullloader batch. Skips when
oracle/_ref/ was not built, like test_gpu_train_py.py."""
import math
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "semantic-segmentation")
PKG = os.path.join(ROOT, "semantic-segmentation_b200")


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("arch,extra", [("basic.HRNet_ASP", []),
                                        ("mscale.HRNet_ASP", ["--n_scales", "0.5,1.0,2.0"])])
def test_reference_train_py_trains_and_validates_hrnet_asp(tmp_path, arch, extra):
    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("oracle/_ref/semantic-segmentation is absent (__graft_entry__.build() with a reference checkout)")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, os.path.join(PKG, "shims"), REF])
    env["B200SEG_HRNET_CHECKPOINT"] = ""
    env.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    args = ["--dataset", "nullloader", "--arch", arch, "--crop_size", "256,512", "--bs_trn", "1", "--bs_val", "1",
            "--class_uniform_pct", "0", "--num_workers", "0", "--test_mode", "--result_dir",
            str(tmp_path / "logs")] + extra
    out = subprocess.run([sys.executable, os.path.join(REF, "train.py")] + args, cwd=str(tmp_path), env=env,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    losses = [float(m) for m in re.findall(r"train main loss ([0-9.naninf+-e]+)\]", out.stdout)]
    assert len(losses) >= 20, out.stdout[-2000:]
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] <= losses[0] + 1e-3, losses
    assert "mean_iu" in out.stdout                                    # the reference's validate() ran
