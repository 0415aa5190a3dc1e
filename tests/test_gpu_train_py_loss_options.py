"""The UNMODIFIED reference train.py on the overlay with the two loss options: --img_wt_loss --wt_bound 2.0 and
--rmi_loss --ocr_aux_loss_rmi on ocrnet.HRNet_Mscale (nullloader, --test_mode). The losses are finite and do not
increase on the constant batch. Skips when oracle/_ref/ was not built, like test_gpu_train_py.py."""
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
@pytest.mark.parametrize("flags", [["--img_wt_loss", "--wt_bound", "2.0"], ["--rmi_loss", "--ocr_aux_loss_rmi"]])
def test_reference_train_py_with_loss_options(tmp_path, flags):
    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("oracle/_ref/semantic-segmentation is absent (__graft_entry__.build() with a reference checkout)")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, os.path.join(PKG, "shims"), REF])
    env["B200SEG_HRNET_CHECKPOINT"] = ""
    env.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    args = ["--dataset", "nullloader", "--arch", "ocrnet.HRNet_Mscale", "--crop_size", "256,512", "--bs_trn", "1",
            "--bs_val", "1", "--class_uniform_pct", "0", "--num_workers", "0", "--test_mode",
            "--result_dir", str(tmp_path / "logs")] + flags
    out = subprocess.run([sys.executable, os.path.join(REF, "train.py")] + args, cwd=str(tmp_path), env=env,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    losses = [float(m) for m in re.findall(r"train main loss ([0-9.naninf+-e]+)\]", out.stdout)]
    assert len(losses) >= 20, out.stdout[-2000:]
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] <= losses[0] + 1e-3, losses
