"""The UNMODIFIED reference train.py on the overlay with the attention-head ablations on ocrnet.HRNet_Mscale:
--mscale_no3x3 --mscale_dropout together, and --mscale_old_arch. Training and validate() run, the losses are finite,
and the checkpoint logx.save_model wrote is restored by --snapshot (the variant's parameter names) and evaluated. Skips
when oracle/_ref/ was not built, like test_gpu_train_py.py."""
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


def _run(args, cwd):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, os.path.join(PKG, "shims"), REF])
    env["B200SEG_HRNET_CHECKPOINT"] = ""
    env.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    return subprocess.run([sys.executable, os.path.join(REF, "train.py")] + args, cwd=cwd, env=env,
                          capture_output=True, text=True, timeout=900)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("flags", [["--mscale_no3x3", "--mscale_dropout"], ["--mscale_old_arch"]])
def test_reference_train_py_with_attention_head_flags(tmp_path, flags):
    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("oracle/_ref/semantic-segmentation is absent (__graft_entry__.build() with a reference checkout)")
    logs = str(tmp_path / "logs")
    common = ["--dataset", "nullloader", "--arch", "ocrnet.HRNet_Mscale", "--crop_size", "256,512", "--bs_trn", "1",
              "--bs_val", "1", "--class_uniform_pct", "0", "--num_workers", "0", "--test_mode", "--result_dir",
              logs] + flags
    out = _run(common, str(tmp_path))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    losses = [float(m) for m in re.findall(r"train main loss ([0-9.naninf+-e]+)\]", out.stdout)]
    assert len(losses) >= 20, out.stdout[-2000:]
    assert all(math.isfinite(v) for v in losses), losses
    assert "mean_iu" in out.stdout
    ckpts = sorted(f for f in os.listdir(logs) if f.endswith(".pth"))
    assert ckpts, os.listdir(logs)
    out2 = _run(common + ["--snapshot", os.path.join(logs, ckpts[-1]), "--eval", "val"], str(tmp_path))
    assert out2.returncode == 0, out2.stdout[-3000:] + out2.stderr[-3000:]
    assert "mean_iu" in out2.stdout
