"""Boundary proof (SURVEY.md §8b): the UNMODIFIED reference train.py (oracle/_ref/semantic-segmentation/train.py, a
verbatim copy of the reference checkout made by oracle/reference_build.py in __graft_entry__.build()) runs on the
overlay: `import network` resolves to
semantic-segmentation_b200/network, network.get_net / wrap_network_in_dataparallel / optimizer / validate / checkpoint
code of the reference run unchanged (train.py:377-383, 488-509, utils/trnval_utils.py), the loss is finite and does not
increase on the (constant) nullloader batch, and the checkpoint logx.save_model wrote is restored by --snapshot."""
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
    env["B200SEG_HRNET_CHECKPOINT"] = ""          # no ImageNet checkpoint offline: random initialisation
    env.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    out = subprocess.run([sys.executable, os.path.join(REF, "train.py")] + args, cwd=cwd, env=env, capture_output=True,
                         text=True, timeout=900)
    return out


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("arch,crop", [("ocrnet.HRNet_Mscale", "256,512"), ("basic.HRNet", "256,512"),
                                       ("mscale.HRNet", "128,256")])
def test_reference_train_py_runs_unchanged_on_the_overlay(tmp_path, arch, crop):
    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("oracle/_ref/semantic-segmentation is absent (__graft_entry__.build() with a reference checkout)")
    logs = str(tmp_path / "logs")
    common = ["--dataset", "nullloader", "--arch", arch, "--crop_size", crop, "--bs_trn", "1", "--bs_val", "1",
              "--class_uniform_pct", "0", "--num_workers", "0", "--test_mode", "--result_dir", logs]
    out = _run(common, str(tmp_path))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "B200SegModule" in out.stdout or "Model params" in out.stdout
    losses = [float(m) for m in re.findall(r"train main loss ([0-9.naninf+-e]+)\]", out.stdout)]
    assert len(losses) >= 20, out.stdout[-2000:]                      # --test_mode: 2 epochs x 11 iterations
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] <= losses[0] + 1e-3, losses                     # running average on a constant batch: no increase
    assert "mean_iu" in out.stdout                                    # the reference's validate() ran on the eval dict
    ckpts = sorted(f for f in os.listdir(logs) if f.endswith(".pth"))
    assert ckpts, os.listdir(logs)
    # reload through the reference's own restore path (loss/optimizer.py:restore_snapshot) and evaluate
    out2 = _run(common + ["--snapshot", os.path.join(logs, ckpts[-1]), "--eval", "val"], str(tmp_path))
    assert out2.returncode == 0, out2.stdout[-3000:] + out2.stderr[-3000:]
    assert "mean_iu" in out2.stdout
