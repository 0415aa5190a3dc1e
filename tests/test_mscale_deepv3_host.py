"""arch 'mscale.DeepV3W38' (MscaleV3Plus over the WideResNet-38 trunk, network/mscale.py:232-336) on the CPU: the
oracle restatement (tests/_mscale_deepv3_oracle.py) against the unmodified reference
(tests/golden/make_golden_mscale_deepv3.py), the module's parameter table, the overlay factory, and the convolution
FLOPs of the traced training step against the reference module's own count."""
import os
import re
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import seg_oracle as O  # noqa: E402
import _mscale_deepv3_oracle as MD  # noqa: E402

torch.set_num_threads(8)
ARCH = "mscale.DeepV3W38"


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_mscale_deepv3.pt"), map_location="cpu")


def close(a, b, rtol=2e-4, atol=0.0):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-30
    assert err <= rtol * scale + atol, "max err %.3e vs scale %.3e" % (err, scale)


@pytest.mark.parametrize("loss_name,sup", [("ce", 0.0), ("ce", 0.05), ("rmi", 0.05)])
def test_oracle_matches_reference(golden, loss_name, sup):
    g = golden["%s/sup%g" % (loss_name, sup)]
    sd = MD.synth_state_dict(O.WRN38, seed=4)
    assert list(sd.keys()) == golden["state_dict_keys"]
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    images, gts = O.synth_batch(2, 64, 128, seed=6)
    crit = O.criterion_ce if loss_name == "ce" else O.criterion_rmi
    loss = MD.two_scale(O.Ctx(sd, training=True), images, gts, criterion=crit, supervised_mscale_wt=sup)
    loss.backward()
    close(loss.detach(), g["loss"], rtol=1e-5)
    for name, ref in g["grads"].items():
        close(O.sample_like(sd[name].grad), ref, rtol=2e-3 if loss_name == "rmi" else 1e-3)
    close(sd["scale_attn.bn0.running_mean"].detach(), g["running_mean_attn_bn0"], atol=1e-6)
    close(sd["scale_attn.bn0.running_var"].detach(), g["running_var_attn_bn0"])
    close(sd["backbone.mod5.block3.convs.bn2.0.running_var"].detach(), g["running_var_mod5"])
    assert int(sd["scale_attn.bn0.num_batches_tracked"]) == g["nbt_attn_bn0"] == 2
    if loss_name != "ce" or sup:
        return
    # evaluation continues from the state the training step left behind, like the reference run
    sd = {k: v.detach() for k, v in sd.items()}
    ctx = O.Ctx(sd, training=False)
    with torch.no_grad():
        o2 = MD.two_scale(ctx, images)
        o3 = MD.nscale(ctx, images, [0.5, 1.0, 2.0])
    assert sorted(o2.keys()) == golden["eval_two_scale_keys"]
    assert sorted(o3.keys()) == golden["eval_three_scale_keys"]
    for k, ref in golden["eval_two_scale"].items():
        close(O.sample_like(o2[k]), ref)
    for k, ref in golden["eval_three_scale"].items():
        close(O.sample_like(o3[k]), ref)


def test_module_state_dict_matches_reference(golden):
    """Full width: the reference's names, shapes and registration order, and its parameter count."""
    from b200seg.module import B200SegModule
    net = B200SegModule(ARCH, 19)
    sd = net.state_dict()
    assert list(sd.keys()) == golden["state_dict_keys"] and len(sd) == 281
    assert [tuple(v.shape) for v in sd.values()] == golden["shapes"]
    assert [n for n, _ in net.named_parameters()] == golden["param_order"]
    assert sum(p.numel() for p in net.parameters()) == golden["nparams"] == 138395456
    assert net.is_deepv3 and net.hcfg["structure"] == [3, 3, 6, 3, 1, 1]


def test_module_initialisation_follows_the_reference():
    """Only `final` gets initialize_weights (kaiming_normal_, std sqrt(2 / fan_in)); ASPP, bot_* and scale_attn keep
    the nn.Conv2d default (kaiming_uniform(a=sqrt(5)), std sqrt(1 / (3 fan_in))), unless INIT_DECODER is set."""
    from b200seg.module import B200SegModule

    def normal(net, name):
        w = net.get_parameter(name).detach()
        fan_in = w[0].numel()
        return abs(float(w.std()) * (fan_in / 2.0) ** 0.5 - 1.0) < 0.1

    torch.manual_seed(0)
    net = B200SegModule(ARCH, 19, hcfg=dict(structure=[1, 1, 1, 1, 1, 1], channels=[(16, 16), (32, 32), (32, 32),
                                                                                     (32, 64), (32, 64, 128),
                                                                                     (64, 128, 256)]))
    assert normal(net, "final.0.weight") and normal(net, "final.3.weight")
    for name in ("aspp.features.1.0.weight", "bot_fine.weight", "bot_aspp.weight", "scale_attn.conv0.weight",
                 "scale_attn.conv1.weight"):
        assert not normal(net, name), name
    net = B200SegModule(ARCH, 19, hcfg=net.hcfg, init_decoder=True)
    for name in ("final.0.weight", "bot_aspp.weight", "scale_attn.conv0.weight", "scale_attn.conv1.weight"):
        assert normal(net, name), name
    assert not normal(net, "aspp.features.1.0.weight")


def test_tensor_specs_follow_segattn_bot_ch():
    from b200seg import arch as A
    ocfg = dict(A.OCR_DEFAULT, segattn_bot_ch=128)
    shapes = {n: s for n, s, _k in A.tensor_specs(ARCH, A.WRN38, ocfg)}
    assert shapes["final.0.weight"] == (128, 304, 3, 3) and shapes["final.6.weight"] == (19, 128, 1, 1)
    assert shapes["scale_attn.conv0.weight"] == (128, 304, 3, 3) and shapes["scale_attn.conv2.weight"] == (1, 128, 1, 1)
    assert A.is_two_scale(ARCH) and A.has_wrn38_trunk(ARCH) and not A.has_ocr(ARCH)


def _cfg():
    model = types.SimpleNamespace(OCR_EXTRA=None, OCR=types.SimpleNamespace(MID_CHANNELS=512, KEY_CHANNELS=256),
                                  SEGATTN_BOT_CH=256, MSCALE_LO_SCALE=0.5, N_SCALES=[0.5, 1.0, 2.0],
                                  ALIGN_CORNERS=False, OCR_ASPP=False, MSCALE_OLDARCH=False, MSCALE_INNER_3x3=True,
                                  MSCALE_DROPOUT=False, BNFUNC=torch.nn.BatchNorm2d, HRNET_CHECKPOINT="")
    return types.SimpleNamespace(MODEL=model, OPTIONS=types.SimpleNamespace(INIT_DECODER=False),
                                 LOSS=types.SimpleNamespace(OCR_ALPHA=0.4, SUPERVISED_MSCALE_WT=0.05, OCR_AUX_RMI=False),
                                 DATASET=types.SimpleNamespace(IGNORE_LABEL=255))


def test_overlay_get_model_reads_the_reference_cfg():
    import network
    from b200seg.module import B200SegModule
    mod = types.ModuleType("config")
    saved = sys.modules.get("config")
    sys.modules["config"] = mod
    try:
        mod.cfg = _cfg()
        net = network.get_model("network.mscale.DeepV3W38", 19, "ce")
        assert isinstance(net, B200SegModule) and net.arch == ARCH
        assert net.n_scales == [0.5, 1.0, 2.0] and net.sup_wt == 0.05 and net.lo_scale == 0.5
        assert net.syncbn is False and net.hcfg["structure"] == [3, 3, 6, 3, 1, 1]
        mod.cfg.MODEL.SEGATTN_BOT_CH = 128
        assert tuple(network.get_model("network.mscale.DeepV3W38", 19, None).get_parameter(
            "scale_attn.conv1.weight").shape) == (128, 128, 3, 3)
        mod.cfg = _cfg()
        mod.cfg.MODEL.ALIGN_CORNERS = True
        with pytest.raises(NotImplementedError, match="align_corners"):
            network.get_model("network.mscale.DeepV3W38", 19, None)
        mod.cfg = _cfg()
        mod.cfg.MODEL.MSCALE_OLDARCH = True
        with pytest.raises(NotImplementedError):
            network.get_model("network.mscale.DeepV3W38", 19, None)
        mod.cfg = _cfg()
        with pytest.raises(NotImplementedError, match="19"):
            network.get_model("network.mscale.DeepV3W38", 65, None)
        with pytest.raises(AttributeError):
            network.get_model("network.mscale.DeepV3W38Fuse", 19, None)
    finally:
        if saved is None:
            sys.modules.pop("config", None)
        else:
            sys.modules["config"] = saved


def test_traced_step_flops_equal_the_reference_convolutions(golden):
    """tools/trace_step.py at 1024x2048: forward of both passes, weight gradients of all but the dead 1.0x attention
    head, data gradients of those minus the two stems. The stem reads the image padded to 16 channels; the data
    gradients of the two logit heads read their output gradient padded to a multiple of 8 channels (19 -> 24, 1 -> 8)."""
    out = subprocess.run([sys.executable, "-O", os.path.join(ROOT, "tools", "trace_step.py"), "--arch", ARCH],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"^(\w+)\s+(\d+)\s+([\d.]+)\s+([\d.]+)\s+([\d.]+)$", line.strip())
        if m:
            rows[m.group(1)] = (int(m.group(2)), float(m.group(3)))
    f = golden["conv_flops_1024x2048"]
    stem = "backbone.mod1.conv1"
    fwd = wgrad = dgrad = 0.0
    for scale in ("0.5", "1.0"):
        for name, v in f[scale].items():
            v = v * 16 / 3 if name == stem else v
            fwd += v
            if scale == "1.0" and name.startswith("scale_attn."):
                continue
            wgrad += v
            if name != stem:
                dgrad += v * {"final.6": 24 / 19, "scale_attn.conv2": 8.0}.get(name, 1.0)
    assert abs(sum(f["1.0"].values()) / 1e12 - 13.00) < 0.01
    assert abs(rows["conv2d_wgrad"][1] - wgrad / 1e12) <= 1e-3, (rows["conv2d_wgrad"], wgrad)
    assert abs(rows["conv2d_dgrad"][1] - dgrad / 1e12) <= 1e-3, (rows["conv2d_dgrad"], dgrad)
    want = fwd + wgrad + dgrad
    assert abs(rows["total"][1] - want / 1e12) <= 2e-3, (rows["total"], want)
    assert rows["maxpool3x3s2_fwd"][0] == 4 and rows["mscale_lo_bwd"][0] == 1
