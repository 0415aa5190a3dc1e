"""archs 'basic.HRNet_ASP' and 'mscale.HRNet_ASP' (the ASPP models over the HRNet trunk, network/basic.py:67-111,
network/mscale.py:479-515) on the CPU: the oracle restatement (tests/_hrnet_asp_oracle.py) against the unmodified
reference (tests/golden/make_golden_hrnet_asp.py), the module's parameter table and initialisation, the overlay
factories, and the convolution FLOPs of the traced training step against the reference modules' own count."""
import json
import os
import re
import subprocess
import sys
import types
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import seg_oracle as O  # noqa: E402
import _hrnet_asp_oracle as HA  # noqa: E402

torch.set_num_threads(8)
SAMPLE = 1024         # tests/golden/make_golden_hrnet_asp.py records strided samples of this many elements
RUNS = [("basic.HRNet_ASP", "ce", 0.0), ("mscale.HRNet_ASP", "ce", 0.0), ("mscale.HRNet_ASP", "ce", 0.05),
        ("mscale.HRNet_ASP", "rmi", 0.05)]


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_hrnet_asp.pt"), map_location="cpu")


def close(a, b, rtol=2e-4, atol=0.0):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-30
    assert err <= rtol * scale + atol, "max err %.3e vs scale %.3e" % (err, scale)


@pytest.mark.parametrize("arch,loss_name,sup", RUNS)
def test_oracle_matches_reference(golden, arch, loss_name, sup):
    g = golden["%s/%s/sup%g" % (arch, loss_name, sup)]
    sd = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=4)
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    images, gts = O.synth_batch(2, 64, 128, seed=6)
    crit = O.criterion_ce if loss_name == "ce" else O.criterion_rmi
    loss = HA.forward(O.Ctx(sd, training=True), arch, images, gts, crit, supervised_mscale_wt=sup)
    loss.backward()
    close(loss.detach(), g["loss"], rtol=1e-5)
    for name, ref in g["grads"].items():
        close(O.sample_like(sd[name].grad, SAMPLE), ref, rtol=2e-3 if loss_name == "rmi" else 1e-3)
    close(sd["aspp.img_conv.1.running_var"].detach(), g["running_var_img_bn"])
    close(sd["aspp.features.3.1.running_mean"].detach(), g["running_mean_d36_bn"], atol=1e-6)
    close(sd["final.4.running_var"].detach(), g["running_var_final_bn"])
    passes = 2 if arch == "mscale.HRNet_ASP" else 1
    assert int(sd["final.1.num_batches_tracked"]) == g["nbt_final_bn"] == passes
    if arch == "mscale.HRNet_ASP":
        # the 1.0x pass's attention head runs forward only, but its BatchNorms count and update like the 0.5x pass's
        close(sd["scale_attn.bn0.running_mean"].detach(), g["running_mean_attn_bn0"], atol=1e-6)
        close(sd["scale_attn.bn1.running_var"].detach(), g["running_var_attn_bn1"])
        assert int(sd["scale_attn.bn0.num_batches_tracked"]) == g["nbt_attn_bn0"] == 2
    if loss_name != "ce" or sup:
        return
    # evaluation continues from the state the training step left behind, like the reference run
    sd = {k: v.detach() for k, v in sd.items()}
    ctx = O.Ctx(sd, training=False)
    with torch.no_grad():
        o2 = HA.forward(ctx, arch, images)
        assert sorted(o2.keys()) == g["eval_keys"]
        for k, ref in g["eval"].items():
            close(O.sample_like(o2[k], SAMPLE), ref)
        if arch == "mscale.HRNet_ASP":
            o3 = HA.nscale(ctx, images, [0.5, 1.0, 2.0])
            assert sorted(o3.keys()) == g["eval_three_scale_keys"]
            for k, ref in g["eval_three_scale"].items():
                close(O.sample_like(o3[k], SAMPLE), ref)


@pytest.mark.parametrize("arch", HA.ARCHS)
@pytest.mark.parametrize("red", [256, 128])
def test_module_state_dict_matches_reference(golden, arch, red):
    """W48: the reference's names, shapes and registration order, and its parameter count, at the default
    ASPP_BOT_CH and at 128."""
    from b200seg import arch as A
    from b200seg.module import B200SegModule
    g = golden["w48/%s/aspp%d" % (arch, red)]
    table = json.loads(zlib.decompress(g["table_zlib"]))
    net = B200SegModule(arch, 19, ocfg=dict(A.OCR_DEFAULT, aspp_bot_ch=red))
    sd = net.state_dict()
    assert list(sd.keys()) == table["keys"] and len(sd) == (1887 if arch == "mscale.HRNet_ASP" else 1874)
    assert [list(v.shape) for v in sd.values()] == table["shapes"]
    assert [n for n, _ in net.named_parameters()] == table["param_order"]
    assert sum(p.numel() for p in net.parameters()) == g["nparams"]
    assert not net.is_deepv3 and net.hcfg == A.HRNET_W48
    assert A.is_two_scale(arch) == (arch == "mscale.HRNet_ASP") and not A.has_wrn38_trunk(arch)
    assert A.has_hrnet_aspp(arch) and not A.has_ocr(arch)


def _normal(net, name):
    """kaiming_normal_ (std sqrt(2 / fan_in)) rather than the nn.Conv2d default (std sqrt(1 / (3 fan_in)))."""
    w = net.get_parameter(name).detach()
    return abs(float(w.std()) * (w[0].numel() / 2.0) ** 0.5 - 1.0) < 0.1


def test_module_initialisation_follows_the_reference():
    """basic: initialize_weights(final, bot_aspp, aspp); mscale: initialize_weights(final) only, so aspp, bot_aspp and
    scale_attn keep the nn.Conv2d default. The trunk is N(0, 1e-3) in both (network/hrnetv2.py:451-461)."""
    from b200seg.module import B200SegModule
    torch.manual_seed(0)
    net = B200SegModule("basic.HRNet_ASP", 19, hcfg=O.HRNET_W16_TEST)
    for name in ("final.0.weight", "final.3.weight", "final.6.weight", "bot_aspp.weight", "aspp.features.0.0.weight",
                 "aspp.features.2.0.weight", "aspp.img_conv.0.weight"):
        assert _normal(net, name), name
    assert abs(float(net.get_parameter("backbone.stage4.0.branches.3.0.conv1.weight").detach().std()) - 1e-3) < 1e-4
    net = B200SegModule("mscale.HRNet_ASP", 19, hcfg=O.HRNET_W16_TEST)
    for name in ("final.0.weight", "final.3.weight"):
        assert _normal(net, name), name
    for name in ("aspp.features.0.0.weight", "aspp.features.2.0.weight", "aspp.img_conv.0.weight", "bot_aspp.weight",
                 "scale_attn.conv0.weight", "scale_attn.conv1.weight"):
        assert not _normal(net, name), name
    assert abs(float(net.get_parameter("backbone.stage4.0.branches.3.0.conv1.weight").detach().std()) - 1e-3) < 1e-4
    assert float(net.get_parameter("final.1.weight").min()) == 1.0 == float(net.get_parameter("final.1.weight").max())


def _cfg(**model):
    m = dict(OCR_EXTRA=None, OCR=types.SimpleNamespace(MID_CHANNELS=512, KEY_CHANNELS=256), SEGATTN_BOT_CH=256,
             ASPP_BOT_CH=256, MSCALE_LO_SCALE=0.5, N_SCALES=[0.5, 1.0, 2.0], ALIGN_CORNERS=False, OCR_ASPP=False,
             MSCALE_OLDARCH=False, MSCALE_INNER_3x3=True, MSCALE_DROPOUT=False, BNFUNC=torch.nn.BatchNorm2d,
             HRNET_CHECKPOINT="")
    m.update(model)
    return types.SimpleNamespace(MODEL=types.SimpleNamespace(**m),
                                 OPTIONS=types.SimpleNamespace(INIT_DECODER=False),
                                 LOSS=types.SimpleNamespace(OCR_ALPHA=0.4, SUPERVISED_MSCALE_WT=0.05,
                                                            OCR_AUX_RMI=False),
                                 DATASET=types.SimpleNamespace(IGNORE_LABEL=255))


@pytest.fixture
def ref_cfg(monkeypatch):
    """A stand-in for the reference's `config` module (OCR_EXTRA None: the narrow test trunk is passed explicitly)."""
    from b200seg import arch as A
    mod = types.ModuleType("config")
    monkeypatch.setitem(sys.modules, "config", mod)
    monkeypatch.setattr(A, "hrnet_cfg_from_reference_cfg", lambda cfg: O.HRNET_W16_TEST)
    return mod


@pytest.mark.parametrize("arch", HA.ARCHS)
def test_overlay_get_model_reads_the_reference_cfg(ref_cfg, arch):
    import network
    from b200seg.module import B200SegModule
    ref_cfg.cfg = _cfg(ASPP_BOT_CH=128, SEGATTN_BOT_CH=64)
    net = network.get_model("network." + arch, 19, "ce")
    assert isinstance(net, B200SegModule) and net.arch == arch
    assert net.ocfg["aspp_bot_ch"] == 128 and net.ocfg["segattn_bot_ch"] == 64
    shapes = {n: tuple(p.shape) for n, p in net.named_parameters()}
    assert shapes["aspp.features.3.0.weight"] == (128, 240, 3, 3) and shapes["bot_aspp.weight"] == (256, 640, 1, 1)
    assert shapes["final.0.weight"] == (64, 256, 3, 3) and shapes["final.6.weight"] == (19, 64, 1, 1)
    if arch == "mscale.HRNet_ASP":
        assert shapes["scale_attn.conv0.weight"] == (64, 256, 3, 3)
        assert net.n_scales == [0.5, 1.0, 2.0] and net.sup_wt == 0.05 and net.lo_scale == 0.5
    else:
        assert "scale_attn.conv0.weight" not in shapes


@pytest.mark.parametrize("arch", HA.ARCHS)
def test_refusals(ref_cfg, arch):
    import network
    ref_cfg.cfg = _cfg()
    with pytest.raises(NotImplementedError, match="19"):
        network.get_model("network." + arch, 65, None)
    for red in (120, 8, 0):
        ref_cfg.cfg = _cfg(ASPP_BOT_CH=red)
        with pytest.raises(NotImplementedError, match="ASPP_BOT_CH"):
            network.get_model("network." + arch, 19, None)
    ref_cfg.cfg = _cfg(ALIGN_CORNERS=True)
    with pytest.raises(NotImplementedError, match="align_corners"):
        network.get_model("network." + arch, 19, None)


def _trace(arch):
    out = subprocess.run([sys.executable, "-O", os.path.join(ROOT, "tools", "trace_step.py"), "--arch", arch],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"^(\w+)\s+(\d+)\s+([\d.]+)\s+([\d.]+)\s+([\d.]+)$", line.strip())
        if m:
            rows[m.group(1)] = (int(m.group(2)), float(m.group(3)))
    return rows


@pytest.mark.parametrize("arch", HA.ARCHS)
def test_traced_step_flops_equal_the_reference_convolutions(golden, arch):
    """tools/trace_step.py at 1024x2048 against the reference modules' convolutions: forward of every pass, weight
    gradients of all but the dead 1.0x attention head, data gradients of those minus the stem. The stem reads the image
    padded to 16 channels; the data gradients of the logit heads read their output gradient padded to a multiple of 8
    channels (19 -> 24, 1 -> 8)."""
    f = golden["conv_flops_1024x2048/" + arch]
    # the three dilated 720 -> 256 ASPP branches of one 1.0x forward: 256 x 512 x 256 x 720 x 9 x 2 FLOP each
    for i in (1, 2, 3):
        assert f["1.0"]["aspp.features.%d.0" % i] == 2 * 256 * 512 * 256 * 720 * 9
    stem = "backbone.conv1"
    fwd = wgrad = dgrad = 0.0
    for scale, flops in f.items():
        for name, v in flops.items():
            v = v * 16 / 3 if name == stem else v
            fwd += v
            if scale == "1.0" and name.startswith("scale_attn."):
                continue
            wgrad += v
            if name != stem:
                dgrad += v * {"final.6": 24 / 19, "scale_attn.conv2": 8.0}.get(name, 1.0)
    rows = _trace(arch)
    assert abs(rows["conv2d_wgrad"][1] - wgrad / 1e12) <= 1e-3, (rows["conv2d_wgrad"], wgrad)
    assert abs(rows["conv2d_dgrad"][1] - dgrad / 1e12) <= 1e-3, (rows["conv2d_dgrad"], dgrad)
    assert abs(rows["total"][1] - (fwd + wgrad + dgrad) / 1e12) <= 2e-3, (rows["total"], fwd + wgrad + dgrad)
