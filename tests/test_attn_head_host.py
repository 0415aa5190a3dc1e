"""The attention-head ablations --mscale_no3x3, --mscale_dropout and --mscale_old_arch on the CPU: the oracle
restatement (tests/_attn_head_oracle.py) against the unmodified reference (tests/golden/make_golden_attn_head.py), the
module's W48 parameter tables per variant, the old head's initialisation, the overlay factory's cfg handling, and the
convolution FLOPs of the traced training step against the reference modules' own count."""
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
import _attn_head_oracle as AH  # noqa: E402

torch.set_num_threads(8)
SAMPLE = 1024          # tests/golden/make_golden_attn_head.py records strided samples of this many elements
MASK_SEED = 1234       # ... and runs the dropout variants with AH.seeded_masks(MASK_SEED)
CASES = [(a, v, "ce", 0.0) for a in AH.ARCHS for v in ("no3x3", "dropout", "oldarch", "no3x3_dropout")
         if AH.supported(a, v)] + [("ocrnet.HRNet_Mscale", "no3x3_dropout", "rmi", 0.05)]
TABLES = [(a, v) for a in AH.ARCHS for v in ("default", "no3x3", "dropout", "oldarch") if AH.supported(a, v)]


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_attn_head.pt"), map_location="cpu")


def close(a, b, rtol=2e-4, atol=0.0):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-30
    assert err <= rtol * scale + atol, "max err %.3e vs scale %.3e" % (err, scale)


@pytest.mark.parametrize("arch,variant,loss_name,sup", CASES)
def test_oracle_matches_reference(golden, arch, variant, loss_name, sup):
    g = golden["%s/%s/%s/sup%g" % (arch, variant, loss_name, sup)]
    sd = AH.synth_state_dict(arch, variant)
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    images, gts = O.synth_batch(2, 64, 128, seed=6)
    crit = O.criterion_ce if loss_name == "ce" else O.criterion_rmi
    loss = AH.forward(arch, variant, O.Ctx(sd, training=True), images, gts, AH.seeded_masks(MASK_SEED), crit,
                      sup_wt=sup)
    loss.backward()
    close(loss.detach(), g["loss"], rtol=1e-5)
    assert sorted(g["grads"]) == sorted([k for k in sd if k.startswith("scale_attn.") and "running" not in k
                                         and "num_batches" not in k] + [k for k in g["grads"] if k.startswith("back")])
    for name, ref in g["grads"].items():
        close(O.sample_like(sd[name].grad, SAMPLE), ref, rtol=2e-3 if loss_name == "rmi" else 1e-3)
    bn_last = AH.head_layers(variant)[0][-1][1]
    close(sd[bn_last + ".running_mean"].detach(), g["running_mean_attn_bn_last"], atol=1e-6)
    close(sd[bn_last + ".running_var"].detach(), g["running_var_attn_bn_last"])
    assert int(sd[bn_last + ".num_batches_tracked"]) == g["nbt_attn_bn_last"] == 2
    if "eval" not in g:
        return
    sd = {k: v.detach() for k, v in sd.items()}
    ctx = O.Ctx(sd, training=False)
    with torch.no_grad():
        for key, scales in (("eval", None), ("eval_three_scale", [0.5, 1.0, 2.0])):
            out = AH.forward(arch, variant, ctx, images, scales=scales)
            assert sorted(out) == sorted(g[key])
            for k, ref in g[key].items():
                close(O.sample_like(out[k], SAMPLE), ref)


@pytest.mark.parametrize("arch,variant", TABLES)
def test_module_state_dict_matches_reference(golden, arch, variant):
    """W48 / WRN-38: the reference's names, shapes, registration order and parameter count per variant."""
    from b200seg import arch as A
    from b200seg.module import B200SegModule
    g = golden["w48/%s/%s" % (arch, variant)]
    table = json.loads(zlib.decompress(g["table_zlib"]))
    ocfg = dict(A.OCR_DEFAULT, **AH.ocfg_keys(variant))
    specs = A.tensor_specs(arch, A.WRN38 if A.has_wrn38_trunk(arch) else A.HRNET_W48, ocfg)
    assert [n for n, _s, _k in specs] == table["keys"]
    assert [list(s) for _n, s, _k in specs] == table["shapes"]
    net = B200SegModule(arch, 19, ocfg=ocfg)
    assert list(net.state_dict().keys()) == table["keys"]
    assert [n for n, _ in net.named_parameters()] == table["param_order"]
    assert sum(p.numel() for p in net.parameters()) == g["nparams"]
    zero = all(float(p.detach().abs().max()) == 0.0 for n, p in net.named_parameters()
               if n.startswith("scale_attn.") and p.dim() == 4)
    assert zero == g["attn_conv_zero"] == (variant == "oldarch")
    for n, p in net.named_parameters():
        if n.startswith("scale_attn.") and p.dim() == 1:
            assert float(p.detach().abs().max()) == (1.0 if n.endswith("weight") else 0.0), n


def test_old_head_ignores_the_other_flags():
    from b200seg import arch as A
    old = A.tensor_specs("mscale.HRNet", A.HRNET_W48, dict(A.OCR_DEFAULT, mscale_oldarch=True))
    mixed = A.tensor_specs("mscale.HRNet", A.HRNET_W48, dict(A.OCR_DEFAULT, mscale_oldarch=True,
                                                             mscale_inner_3x3=False, mscale_dropout=True))
    assert old == mixed
    assert A.attn_head_plan(dict(mscale_oldarch=True, mscale_dropout=True))[2] is False


def _cfg(**model):
    m = dict(OCR_EXTRA=None, OCR=types.SimpleNamespace(MID_CHANNELS=512, KEY_CHANNELS=256), SEGATTN_BOT_CH=256,
             ASPP_BOT_CH=256, MSCALE_LO_SCALE=0.5, N_SCALES=None, ALIGN_CORNERS=False, OCR_ASPP=False,
             MSCALE_OLDARCH=False, MSCALE_INNER_3x3=True, MSCALE_DROPOUT=False, BNFUNC=torch.nn.BatchNorm2d,
             HRNET_CHECKPOINT="")
    m.update(model)
    return types.SimpleNamespace(MODEL=types.SimpleNamespace(**m),
                                 OPTIONS=types.SimpleNamespace(INIT_DECODER=False),
                                 LOSS=types.SimpleNamespace(OCR_ALPHA=0.4, SUPERVISED_MSCALE_WT=0.0,
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


@pytest.mark.parametrize("arch", ["ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.HRNet_ASP"])
def test_factory_reads_the_flags(ref_cfg, arch):
    import network
    ref_cfg.cfg = _cfg(MSCALE_INNER_3x3=False, MSCALE_DROPOUT=True)
    net = network.get_model("network." + arch, 19, "ce")
    names = [n for n, _ in net.named_parameters() if n.startswith("scale_attn.")]
    assert names == ["scale_attn.conv0.weight", "scale_attn.bn0.weight", "scale_attn.bn0.bias",
                     "scale_attn.conv2.weight"]
    assert net.ocfg["mscale_dropout"] and not net.ocfg["mscale_inner_3x3"]
    ref_cfg.cfg = _cfg(MSCALE_OLDARCH=True)
    net = network.get_model("network." + arch, 19, "ce")
    assert [n for n, _ in net.named_parameters() if n.startswith("scale_attn.") and n.endswith("weight")] == [
        "scale_attn.0.weight", "scale_attn.1.weight", "scale_attn.3.weight", "scale_attn.4.weight",
        "scale_attn.6.weight"]


@pytest.mark.parametrize("arch", ["ocrnet.HRNet", "basic.HRNet", "basic.HRNet_ASP"])
def test_flags_do_not_change_archs_without_a_head(ref_cfg, arch):
    import network
    ref_cfg.cfg = _cfg()
    base = [(n, tuple(p.shape)) for n, p in network.get_model("network." + arch, 19, "ce").named_parameters()]
    for flags in (dict(MSCALE_INNER_3x3=False, MSCALE_DROPOUT=True), dict(MSCALE_OLDARCH=True)):
        ref_cfg.cfg = _cfg(**flags)
        net = network.get_model("network." + arch, 19, "ce")
        assert [(n, tuple(p.shape)) for n, p in net.named_parameters()] == base


def test_refusals(ref_cfg):
    import network
    ref_cfg.cfg = _cfg(OCR_ASPP=True)
    with pytest.raises(NotImplementedError, match="NameError"):
        network.get_model("network.ocrnet.HRNet_Mscale", 19, None)
    ref_cfg.cfg = _cfg(ALIGN_CORNERS=True, MSCALE_INNER_3x3=False)
    with pytest.raises(NotImplementedError, match="align_corners"):
        network.get_model("network.ocrnet.HRNet_Mscale", 19, None)
    from b200seg.module import B200SegModule
    with pytest.raises(NotImplementedError, match="Dropout2d"):
        B200SegModule("mscale.DeepV3W38", 19, ocfg=dict(mscale_dropout=True))


def _trace(arch, variant):
    out = subprocess.run([sys.executable, "-O", os.path.join(ROOT, "tools", "trace_step.py"), "--arch", arch,
                          "--attn-head", variant], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"^(\w+)\s+(\d+)\s+([\d.]+)\s+([\d.]+)\s+([\d.]+)$", line.strip())
        if m:
            rows[m.group(1)] = (int(m.group(2)), float(m.group(3)))
    return rows


def _expected(flops, stem):
    """Forward + weight-gradient + data-gradient FLOPs of the training step from the reference's forward convolutions:
    both passes forward, weight gradients of all but the dead 1.0x attention head, data gradients of those minus the
    stem. The stem reads the image padded to 16 channels, the attention logit's data gradient an 8-channel padded
    output gradient."""
    tot = 0.0
    for scale, fl in flops.items():
        for name, v in fl.items():
            v = v * 16 / 3 if name == stem else v
            tot += v
            if scale == "1.0" and name.startswith("scale_attn."):
                continue
            tot += v
            if name != stem:
                tot += v * (8.0 if name in ("scale_attn.conv2", "scale_attn.6") else 1.0)
    return tot


@pytest.mark.parametrize("arch,variant", [(a, v) for a, v in TABLES if v != "default"])
def test_traced_step_flops_follow_the_reference_head(golden, arch, variant):
    """tools/trace_step.py at 1024x2048: the traced step of the variant differs from the default's by what the
    reference modules' convolutions differ by (the rest of the step is the same program). Under no3x3 the reference
    forward differs by exactly the conv1 FLOPs of both passes; dropout and the old head change no convolution."""
    stem = "backbone.mod1.conv1" if arch == "mscale.DeepV3W38" else "backbone.conv1"
    f = golden["conv_flops_1024x2048/%s/%s" % (arch, variant)]
    d = golden["conv_flops_1024x2048/%s/default" % arch]
    total = lambda x: sum(sum(v.values()) for v in x.values())  # noqa: E731
    if variant == "no3x3":
        assert total(d) - total(f) == d["1.0"]["scale_attn.conv1"] + d["0.5"]["scale_attn.conv1"]
        assert d["1.0"]["scale_attn.conv1"] == 2 * 256 * 512 * 256 * 256 * 9 * (4 if arch == "mscale.DeepV3W38" else 1)
    else:
        assert total(d) == total(f)
    delta = (_expected(d, stem) - _expected(f, stem)) / 1e12
    traced = _trace(arch, "default")["total"][1] - _trace(arch, variant)["total"][1]
    assert abs(traced - delta) <= 2e-3, (traced, delta)



def test_deepv3_factory_reads_no3x3_and_refuses_the_other_flags(ref_cfg):
    """mscale.DeepV3W38 takes --mscale_no3x3 through the overlay factory; --mscale_old_arch and --mscale_dropout (a
    Dropout2d in the reference on this arch) are refused."""
    import network
    ref_cfg.cfg = _cfg(MSCALE_INNER_3x3=False)
    net = network.get_model("network.mscale.DeepV3W38", 19, "ce")
    assert [n for n, _ in net.named_parameters() if n.startswith("scale_attn.")] == [
        "scale_attn.conv0.weight", "scale_attn.bn0.weight", "scale_attn.bn0.bias", "scale_attn.conv2.weight"]
    assert tuple(net.get_parameter("scale_attn.conv0.weight").shape) == (256, 304, 3, 3)
    ref_cfg.cfg = _cfg(MSCALE_OLDARCH=True)
    with pytest.raises(NotImplementedError, match="MSCALE_OLDARCH"):
        network.get_model("network.mscale.DeepV3W38", 19, None)
    ref_cfg.cfg = _cfg(MSCALE_DROPOUT=True)
    with pytest.raises(NotImplementedError, match="Dropout2d"):
        network.get_model("network.mscale.DeepV3W38", 19, None)
