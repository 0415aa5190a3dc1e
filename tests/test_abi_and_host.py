"""CPU-side checks: the C-ABI library loads and exports every symbol include/b200seg.h declares, the Python binding
table covers the header, the module reproduces the reference's state_dict naming/registration order, and the
reference-facing factory (network.get_model) returns it. No kernel is launched here."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "b200seg.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200seg_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from b200seg import _lib
    L = _lib.lib()
    assert L.b200seg_abi_version() == 1
    assert b"sm_90a" in L.b200seg_build_info()
    syms = header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(L, s), "libb200seg.so does not export %s" % s
        assert s in _lib.SIGNATURES, "ctypes table lacks %s" % s
    for s in _lib.SIGNATURES:
        assert s in syms, "%s is bound but not declared in include/b200seg.h" % s
    # the test-only kernels live in their own library: the product library does not export them
    T = _lib.test_lib()
    for s in _lib.PROBE_SIGNATURES:
        assert hasattr(T, s) and not hasattr(L, s), s


def test_no_torch_types_in_the_abi():
    src = open(os.path.join(ROOT, "include", "b200seg.h")).read()
    assert "torch" not in src.lower() and "at::" not in src and "#include <cuda" not in src


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "semantic-segmentation_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert "oracle" not in txt.replace("# oracle", ""), "%s references the oracle" % os.path.join(dp, f)


@pytest.mark.parametrize("arch", ["ocrnet.HRNet_Mscale", "ocrnet.HRNet", "basic.HRNet"])
def test_state_dict_names_and_order_match_reference(golden, arch):
    from b200seg.module import B200SegModule
    from oracle import seg_oracle as O
    net = B200SegModule(arch, 19)
    keys = list(net.state_dict().keys())
    assert keys == golden["state_dict_keys_w48"][arch]
    sd = O.synth_state_dict(arch, O.HRNET_W48)
    for k, v in net.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    if arch == "ocrnet.HRNet_Mscale":
        assert [n for n, _ in net.named_parameters()] == golden["param_order_w48"][arch]   # optimizer state order
        assert len(keys) == 1903 and sum(p.numel() for p in net.parameters()) == 72143430


def test_factory_contract_and_cpu_refusal():
    import network
    net = network.get_model("network.ocrnet.HRNet_Mscale", 19, None)
    assert type(net).__name__ == "B200SegModule" and net.arch == "ocrnet.HRNet_Mscale"
    assert network.get_model("network.basic.HRNet", 19, None).arch == "basic.HRNet"
    assert network.get_model("network.mscale.HRNet", 19, None).arch == "mscale.HRNet"      # network/mscale.py:473-475
    assert network.get_model("network.deepv3.DeepV3PlusW38", 19, None).arch == "deepv3.DeepV3PlusW38"
    with pytest.raises((ImportError, ModuleNotFoundError, AttributeError)):
        network.get_model("network.deepv3.DeepV3PlusSRNX50V3PlusD_m1", 19, None)   # other trunks: not provided
    net.train()
    with pytest.raises(RuntimeError, match="CUDA only"):                 # no CPU fallback
        net({"images": torch.zeros(1, 3, 64, 64), "gts": torch.zeros(1, 64, 64, dtype=torch.long)})


def test_conv_planner_rejects_bad_shapes():
    import ctypes
    from b200seg import _lib
    L = _lib.lib()
    d = _lib.ConvDesc()
    d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride, d.pad, d.x_ld, d.y_ld = 1, 32, 32, 48, 48, 3, 1, 1, 48, 48
    d.emit_stats = 1
    assert L.b200seg_conv2d_stats_elems(ctypes.byref(d)) == 264 * 2 * 48
    assert L.b200seg_conv2d_wgrad_ws_bytes(ctypes.byref(d)) > 0
    d.cin = 50                                                          # not a multiple of 8
    assert L.b200seg_conv2d_stats_elems(ctypes.byref(d)) == 0
    d.cin, d.ksize = 48, 5
    assert L.b200seg_conv2d_stats_elems(ctypes.byref(d)) == 0
    assert L.b200seg_conv2d_fwd(ctypes.byref(d), None, None, None, None, None, None, None) == -1


def test_deepv3_parameter_spec_matches_reference_order():
    """SURVEY §8(f) f2 groundwork: the parameter table of deepv3.DeepV3PlusW38 equals the reference's state_dict
    (names, registration order, 137.1 M parameters) as recorded by tests/golden/make_golden_deepv3.py."""
    from b200seg import arch as A
    g = torch.load(os.path.join(ROOT, "tests", "golden", "reference_deepv3.pt"), map_location="cpu")
    specs = A.deepv3_tensor_specs(19)
    assert [n for n, _s, _k in specs] == g["keys"]
    nparams = 0
    for n, shape, kind in specs:
        if kind in ("conv_w", "bn_w", "bn_b"):
            k = 1
            for d in shape:
                k *= d
            nparams += k
    assert nparams == g["nparams"]


def test_factory_reads_bnfunc_and_backbone_checkpoint(tmp_path):
    """network/_factory.build honours what the reference constructors read from cfg: BNFUNC (config.py:216-225) decides
    SyncBN, HRNET_CHECKPOINT (hrnetv2.py:451-477) is loaded into backbone.* with the reference's key remapping, a missing
    file raises, other class counts are refused loudly."""
    import types
    from network import _factory
    from b200seg.module import B200SegModule
    net = B200SegModule("basic.HRNet", 19)
    ck = {"model.conv1.weight": torch.full((64, 3, 3, 3), 0.5), "bn1.bias": torch.full((64,), 0.25),
          "last_layer.0.weight": torch.zeros(3), "conv2.weight": torch.zeros(1)}       # wrong shape / foreign: dropped
    path = str(tmp_path / "hrnet.pth")
    torch.save(ck, path)
    assert _factory.load_backbone_checkpoint(net, path) == 2
    assert float(net.backbone.conv1.weight.min()) == 0.5 and float(net.backbone.bn1.bias.max()) == 0.25
    assert _factory.load_backbone_checkpoint(net, "") == 0
    with pytest.raises(RuntimeError, match="No such file"):
        _factory.load_backbone_checkpoint(net, str(tmp_path / "missing.pth"))
    with pytest.raises(NotImplementedError, match="19"):
        _factory.build("ocrnet.HRNet", 65, None)
    # a stand-in for the reference's config module
    class SyncBatchNorm:    # noqa
        pass
    ex = types.SimpleNamespace(**{k: types.SimpleNamespace(NUM_MODULES=1, NUM_BLOCKS=b, NUM_CHANNELS=c) for k, b, c in (
        ("STAGE1", [1], [32]), ("STAGE2", [1, 1], [16, 32]), ("STAGE3", [1, 1, 1], [16, 32, 64]),
        ("STAGE4", [1, 1, 1, 1], [16, 32, 64, 128]))})
    cfg = types.SimpleNamespace(
        MODEL=types.SimpleNamespace(OCR_EXTRA=ex, OCR=types.SimpleNamespace(MID_CHANNELS=512, KEY_CHANNELS=256),
                                    SEGATTN_BOT_CH=256, MSCALE_LO_SCALE=0.5, N_SCALES=None, ALIGN_CORNERS=False,
                                    OCR_ASPP=False, MSCALE_OLDARCH=False, MSCALE_INNER_3x3=True, MSCALE_DROPOUT=False,
                                    BNFUNC=SyncBatchNorm, HRNET_CHECKPOINT=""),
        LOSS=types.SimpleNamespace(OCR_ALPHA=0.4, SUPERVISED_MSCALE_WT=0.05, OCR_AUX_RMI=False),
        DATASET=types.SimpleNamespace(IGNORE_LABEL=255))
    mod = types.ModuleType("config")
    mod.cfg = cfg
    import sys
    sys.modules["config"] = mod
    try:
        net = _factory.build("ocrnet.HRNet_Mscale", 19, None)
        assert net.syncbn is True and net.sup_wt == 0.05
        cfg.MODEL.BNFUNC = torch.nn.BatchNorm2d
        assert _factory.build("basic.HRNet", 19, None).syncbn is False
        cfg.MODEL.HRNET_CHECKPOINT = str(tmp_path / "missing.pth")
        with pytest.raises(RuntimeError, match="No such file"):
            _factory.build("basic.HRNet", 19, None)
    finally:
        del sys.modules["config"]
