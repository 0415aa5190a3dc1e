"""The two loss options on the host: the fp32 restatements (oracle/seg_oracle.py, tests/_img_wt_oracle.py) against
outputs of the UNMODIFIED reference (tests/golden/reference_losses.pt, made by tests/golden/make_golden_losses.py),
and the factory / module accepting
--img_wt_loss and --ocr_aux_loss_rmi while refusing the criteria and options that stay outside the hot path. CPU only."""
import os
import sys
import types

import pytest
import torch

from oracle import seg_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _img_wt_oracle as W  # noqa: E402

torch.set_num_threads(8)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden_losses():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_losses.pt"), map_location="cpu")


def close(a, b, rtol):
    a, b = a.double(), b.double()
    scale = b.abs().max().item() + 1e-30
    err = (a - b).abs().max().item()
    assert err <= rtol * scale, "max err %.3e vs scale %.3e" % (err, scale)


def _oracle_step(arch, crit, sup=0.0, ocr_aux_rmi=False, empty_second=False):
    sd = O.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    ctx = O.Ctx(sd, training=True)
    images, gts = W.synth_batch_mixed(2, 64, 128, seed=5, empty_second=empty_second)
    if arch == "ocrnet.HRNet_Mscale":
        loss = O.mscale_two_scale(ctx, images, gts, criterion=crit, hcfg=O.HRNET_W16_TEST, ocr_aux_rmi=ocr_aux_rmi,
                                  supervised_mscale_wt=sup)
    else:
        loss = O.ocrnet_forward(ctx, images, gts, criterion=crit, hcfg=O.HRNET_W16_TEST, ocr_aux_rmi=ocr_aux_rmi)
    loss.backward()
    return sd, loss.detach()


@pytest.mark.parametrize("ub,bw,sup", [(1.0, 0, 0.0), (1.0, 1, 0.0), (2.5, 0, 0.0), (2.5, 1, 0.0), (2.5, 0, 0.05)])
def test_image_weighted_ce_matches_reference(golden_losses, ub, bw, sup):
    g = golden_losses["ocrnet.HRNet_Mscale/img_wt/ub%g/bw%d/sup%g" % (ub, bw, sup)]
    sd, loss = _oracle_step("ocrnet.HRNet_Mscale", W.criterion_img_wt(ub, bool(bw), fp16=False), sup)
    close(loss, g["loss"], 1e-5)
    for name, ref in g["grads"].items():
        close(O.sample_like(sd[name].grad), ref, 5e-4)


def test_image_weighted_ce_with_an_all_ignored_image(golden_losses):
    """The reference's 0/0 for an image without a valid pixel: the loss is NaN, the gradient is the other image's."""
    g = golden_losses["ocrnet.HRNet_Mscale/img_wt/ub2.5/bw0/sup0/empty_second"]
    assert torch.isnan(g["loss"])
    sd, loss = _oracle_step("ocrnet.HRNet_Mscale", W.criterion_img_wt(2.5, False, fp16=False), empty_second=True)
    assert torch.isnan(loss)
    for name, ref in g["grads"].items():
        assert torch.isfinite(ref).all()
        close(O.sample_like(sd[name].grad), ref, 5e-4)


@pytest.mark.parametrize("arch", ["ocrnet.HRNet_Mscale", "ocrnet.HRNet"])
def test_rmi_on_the_auxiliary_head_matches_reference(golden_losses, arch):
    g = golden_losses["%s/rmi/ocr_aux_rmi" % arch]
    sd, loss = _oracle_step(arch, O.criterion_rmi, ocr_aux_rmi=True)
    close(loss, g["loss"], 1e-5)
    for name, ref in g["grads"].items():
        close(O.sample_like(sd[name].grad), ref, 2e-3)


def test_binary16_rounding_of_the_class_weights():
    """fp16 without --batch_weighting: weights.half(), read back as fp32 (the branch the CPU reference cannot run)."""
    _, gts = W.synth_batch_mixed(2, 64, 128, seed=5)
    w = W.img_wt_class_weights(gts, 2.5)
    logits = torch.randn((2, 19, 64, 128), generator=torch.Generator().manual_seed(1))
    rounded = W.criterion_img_wt(2.5, batch_weights=False, fp16=True)(logits, gts)
    batch = W.criterion_img_wt(2.5, batch_weights=True, fp16=True)(logits, gts)
    plain = W.criterion_img_wt(2.5, batch_weights=False, fp16=False)(logits, gts)
    assert float(batch) == float(plain)
    assert not torch.equal(w.half().float(), w)              # the rounding is visible on these labels
    import torch.nn.functional as F
    want = sum(F.nll_loss(F.log_softmax(logits[i:i + 1], 1), gts[i:i + 1], weight=w.half().float(), ignore_index=255)
               for i in range(2))
    close(rounded, want, 1e-6)


def test_criterion_kinds_and_refusals():
    from b200seg.module import B200SegModule, _criterion_kind, _img_wt_options

    class ImageBasedCrossEntropyLoss2d:    # noqa: the attributes loss/utils.py:73-84 sets
        def __init__(self, ub, bw, fp16, classes=19, ignore=255, norm=False):
            self.num_classes, self.upper_bound, self.batch_weights, self.fp16, self.norm = classes, ub, bw, fp16, norm
            self.nll_loss = types.SimpleNamespace(ignore_index=ignore)

    class ImgWtLossSoftNLL:    # noqa
        pass

    assert _criterion_kind(ImageBasedCrossEntropyLoss2d(2.0, False, True)) == "img_wt"
    assert _img_wt_options(ImageBasedCrossEntropyLoss2d(2.0, False, True)) == (2.0, True)
    assert _img_wt_options(ImageBasedCrossEntropyLoss2d(2.0, True, True)) == (2.0, False)
    assert _img_wt_options(ImageBasedCrossEntropyLoss2d(1.0, False, False)) == (1.0, False)
    assert _criterion_kind("img_wt:2.5:half") == "img_wt" and _img_wt_options("img_wt:2.5:half") == (2.5, True)
    assert _img_wt_options("img_wt") == (1.0, False)
    net = B200SegModule("ocrnet.HRNet", 19, criterion=ImageBasedCrossEntropyLoss2d(2.5, False, True))
    assert net.loss_kind == "img_wt" and net.img_wt == (2.5, True)
    with pytest.raises(NotImplementedError, match="jointwtborder"):
        B200SegModule("ocrnet.HRNet", 19, criterion=ImgWtLossSoftNLL())
    with pytest.raises(NotImplementedError, match="19"):
        B200SegModule("ocrnet.HRNet", 19, criterion=ImageBasedCrossEntropyLoss2d(1.0, False, False, classes=65))
    with pytest.raises(NotImplementedError, match="ignore_index"):
        B200SegModule("ocrnet.HRNet", 19, criterion=ImageBasedCrossEntropyLoss2d(1.0, False, False, ignore=0))
    with pytest.raises(NotImplementedError, match="norm"):
        B200SegModule("ocrnet.HRNet", 19, criterion=ImageBasedCrossEntropyLoss2d(1.0, False, False, norm=True))
    with pytest.raises(NotImplementedError):
        B200SegModule("ocrnet.HRNet", 19, criterion="focal")


def _cfg(**loss):
    ex = types.SimpleNamespace(**{k: types.SimpleNamespace(NUM_MODULES=1, NUM_BLOCKS=b, NUM_CHANNELS=c) for k, b, c in (
        ("STAGE1", [1], [32]), ("STAGE2", [1, 1], [16, 32]), ("STAGE3", [1, 1, 1], [16, 32, 64]),
        ("STAGE4", [1, 1, 1, 1], [16, 32, 64, 128]))})
    model = types.SimpleNamespace(OCR_EXTRA=ex, OCR=types.SimpleNamespace(MID_CHANNELS=512, KEY_CHANNELS=256),
                                  SEGATTN_BOT_CH=256, MSCALE_LO_SCALE=0.5, N_SCALES=None, ALIGN_CORNERS=False,
                                  OCR_ASPP=False, MSCALE_OLDARCH=False, MSCALE_INNER_3x3=True, MSCALE_DROPOUT=False,
                                  BNFUNC=torch.nn.BatchNorm2d, HRNET_CHECKPOINT="")
    args = dict(OCR_ALPHA=0.4, SUPERVISED_MSCALE_WT=0.0, OCR_AUX_RMI=False)
    args.update(loss)
    return types.SimpleNamespace(MODEL=model, LOSS=types.SimpleNamespace(**args),
                                 DATASET=types.SimpleNamespace(IGNORE_LABEL=255))


def test_factory_accepts_both_options_and_keeps_the_other_refusals():
    from network import _factory
    mod = types.ModuleType("config")
    saved = sys.modules.get("config")
    sys.modules["config"] = mod
    try:
        mod.cfg = _cfg(OCR_AUX_RMI=True)
        assert _factory.build("ocrnet.HRNet_Mscale", 19, "rmi").ocr_aux_rmi is True
        assert _factory.build("ocrnet.HRNet", 19, "img_wt:2.0").ocr_aux_rmi is True     # a no-op for this criterion
        mod.cfg = _cfg()
        net = _factory.build("ocrnet.HRNet_Mscale", 19, "img_wt:2.0:half")
        assert net.ocr_aux_rmi is False and net.loss_kind == "img_wt" and net.img_wt == (2.0, True)
        mod.cfg.MODEL.ALIGN_CORNERS = True
        with pytest.raises(NotImplementedError, match="align_corners"):
            _factory.build("ocrnet.HRNet_Mscale", 19, "img_wt")
        mod.cfg = _cfg()
        mod.cfg.MODEL.OCR_ASPP = True
        with pytest.raises(NotImplementedError, match="OCR"):
            _factory.build("ocrnet.HRNet_Mscale", 19, "img_wt")
        mod.cfg = _cfg()
        with pytest.raises(NotImplementedError, match="19"):
            _factory.build("ocrnet.HRNet_Mscale", 65, "img_wt")

        class ImgWtLossSoftNLL:    # noqa
            pass
        with pytest.raises(NotImplementedError, match="jointwtborder"):
            _factory.build("ocrnet.HRNet_Mscale", 19, ImgWtLossSoftNLL())
    finally:
        if saved is None:
            sys.modules.pop("config", None)
        else:
            sys.modules["config"] = saved
