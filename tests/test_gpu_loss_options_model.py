"""Whole training steps with the two loss options (W16 widths, 64x128 crops as in test_gpu_model.py) against the oracle
run on the GPU with bf16-storage emulation: the loss to 5e-3, every gradient within the oracle's own one-bf16-ulp
noise floor (tests/_parity.py), and CUDA-graph replay equal to the eager step bit for bit.

The batch is test_gpu_model.py's. Unequal class mixes, absent classes and an all-ignored image are covered at op level
(test_gpu_loss_options.py) and against the reference (test_loss_options_host.py): on a batch whose second image holds
five classes, the two-scale OCR step's plain cross-entropy already sits 5e-3 from the bf16-emulating oracle (the
oracle's fp32 and bf16-emulated runs differ by as much on it), so that batch cannot separate a loss error from noise."""
import functools
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

WRN_TEST = dict(structure=[2, 1, 1, 1, 1, 1],
                channels=[(32, 32), (64, 64), (64, 64), (64, 128), (64, 128, 256), (128, 256, 512)])


def _oracle_with_aux_rmi(O):
    """The oracle module with cfg.LOSS.OCR_AUX_RMI on: the two OCR forwards call the auxiliary head with do_rmi=True."""
    ns = types.SimpleNamespace(**{k: getattr(O, k) for k in dir(O) if not k.startswith("__")})
    ns.mscale_two_scale = functools.partial(O.mscale_two_scale, ocr_aux_rmi=True)
    ns.ocrnet_forward = functools.partial(O.ocrnet_forward, ocr_aux_rmi=True)
    return ns


def _product(B200SegModule, O, arch, hcfg, sd0, images, gts, sup, criterion, ocr_aux_rmi, graph):
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    net = B200SegModule(arch, 19, criterion=criterion, hcfg=hcfg, ocfg=ocfg, supervised_mscale_wt=sup,
                        use_cuda_graph=graph, ocr_aux_rmi=ocr_aux_rmi)
    net.load_state_dict(sd0)
    net.wrn_dropout_scale = 0.0
    net = net.cuda().train()
    for _ in range(3 if graph else 1):               # eager warm-up, capture, replay
        net.load_state_dict(sd0)
        net.zero_grad(set_to_none=True)
        loss = net({"images": images.cuda(), "gts": gts.cuda()})
        loss.backward()
    torch.cuda.synchronize()
    return net, loss.detach().clone(), {n: p.grad.detach().clone() for n, p in net.named_parameters()}


def _step(arch, sup, criterion, oracle_crit, ocr_aux_rmi=False):
    import _parity as P
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    deepv3 = arch == "deepv3.DeepV3PlusW38"
    hcfg = WRN_TEST if deepv3 else O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    OO = _oracle_with_aux_rmi(O) if ocr_aux_rmi else O
    sd_ref, loss_ref = P.oracle_train_step(OO, arch, hcfg, sd0, images, gts, sup, crit=oracle_crit)
    net, loss, grads = _product(B200SegModule, O, arch, hcfg, sd0, images, gts, sup, criterion, ocr_aux_rmi, False)
    _, loss_g, grads_g = _product(B200SegModule, O, arch, hcfg, sd0, images, gts, sup, criterion, ocr_aux_rmi, True)
    assert torch.equal(loss, loss_g), (float(loss), float(loss_g))
    differ = [n for n in grads if not torch.equal(grads[n], grads_g[n])]
    assert not differ, differ[:8]
    lv = float(loss)
    assert abs(lv - loss_ref) <= 5e-3 * abs(loss_ref), (lv, loss_ref)
    for name, g in grads.items():
        assert torch.isfinite(g).all(), name
    if deepv3:
        # the batch-normalised 1x1 image-pooling branch makes whole-trunk DeepLab gradients chaotic for two crops
        # (tests/test_gpu_deepv3.py); the head next to the loss is still compared tightly
        c, _ = P.cos_rel(grads["final.6.weight"], sd_ref["final.6.weight"].grad)
        assert c >= 0.99, c
        return net
    floor, run_floor = P.noise_floor(OO, arch, hcfg, sd0, images, gts, sd_ref, sup, crit=oracle_crit)
    skip = lambda k: k.endswith(".0.bias") and (".conv3x3_ocr." in k or ".aux_head.0" in k)
    rep = {k: v for k, v in P.grad_report(net, sd_ref).items() if not skip(k)}
    bad, summary = P.check_against_floor(rep, floor, P.running_report(net, sd_ref), run_floor)
    assert not bad, (summary, bad[:8])
    last = {"basic.HRNet": "seg_head.6.weight", "mscale.HRNet": "cls_head.6.weight"}.get(arch, "ocr.aux_head.2.bias")
    assert rep[last][0] >= 0.99, (last, rep[last])
    return net


@pytest.mark.parametrize("arch,sup", [("ocrnet.HRNet_Mscale", 0.0), ("ocrnet.HRNet_Mscale", 0.05),
                                      ("ocrnet.HRNet", 0.0), ("basic.HRNet", 0.0), ("mscale.HRNet", 0.05),
                                      ("deepv3.DeepV3PlusW38", 0.0)])
def test_train_step_with_image_weighted_ce(arch, sup):
    import _img_wt_oracle as W
    _step(arch, sup, "img_wt:2.5:half", W.criterion_img_wt(2.5, batch_weights=False, fp16=True))


@pytest.mark.parametrize("arch,sup", [("ocrnet.HRNet_Mscale", 0.05), ("ocrnet.HRNet", 0.0)])
def test_train_step_with_rmi_on_the_auxiliary_head(arch, sup):
    from oracle import seg_oracle as O
    net = _step(arch, sup, "rmi", O.criterion_rmi, ocr_aux_rmi=True)
    assert float(net.last_loss_terms[6]) != 0.0
