"""SURVEY §8(f) row f2: deepv3.DeepV3PlusW38 (WideResNet-38 trunk, ASPP, decoder) on the sm_90a kernels against the
oracle restatement (oracle/seg_oracle.py deepv3_forward, pinned to the reference by tests/test_oracle_golden.py).
A reduced-width WRN keeps the oracle at seconds; the structure (pools, stride, dilations 2/4, bottleneck blocks,
dilated ASPP 12/24/36, image pooling, 304-channel decoder concat) is the full one."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

WRN_TEST = dict(structure=[2, 1, 1, 1, 1, 1],
                channels=[(32, 32), (64, 64), (64, 64), (64, 128), (64, 128, 256), (128, 256, 512)])
ARCH = "deepv3.DeepV3PlusW38"


def _mods():
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    return O, B200SegModule


def _net(B200SegModule, sd0, graph=False):
    net = B200SegModule(ARCH, 19, criterion=None, hcfg=WRN_TEST, use_cuda_graph=graph)
    assert list(net.state_dict().keys()) == list(sd0.keys())
    net.load_state_dict(sd0)
    net.wrn_dropout_scale = 0.0
    return net.cuda()


def test_deepv3_eval_matches_oracle():
    O, B200SegModule = _mods()
    torch.set_num_threads(8)
    sd0 = O.synth_state_dict(ARCH, WRN_TEST, seed=3)
    images, _ = O.synth_batch(2, 128, 256, seed=5)
    with torch.no_grad():
        ref = O.deepv3_forward(O.Ctx(O.clone_sd(sd0), training=False, emulate_bf16=True), images, wcfg=WRN_TEST)["pred"]
    net = _net(B200SegModule, sd0).eval()
    with torch.no_grad():
        out = net({"images": images.cuda()})["pred"].float().cpu()
    torch.cuda.synchronize()
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 3e-2 * scale, (err, scale)
    agree = (out.argmax(1) == ref.argmax(1)).float().mean().item()
    assert agree > 0.97, agree


def _train_step_vs_floor(sd0, images, gts):
    """Product step vs the GPU-run oracle (bf16-storage emulation) and the oracle's own one-bf16-ulp noise floor."""
    import _parity as P
    O, B200SegModule = _mods()
    sd_ref, loss_ref = P.oracle_train_step(O, ARCH, WRN_TEST, sd0, images, gts)
    floor, run_floor = P.noise_floor(O, ARCH, WRN_TEST, sd0, images, gts, sd_ref)
    net = _net(B200SegModule, sd0).train()
    loss = net({"images": images.cuda(), "gts": gts.cuda()})
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - loss_ref) <= 3e-3 * abs(loss_ref), (float(loss), loss_ref)
    for name, p in net.named_parameters():
        assert (sd_ref[name].grad is None) == (p.grad is None), name
    rep = P.grad_report(net, sd_ref)
    run_rep = P.running_report(net, sd_ref)
    bad, summary = P.check_against_floor(rep, floor, run_rep, run_floor)
    return net, sd_ref, rep, floor, bad, summary


def test_deepv3_train_step_matches_oracle():
    """Loss, every gradient, BatchNorm bookkeeping. Whole-network gradients of a batch-statistics-BN + ReLU network are
    compared relative to the oracle's own noise floor (tests/_parity.py). The image-pooling branch of ASPP normalises a
    1x1 map over the BATCH (network/utils.py:196-202): with two crops its backward is ~ eps / (var + eps) * invstd of two
    nearly equal pooled vectors, i.e. chaotic, and it feeds the whole trunk. This case silences that one term (gamma of
    aspp.img_conv.1 = 0, so the branch sends no gradient into the trunk; measured: product 0.52 vs floor 0.52 median
    relative distance on the trunk, 0.14 vs 0.15 on the head); the next test keeps it live with four crops."""
    O, _ = _mods()
    sd0 = O.synth_state_dict(ARCH, WRN_TEST, seed=3)
    sd0["aspp.img_conv.1.weight"].zero_()
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    net, sd_ref, rep, floor, bad, summary = _train_step_vs_floor(sd0, images, gts)
    assert not bad, (summary, bad[:8])
    assert summary["median_rel"] <= 1.15 * summary["median_rel_floor"] + 0.02, summary
    # next to the loss there is no gate-flip noise from above: tight agreement
    for name in ("final.6.weight", "final.4.weight", "final.4.bias"):
        assert rep[name][0] >= 0.999 and rep[name][1] <= 0.05, (name, rep[name])
    # BatchNorm bookkeeping of a pre-activation layer and a conv-epilogue layer
    for bnn in ("backbone.mod5.block1.bn1.0", "backbone.mod6.block1.convs.bn3.0", "aspp.features.2.1", "final.4"):
        rv = net.state_dict()[bnn + ".running_var"].float().cpu()
        ref = sd_ref[bnn + ".running_var"].detach().cpu()
        assert torch.allclose(rv, ref, rtol=3e-2, atol=1e-4), bnn
        assert int(net.state_dict()[bnn + ".num_batches_tracked"]) == 1


def test_deepv3_train_step_image_pooling_live():
    """The same with the image-pooling branch contributing (four crops: its batch normalisation is conditioned)."""
    O, _ = _mods()
    sd0 = O.synth_state_dict(ARCH, WRN_TEST, seed=3)
    images, gts = O.synth_batch(4, 96, 192, seed=6)
    _net_, _sd, rep, floor, bad, summary = _train_step_vs_floor(sd0, images, gts)
    assert not bad, (summary, bad[:8])
    assert rep["aspp.img_conv.0.weight"][1] <= 2.0 * floor["aspp.img_conv.0.weight"][1] + 0.1


def test_deepv3_graph_replay_and_dropout_masks():
    """Captured step replays bit-identically to eager with dropout on (same masks), and dropout changes the loss."""
    O, B200SegModule = _mods()
    sd0 = O.synth_state_dict(ARCH, WRN_TEST, seed=3)
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    losses = {}
    for graph in (False, True):
        net = _net(B200SegModule, sd0, graph=graph).train()
        net.wrn_dropout_scale = 1.0
        out = []
        for it in range(3):
            torch.manual_seed(100 + it)
            net.zero_grad(set_to_none=True)
            l = net({"images": images.cuda(), "gts": gts.cuda()})
            l.backward()
            out.append((float(l), net.get_parameter("backbone.mod7.block1.convs.conv3.weight").grad.clone()))
        losses[graph] = out
    for (la, ga), (lb, gb) in zip(losses[False], losses[True]):
        assert la == lb and torch.equal(ga, gb)
