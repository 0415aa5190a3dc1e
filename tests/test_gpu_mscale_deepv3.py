"""arch 'mscale.DeepV3W38' (MscaleV3Plus over the WideResNet-38 trunk, network/mscale.py:232-336) on the sm_90a kernels
against the GPU-run oracle (tests/_mscale_deepv3_oracle.py, pinned to the reference by tests/test_mscale_deepv3_host.py)
at the reduced WRN widths of tests/test_gpu_deepv3.py, 2 x 128 x 256 crops. Training runs with dropout on: the oracle
replays the module's two Dropout2d mask sets (0.5x pass, then 1.0x pass)."""
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
ARCH = "mscale.DeepV3W38"


def _net(sd0, criterion=None, sup=0.0, graph=False, n_scales=None):
    from b200seg.module import B200SegModule
    net = B200SegModule(ARCH, 19, criterion=criterion, hcfg=WRN_TEST, supervised_mscale_wt=sup, use_cuda_graph=graph,
                        n_scales=n_scales)
    assert list(net.state_dict().keys()) == list(sd0.keys())
    net.load_state_dict(sd0)
    return net.cuda()


def _keep_masks(net, n, seed):
    """The module's mask draw for this seed, as the oracle's 0/1 [n, c] keep masks in Dropout2d call order."""
    from b200seg import arch as A
    torch.manual_seed(seed)
    flat = net._drop_mask(n, torch.device("cuda"))
    out, off = [], 0
    for _pass in range(2):
        for _bp, c, _p in A.wrn_drop_layout(WRN_TEST):
            out.append((flat[off:off + n * c] > 0).float().view(n, c).cpu())
            off += n * c
    assert off == flat.numel()
    return out


@pytest.mark.parametrize("loss_name,sup", [("ce", 0.0), ("rmi", 0.05)])
def test_train_step_matches_oracle(loss_name, sup):
    """Loss, every gradient against the oracle's own one-bf16-ulp noise floor (tests/_parity.py), the two logit heads
    tightly, BatchNorm bookkeeping of the two passes. gamma of aspp.img_conv.1 = 0 as in tests/test_gpu_deepv3.py: the
    batch-normalised 1x1 image-pooling branch of two crops is chaotic."""
    import _parity as P
    import _mscale_deepv3_oracle as MD
    from oracle import seg_oracle as O
    sd0 = MD.synth_state_dict(WRN_TEST, seed=3)
    sd0["aspp.img_conv.1.weight"].zero_()
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    crit, oracle_crit = ("rmi", O.criterion_rmi) if loss_name == "rmi" else (None, O.criterion_ce)
    net = _net(sd0, crit, sup).train()
    masks = _keep_masks(net, 2, 11)
    sd_ref, loss_ref = MD.oracle_train_step(WRN_TEST, sd0, images, gts, masks, sup, oracle_crit)
    floor, run_floor = MD.noise_floor(WRN_TEST, sd0, images, gts, sd_ref, masks, sup, oracle_crit)
    torch.manual_seed(11)
    loss = net({"images": images.cuda(), "gts": gts.cuda()})
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - loss_ref) <= 3e-3 * abs(loss_ref), (float(loss), loss_ref)
    for name, p in net.named_parameters():
        assert (sd_ref[name].grad is None) == (p.grad is None), name
    rep = P.grad_report(net, sd_ref)
    bad, summary = P.check_against_floor(rep, floor, P.running_report(net, sd_ref), run_floor)
    assert not bad, (summary, bad[:8])
    for name in ("final.6.weight", "scale_attn.conv2.weight"):
        assert rep[name][0] >= 0.999, (name, rep[name])
    sd = net.state_dict()
    for bnn in ("backbone.mod2.block1.bn1.0", "backbone.mod6.block1.convs.bn3.0", "aspp.features.2.1", "final.4",
                "scale_attn.bn0", "scale_attn.bn1"):
        assert int(sd[bnn + ".num_batches_tracked"]) == 2, bnn
        assert int(sd_ref[bnn + ".num_batches_tracked"]) == 2, bnn
        ref = sd_ref[bnn + ".running_var"].detach().cpu()
        assert torch.allclose(sd[bnn + ".running_var"].float().cpu(), ref, rtol=3e-2, atol=1e-4), bnn


@pytest.mark.parametrize("n_scales", [None, [0.5, 1.0, 2.0]])
def test_eval_matches_oracle(n_scales):
    """Evaluation (BatchNorm from non-trivial running statistics, folded into the convolution epilogues) against the
    oracle with bf16-storage emulation: every map of the reference's output dict, attention maps included."""
    import _mscale_deepv3_oracle as MD
    from oracle import seg_oracle as O
    sd0 = MD.synth_state_dict(WRN_TEST, seed=3)
    g = torch.Generator().manual_seed(9)
    for k in sd0:
        if k.endswith("running_mean"):
            sd0[k] = 0.1 * torch.randn(sd0[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd0[k] = 0.5 + torch.rand(sd0[k].shape, generator=g)
    # the random attention head produces logits of ~30 (max ~140), where a bf16 rounding flips a sigmoid: scale them
    # to the O(1) range of a trained network so that the maps can be compared like the predictions
    sd0["scale_attn.conv2.weight"] = 0.1 * sd0["scale_attn.conv2.weight"]
    images, _ = O.synth_batch(2, 128, 256, seed=5)
    ctx = O.Ctx(O.clone_sd(sd0), training=False, emulate_bf16=True)
    with torch.no_grad():
        ref = MD.two_scale(ctx, images, wcfg=WRN_TEST) if n_scales is None else MD.nscale(ctx, images, n_scales, WRN_TEST)
    net = _net(sd0, n_scales=n_scales).eval()
    with torch.no_grad():
        out = net({"images": images.cuda()})
    torch.cuda.synchronize()
    assert sorted(out.keys()) == sorted(ref.keys())
    for k, r in ref.items():
        o = out[k].float().cpu()
        assert o.shape == r.shape, (k, o.shape, r.shape)
        if r.shape[1] == 1:
            # attention: compared as logits like the predictions (the maps are sigmoids of them: near a sigmoid's
            # midpoint a logit error of 0.6 % of the range already moves the map by 4 %)
            o, r = torch.logit(o.double(), eps=1e-7), torch.logit(r.double(), eps=1e-7)
        err = (o - r).abs().max().item()
        rng = (r.max() - r.min()).item()
        assert err <= 3e-2 * rng, (k, err, rng)
        if r.shape[1] == 19:
            agree = (o.argmax(1) == r.argmax(1)).float().mean().item()
            assert agree > 0.97, (k, agree)


def test_graph_replay_is_bitwise_eager_and_dropout_masks():
    """Captured training and evaluation replay bit-identically to eager with dropout on (same masks); two eager runs are
    bit-identical; dropout changes the loss; the two passes draw different masks."""
    import _mscale_deepv3_oracle as MD
    from oracle import seg_oracle as O
    sd0 = MD.synth_state_dict(WRN_TEST, seed=3)
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    runs = {}
    for tag, graph in (("eager", False), ("eager2", False), ("graph", True)):
        net = _net(sd0, graph=graph).train()
        out = []
        for it in range(3):
            torch.manual_seed(100 + it)
            net.zero_grad(set_to_none=True)
            l = net({"images": images.cuda(), "gts": gts.cuda()})
            l.backward()
            out.append((float(l), {n: p.grad.clone() for n, p in net.named_parameters()}))
        net.eval()
        with torch.no_grad():
            ev = [net({"images": images.cuda()})["pred"].clone() for _ in range(3)]
        out.append(ev[-1])
        assert all(torch.equal(ev[0], e) for e in ev[1:])
        runs[tag] = out
    for tag in ("eager2", "graph"):
        for (la, ga), (lb, gb) in zip(runs["eager"][:3], runs[tag][:3]):
            assert la == lb, (tag, la, lb)
            differ = [n for n in ga if not torch.equal(ga[n], gb[n])]
            assert not differ, (tag, differ[:8])
        assert torch.equal(runs["eager"][3], runs[tag][3]), tag
    # dropout off: the same seed gives another loss; the two mask sets of one draw differ
    net = _net(sd0).train()
    net.wrn_dropout_scale = 0.0
    torch.manual_seed(100)
    assert float(net({"images": images.cuda(), "gts": gts.cuda()})) != runs["eager"][0][0]
    masks = _keep_masks(_net(sd0), 2, 100)
    assert len(masks) == 4 and all(not torch.equal(masks[i], masks[i + 2]) for i in range(2))
