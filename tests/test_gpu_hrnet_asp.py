"""archs 'basic.HRNet_ASP' and 'mscale.HRNet_ASP' (the ASPP models over the HRNet trunk, network/basic.py:67-111,
network/mscale.py:479-515) on the sm_90a kernels against the GPU-run oracle (tests/_hrnet_asp_oracle.py, pinned to the
reference by tests/test_hrnet_asp_host.py) with the narrow test trunk, 128 x 256 crops. The stride-4 map is 32 x 64, so
the d = 36 branch reads padding only except for its centre tap."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

TRAIN = [("basic.HRNet_ASP", "ce", 0.0), ("mscale.HRNet_ASP", "ce", 0.0), ("mscale.HRNet_ASP", "rmi", 0.05)]


def _net(arch, sd0, criterion=None, sup=0.0, graph=False, n_scales=None):
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    net = B200SegModule(arch, 19, criterion=criterion, hcfg=O.HRNET_W16_TEST, supervised_mscale_wt=sup,
                        use_cuda_graph=graph, n_scales=n_scales)
    assert list(net.state_dict().keys()) == list(sd0.keys())
    net.load_state_dict(sd0)
    return net.cuda()


def _train_vs_floor(arch, sd0, images, gts, loss_name="ce", sup=0.0):
    import _hrnet_asp_oracle as HA
    import _parity as P
    from oracle import seg_oracle as O
    hcfg = O.HRNET_W16_TEST
    crit, oracle_crit = ("rmi", O.criterion_rmi) if loss_name == "rmi" else (None, O.criterion_ce)
    sd_ref, loss_ref = HA.oracle_train_step(arch, hcfg, sd0, images, gts, sup, oracle_crit)
    floor, run_floor = HA.noise_floor(arch, hcfg, sd0, images, gts, sd_ref, sup, oracle_crit)
    net = _net(arch, sd0, crit, sup).train()
    loss = net({"images": images.cuda(), "gts": gts.cuda()})
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - loss_ref) <= 5e-3 * abs(loss_ref), (float(loss), loss_ref)
    for name, p in net.named_parameters():
        assert (sd_ref[name].grad is None) == (p.grad is None), name
    rep = P.grad_report(net, sd_ref)
    bad, summary = P.check_against_floor(rep, floor, P.running_report(net, sd_ref), run_floor)
    assert not bad, (summary, bad[:8])
    return net, sd_ref, rep, floor


@pytest.mark.parametrize("arch,loss_name,sup", TRAIN)
def test_train_step_matches_oracle(arch, loss_name, sup):
    """Loss, every gradient against the oracle's own one-bf16-ulp noise floor (tests/_parity.py), the logit heads
    tightly, BatchNorm bookkeeping (two passes for the mscale model, the 1.0x attention head included). gamma of
    aspp.img_conv.1 = 0 as in tests/test_gpu_deepv3.py: the batch-normalised 1x1 image-pooling branch of two crops is
    chaotic; the next test keeps it live with four crops."""
    import _hrnet_asp_oracle as HA
    from oracle import seg_oracle as O
    sd0 = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    sd0["aspp.img_conv.1.weight"].zero_()
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    net, sd_ref, rep, _floor = _train_vs_floor(arch, sd0, images, gts, loss_name, sup)
    heads = ("final.6.weight",) + (("scale_attn.conv2.weight",) if arch == "mscale.HRNet_ASP" else ())
    for name in heads:
        assert rep[name][0] >= 0.999, (name, rep[name])
    passes = 2 if arch == "mscale.HRNet_ASP" else 1
    sd = net.state_dict()
    bns = ["backbone.bn1", "aspp.features.0.1", "aspp.features.3.1", "aspp.img_conv.1", "final.4"]
    if arch == "mscale.HRNet_ASP":
        bns += ["scale_attn.bn0", "scale_attn.bn1"]
    for bnn in bns:
        assert int(sd[bnn + ".num_batches_tracked"]) == passes == int(sd_ref[bnn + ".num_batches_tracked"]), bnn
        ref = sd_ref[bnn + ".running_var"].detach().cpu()
        assert torch.allclose(sd[bnn + ".running_var"].float().cpu(), ref, rtol=3e-2, atol=1e-4), bnn


@pytest.mark.parametrize("arch", ["basic.HRNet_ASP", "mscale.HRNet_ASP"])
def test_train_step_image_pooling_live(arch):
    """The same with the image-pooling branch contributing (four crops: its batch normalisation is conditioned)."""
    import _hrnet_asp_oracle as HA
    from oracle import seg_oracle as O
    sd0 = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    images, gts = O.synth_batch(4, 128, 256, seed=6)
    _net_, _sd, rep, floor = _train_vs_floor(arch, sd0, images, gts)
    assert rep["aspp.img_conv.0.weight"][1] <= 2.0 * floor["aspp.img_conv.0.weight"][1] + 0.1


@pytest.mark.parametrize("arch,n_scales", [("basic.HRNet_ASP", None), ("mscale.HRNet_ASP", None),
                                           ("mscale.HRNet_ASP", [0.5, 1.0, 2.0])])
def test_eval_matches_oracle(arch, n_scales):
    """Evaluation (BatchNorm from non-trivial running statistics, folded into the convolution epilogues) against the
    oracle with bf16-storage emulation: every map of the reference's output dict, attention maps included."""
    import _hrnet_asp_oracle as HA
    from oracle import seg_oracle as O
    sd0 = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    g = torch.Generator().manual_seed(9)
    for k in sd0:
        if k.endswith("running_mean"):
            sd0[k] = 0.1 * torch.randn(sd0[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd0[k] = 0.5 + torch.rand(sd0[k].shape, generator=g)
    if arch == "mscale.HRNet_ASP":
        # attention logits in the O(1) range of a trained network: with the random head scaled by 0.1 (as for
        # mscale.DeepV3W38) 93 % of the 1.0x pass's attention map is above 1 - 1e-4, where fp32 steps of the sigmoid
        # are ~1 in logit
        sd0["scale_attn.conv2.weight"] = 0.01 * sd0["scale_attn.conv2.weight"]
    images, _ = O.synth_batch(2, 128, 256, seed=5)
    ctx = O.Ctx(O.clone_sd(sd0), training=False, emulate_bf16=True)
    with torch.no_grad():
        ref = HA.forward(ctx, arch, images) if n_scales is None else HA.nscale(ctx, images, n_scales)
    net = _net(arch, sd0, n_scales=n_scales).eval()
    with torch.no_grad():
        out = net({"images": images.cuda()})
    torch.cuda.synchronize()
    assert sorted(out.keys()) == sorted(ref.keys())
    for k, r in ref.items():
        o = out[k].float().cpu()
        assert o.shape == r.shape, (k, o.shape, r.shape)
        if r.shape[1] == 1:
            # compared as logits like the predictions (near the sigmoid's midpoint a small logit error moves the map)
            o, r = torch.logit(o.double(), eps=1e-7), torch.logit(r.double(), eps=1e-7)
        err = (o - r).abs().max().item()
        rng = (r.max() - r.min()).item()
        assert err <= 3e-2 * rng, (k, err, rng)
        if r.shape[1] == 19:
            agree = (o.argmax(1) == r.argmax(1)).float().mean().item()
            assert agree > 0.97, (k, agree)


@pytest.mark.parametrize("arch", ["basic.HRNet_ASP", "mscale.HRNet_ASP"])
def test_graph_replay_is_bitwise_eager(arch):
    """Captured training and evaluation replay bit-identically to eager; two eager runs are bit-identical."""
    import _hrnet_asp_oracle as HA
    from oracle import seg_oracle as O
    sd0 = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    images, gts = O.synth_batch(2, 128, 256, seed=5)
    runs = {}
    for tag, graph in (("eager", False), ("eager2", False), ("graph", True)):
        net = _net(arch, sd0, graph=graph).train()
        out = []
        for _ in range(3):
            net.zero_grad(set_to_none=True)
            loss = net({"images": images.cuda(), "gts": gts.cuda()})
            loss.backward()
            out.append((float(loss), {n: p.grad.clone() for n, p in net.named_parameters()}))
        net.eval()
        with torch.no_grad():
            ev = [net({"images": images.cuda()})["pred"].clone() for _ in range(3)]
        assert all(torch.equal(ev[0], e) for e in ev[1:])
        out.append(ev[-1])
        runs[tag] = out
    for tag in ("eager2", "graph"):
        for (la, ga), (lb, gb) in zip(runs["eager"][:3], runs[tag][:3]):
            assert la == lb, (tag, la, lb)
            differ = [n for n in ga if not torch.equal(ga[n], gb[n])]
            assert not differ, (tag, differ[:8])
        assert torch.equal(runs["eager"][3], runs[tag][3]), tag
