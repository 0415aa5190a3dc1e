"""The attention-head ablations --mscale_no3x3, --mscale_dropout and --mscale_old_arch on the sm_90a kernels: the
element-wise Dropout(0.5) fused into the BatchNorm apply / backward passes (csrc/dropout.cuh) against PyTorch given the
kernels' own keep mask, its bit statistics, and W16 training / evaluation of the four multi-scale archs against the
GPU-run oracle (tests/_attn_head_oracle.py, pinned to the reference by tests/test_attn_head_host.py)."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

ARCHS = ("ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.HRNet_ASP", "mscale.DeepV3W38")
# narrow WRN-38 of tests/test_gpu_mscale_deepv3.py
WRN_TEST = dict(structure=[2, 1, 1, 1, 1, 1],
                channels=[(32, 32), (64, 64), (64, 64), (64, 128), (64, 128, 256), (128, 256, 512)])


def _hcfg(arch):
    from oracle import seg_oracle as O
    return WRN_TEST if arch == "mscale.DeepV3W38" else O.HRNET_W16_TEST


VARIANTS = ("no3x3", "dropout", "oldarch", "no3x3_dropout")


def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device="cuda")


def _mask(seed, pass_idx, n, h, w, c):
    from b200seg import raw
    return raw.dropout_keep_mask(seed, pass_idx, n * h * w, c).view(n, h, w, c)


# ----------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("cells", [False, True])
def test_dropout_apply_and_backward_match_torch(cells):
    """z = relu(bn(y)) * keep * 2 and its input gradient, with the keep mask from the test entry point, against
    PyTorch fp32 batch norm on the same bf16 input; the apply pass reproduces the mask exactly (zeros where dropped)."""
    from b200seg import raw
    torch.manual_seed(0)
    n, h, w, c = 2, 24, 40, 256
    y = torch.randn((n, h, w, c), device="cuda").to(torch.bfloat16)
    gamma = (1.0 + 0.1 * torch.randn(c, device="cuda")).contiguous()
    beta = (0.1 * torch.randn(c, device="cuda")).contiguous()
    yf = y.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    mean = yf.detach().mean((0, 2, 3))
    var = yf.detach().var((0, 2, 3), unbiased=False)
    invstd = torch.rsqrt(var + 1e-5)
    scale = (gamma * invstd).contiguous()
    shift = (beta - mean * scale).contiguous()
    seed = _seed(0x1234_5678_9ABC_DEF0 - 2 ** 63)
    keep = _mask(seed, 1, n, h, w, c)
    drop = (seed, 1)
    z = raw.bn_apply(y, scale, shift, None, None, True, dropout=drop)
    ref = torch.relu(torch.nn.functional.batch_norm(yf, None, None, gamma, beta, True, 0.0, 1e-5))
    ref_z = ref * keep.permute(0, 3, 1, 2).float() * 2.0
    zc = z.float().permute(0, 3, 1, 2)
    kept = keep.permute(0, 3, 1, 2) == 1
    assert bool((zc[~kept] == 0).all())                    # dropped elements are exactly zero ...
    assert bool((zc[kept & (ref > 1e-2)] != 0).all())      # ... and kept positive ones are not
    assert (zc - ref_z).abs().max().item() <= 2e-2 * ref_z.abs().max().item()
    dz = torch.randn((n, h, w, c), device="cuda").to(torch.bfloat16)
    ref_z.backward(dz.float().permute(0, 3, 1, 2))
    dgamma = torch.zeros(c, device="cuda")
    dbeta = torch.zeros(c, device="cuda")
    cell = torch.zeros(2 * c, dtype=torch.float64, device="cuda") if cells else None
    dy = raw.bn_bwd(dz, z, None, y, mean.contiguous(), invstd.contiguous(), gamma, dgamma, dbeta, cells=cell,
                    dropout=drop)
    torch.cuda.synchronize()
    g_ref = yf.grad.permute(0, 2, 3, 1)
    err = (dy.float() - g_ref).abs().max().item()
    assert err <= 2e-2 * g_ref.abs().max().item(), err
    cos = torch.nn.functional.cosine_similarity(dy.float().flatten(), g_ref.flatten(), dim=0).item()
    assert cos > 0.9999, cos


def test_dropout_mask_statistics():
    """Keep fraction over 10^7 elements within 5 sigma of 1/2; same key -> same bits; another seed or another pass
    index -> independent bits (agreement within 5 sigma of 1/2)."""
    npix, c = 39064, 256          # 10 000 384 elements
    nel = npix * c
    sig = 5.0 * math.sqrt(0.25 / nel)
    a = _mask(_seed(17), 0, 1, npix, 1, c).flatten().float()
    assert abs(a.mean().item() - 0.5) <= sig
    assert torch.equal(a, _mask(_seed(17), 0, 1, npix, 1, c).flatten().float())
    for other in (_mask(_seed(18), 0, 1, npix, 1, c), _mask(_seed(17), 1, 1, npix, 1, c),
                  _mask(_seed(-(2 ** 62)), 0, 1, npix, 1, c)):
        agree = (other.flatten().float() == a).float().mean().item()
        assert abs(agree - 0.5) <= sig, agree
    # runs of 128 elements come from one generator call: neighbouring blocks must not repeat
    blocks = a.view(-1, 128)
    assert not torch.equal(blocks[0], blocks[1])


# ----------------------------------------------------------------------------------------------- models
def _net(arch, variant, sd0, graph=False, n_scales=None, criterion=None, sup=0.0):
    import _attn_head_oracle as AH
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    ocfg = dict(O.OCR_CFG, dropout=0.0, **AH.ocfg_keys(variant))
    hcfg = _hcfg(arch)
    net = B200SegModule(arch, 19, criterion=criterion, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=graph, n_scales=n_scales,
                        supervised_mscale_wt=sup)
    net.wrn_dropout_scale = 0.0
    assert list(net.state_dict().keys()) == list(sd0.keys())
    net.load_state_dict(sd0)
    return net.cuda()


def _kernel_keep_fn(net, n, hw_lo, hw_hi):
    """The keep masks the step's kernels used (0.5x pass, then 1.0x pass), NCHW, for the oracle's head."""
    masks = []
    for p, (h, w) in enumerate((hw_lo, hw_hi)):
        masks.append(_mask(net.last_attn_seed, p, n, h, w, 256).permute(0, 3, 1, 2).float())
    it = iter(masks)

    def fn(shape):
        m = next(it)
        assert tuple(m.shape) == tuple(shape), (m.shape, shape)
        return m
    return fn


def _cases():
    import _attn_head_oracle as AH
    return [(a, v) for a in ARCHS for v in VARIANTS if AH.supported(a, v)]


@pytest.mark.parametrize("arch,variant", _cases())
def test_train_step_matches_oracle(arch, variant):
    """W16 (narrow WRN-38 for mscale.DeepV3W38) training step: loss within 5e-3, every gradient against the oracle's
    one-ulp noise floor (tests/_parity.py), the attention head's BatchNorm bookkeeping; dropout variants are given the
    kernels' keep masks. mscale.DeepV3W38 as in tests/test_gpu_mscale_deepv3.py: 128 x 256 crops and gamma of
    aspp.img_conv.1 = 0 (the batch-normalised image-pooling branch of two crops is chaotic)."""
    import _attn_head_oracle as AH
    import _parity as P
    from oracle import seg_oracle as O
    hcfg = _hcfg(arch)
    sd0 = AH.synth_state_dict(arch, variant, hcfg, seed=3)
    n, H, W = 2, 64, 128
    if arch == "mscale.DeepV3W38":
        sd0["aspp.img_conv.1.weight"].zero_()
        H, W = 128, 256
    images, gts = O.synth_batch(n, H, W, seed=5)
    net = _net(arch, variant, sd0).train()
    torch.manual_seed(11)
    torch.cuda.manual_seed(11)
    loss = net({"images": images.cuda(), "gts": gts.cuda()})
    loss.backward()
    torch.cuda.synchronize()
    drop = AH.head_layers(variant)[2]
    f = 2 if arch == "mscale.DeepV3W38" else 4
    factory = (lambda: _kernel_keep_fn(net, n, (H // 2 // f, W // 2 // f), (H // f, W // f))) if drop else None
    sd_ref, loss_ref = AH.oracle_train_step(arch, variant, hcfg, sd0, images, gts, factory() if drop else None)
    floor, run_floor = AH.noise_floor(arch, variant, hcfg, sd0, images, gts, sd_ref, factory)
    assert abs(float(loss) - loss_ref) <= 5e-3 * abs(loss_ref), (float(loss), loss_ref)
    for name, p in net.named_parameters():
        assert (sd_ref[name].grad is None) == (p.grad is None), name
    rep = P.grad_report(net, sd_ref)
    bad, summary = P.check_against_floor(rep, floor, P.running_report(net, sd_ref), run_floor)
    assert not bad, (summary, bad[:8])
    sd = net.state_dict()
    for _c, b in AH.head_layers(variant)[0]:
        assert int(sd[b + ".num_batches_tracked"]) == 2 == int(sd_ref[b + ".num_batches_tracked"]), b


@pytest.mark.parametrize("arch", ["ocrnet.HRNet_Mscale", "mscale.HRNet"])
def test_dropout_replays_draw_fresh_masks_and_match_eager(arch):
    """Captured steps draw a new seed per replay (different keep masks, different gradients); with the same torch
    seed an eager step and a graph replay are bit-identical."""
    import _attn_head_oracle as AH
    from oracle import seg_oracle as O
    variant = "dropout"
    sd0 = AH.synth_state_dict(arch, variant, O.HRNET_W16_TEST, seed=3)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    runs = {}
    for tag, graph in (("eager", False), ("graph", True)):
        net = _net(arch, variant, sd0, graph=graph).train()
        out = []
        for i in range(4):
            torch.cuda.manual_seed(100 + i)
            net.zero_grad(set_to_none=True)
            loss = net({"images": images.cuda(), "gts": gts.cuda()})
            loss.backward()
            torch.cuda.synchronize()
            out.append((float(loss), int(net.last_attn_seed.item()),
                        {n: p.grad.clone() for n, p in net.named_parameters()}))
        runs[tag] = out
    for (la, sa, ga), (lb, sb, gb) in zip(runs["eager"], runs["graph"]):
        assert sa == sb and la == lb, (sa, sb, la, lb)
        differ = [n for n in ga if not torch.equal(ga[n], gb[n])]
        assert not differ, differ[:8]
    g = runs["graph"]
    assert g[2][1] != g[3][1]
    m2 = _mask(_seed(g[2][1]), 0, 2, 8, 16, 256)
    m3 = _mask(_seed(g[3][1]), 0, 2, 8, 16, 256)
    assert not torch.equal(m2, m3)
    assert not torch.equal(g[2][2]["scale_attn.conv2.weight"], g[3][2]["scale_attn.conv2.weight"])


@pytest.mark.parametrize("arch,variant,n_scales", [(a, v, s) for a, v in _cases() if v in ("no3x3", "oldarch")
                                                   for s in (None, [0.5, 1.0, 2.0])])
def test_eval_matches_oracle(arch, variant, n_scales):
    """Two- and three-scale evaluation (BatchNorm from non-trivial running statistics) against the oracle with
    bf16-storage emulation, as in tests/test_gpu_hrnet_asp.py. The softmax / sigmoid inputs of the random heads are
    scaled to the O(1) range of a trained network as in tests/test_gpu_model.py and tests/test_gpu_mscale_deepv3.py."""
    import _attn_head_oracle as AH
    from oracle import seg_oracle as O
    sd0 = AH.synth_state_dict(arch, variant, _hcfg(arch), seed=3)
    g = torch.Generator().manual_seed(9)
    for k in sd0:
        if k.endswith("running_mean"):
            sd0[k] = 0.1 * torch.randn(sd0[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd0[k] = 0.5 + torch.rand(sd0[k].shape, generator=g)
    last = "scale_attn" + (".6" if variant == "oldarch" else ".conv2") + ".weight"
    sd0[last] = 0.01 * sd0[last]
    for k, f in (("ocr.aux_head.2.weight", 0.02), ("ocr.aux_head.2.bias", 0.02),
                 ("ocr.ocr_distri_head.object_context_block.f_pixel.3.0.weight", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_pixel.3.0.bias", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_object.3.0.weight", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_object.3.0.bias", 0.1)):
        if k in sd0:
            sd0[k] = sd0[k] * f
    images, _ = O.synth_batch(2, 128, 256, seed=5)
    ctx = O.Ctx(O.clone_sd(sd0), training=False, emulate_bf16=True)
    with torch.no_grad():
        ref = AH.forward(arch, variant, ctx, images, hcfg=_hcfg(arch), scales=n_scales)
    net = _net(arch, variant, sd0, n_scales=n_scales).eval()
    with torch.no_grad():
        out = net({"images": images.cuda()})
    torch.cuda.synchronize()
    assert sorted(out.keys()) == sorted(ref.keys())
    for k, r in ref.items():
        o = out[k].float().cpu()
        assert o.shape == r.shape, (k, o.shape, r.shape)
        if r.shape[1] == 1:
            o, r = torch.logit(o.double(), eps=1e-7), torch.logit(r.double(), eps=1e-7)
        err = (o - r).abs().max().item()
        rng = (r.max() - r.min()).item()
        assert err <= 3e-2 * rng, (k, err, rng)
        if r.shape[1] == 19:
            agree = (o.argmax(1) == r.argmax(1)).float().mean().item()
            assert agree > 0.97, (k, agree)
