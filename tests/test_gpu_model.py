"""End-to-end parity of the B200 module (through the C ABI) against the oracle on identical weights and inputs.

The product computes in bf16 storage / fp32 accumulate while the oracle is fp32, so whole-network comparisons use
statistical tolerances (loss within a few 1e-2 relative, gradient cosine similarity), as discussed in SURVEY.md §7
"hard part 1"; op-level parity at matched precision lives in test_gpu_ops.py.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mods():
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    return O, B200SegModule


def _oracle_step(O, arch, hcfg, sd, images, gts, sup_wt=0.0, crit=None):
    sd = O.clone_sd(sd)
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    ctx = O.Ctx(sd, training=True)
    crit = crit or O.criterion_ce
    if arch == "mscale.HRNet":
        loss = O.mscale_basic_two_scale(ctx, images, gts, criterion=crit, hcfg=hcfg, supervised_mscale_wt=sup_wt)
    elif arch == "ocrnet.HRNet_Mscale":
        loss = O.mscale_two_scale(ctx, images, gts, criterion=crit, hcfg=hcfg, supervised_mscale_wt=sup_wt)
    elif arch == "ocrnet.HRNet":
        loss = O.ocrnet_forward(ctx, images, gts, criterion=crit, hcfg=hcfg)
    else:
        loss = O.basic_forward(ctx, images, gts, criterion=crit, hcfg=hcfg)
    loss.backward()
    return sd, float(loss)


@pytest.mark.parametrize("arch,sup", [("ocrnet.HRNet_Mscale", 0.0), ("ocrnet.HRNet_Mscale", 0.05),
                                      ("ocrnet.HRNet", 0.0), ("basic.HRNet", 0.0), ("mscale.HRNet", 0.05)])
def test_train_step_matches_oracle_w16(arch, sup):
    """One fused step vs the oracle at matched precision (bf16-storage emulation, run on the GPU through stock PyTorch
    fp32): loss to 5e-3, every per-tensor gradient within the oracle's own one-bf16-ulp noise floor (tests/_parity.py),
    the same zero pattern (the dead 1x attention head gets no gradient), running statistics, step bookkeeping."""
    import _parity as P
    O, B200SegModule = _mods()
    hcfg = O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    sd_ref, loss_ref = P.oracle_train_step(O, arch, hcfg, sd0, images, gts, sup)
    floor, run_floor = P.noise_floor(O, arch, hcfg, sd0, images, gts, sd_ref, sup)
    net, lv = P.product_train_step(B200SegModule, O, arch, hcfg, sd0, images, gts, sup)
    assert list(net.state_dict().keys()) == list(sd0.keys())
    assert abs(lv - loss_ref) <= 5e-3 * abs(loss_ref), (lv, loss_ref)
    for name, p in net.named_parameters():
        g_ref = sd_ref[name].grad
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        ref_zero = g_ref is None or float(g_ref.abs().max()) < 1e-7
        ours_zero = float(p.grad.abs().max()) == 0.0
        if name.endswith(".0.bias") and (".conv3x3_ocr." in name or ".aux_head.0" in name):
            continue    # bias in front of a training-mode BN: analytically zero
        assert ref_zero == ours_zero, (name, ref_zero, ours_zero)
    rep = {k: v for k, v in P.grad_report(net, sd_ref).items()
           if not (k.endswith(".0.bias") and (".conv3x3_ocr." in k or ".aux_head.0" in k))}
    bad, summary = P.check_against_floor(rep, floor, P.running_report(net, sd_ref), run_floor)
    assert not bad, (summary, bad[:8])
    # the tensors next to the loss see no gate-flip noise from above: tight agreement
    last = {"basic.HRNet": "seg_head.6.weight", "mscale.HRNet": "cls_head.6.weight"}.get(arch, "ocr.aux_head.2.bias")
    assert rep[last][0] >= 0.99, (last, rep[last])
    sd_new = net.state_dict()
    assert int(sd_new["backbone.bn1.num_batches_tracked"]) == int(sd_ref["backbone.bn1.num_batches_tracked"])


@pytest.mark.parametrize("arch,sup", [("ocrnet.HRNet_Mscale", 0.05), ("ocrnet.HRNet", 0.0)])
def test_train_step_with_rmi_criterion_w16(arch, sup):
    """The fused step with the RMILoss criterion (scripts/train_cityscapes.yml: rmi_loss: true): loss against the oracle,
    finite gradients everywhere, CUDA-graph replay equals the eager step."""
    O, B200SegModule = _mods()
    torch.set_num_threads(8)
    hcfg = O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    _, loss_ref = _oracle_step(O, arch, hcfg, sd0, images, gts, sup, crit=O.criterion_rmi)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    losses = []
    for use_graph in (False, True):
        net = B200SegModule(arch, 19, criterion="rmi", hcfg=hcfg, ocfg=ocfg, supervised_mscale_wt=sup,
                            use_cuda_graph=use_graph)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        for _ in range(3 if use_graph else 1):       # eager warm-up, capture, replay
            net.load_state_dict(sd0)                  # same weights / running stats for every call
            net.zero_grad(set_to_none=True)
            loss = net({"images": images.cuda(), "gts": gts.cuda()})
            loss.backward()
        torch.cuda.synchronize()
        losses.append(float(loss))
        for name, p in net.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), name
        assert float(net.last_loss_terms[5]) != 0.0
    assert abs(losses[0] - loss_ref) <= 3e-2 * abs(loss_ref), (losses, loss_ref)
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[0]), losses


def test_sgd_on_fixed_batch_tracks_oracle():
    """Optimising one fixed batch: the B200 path and the fp32 oracle must descend alike (bf16 noise is tiny compared
    with the loss decrease), which exercises the whole backward end to end without relying on chaotic per-tensor
    comparisons."""
    O, B200SegModule = _mods()
    torch.set_num_threads(8)
    arch, hcfg = "ocrnet.HRNet_Mscale", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    steps, lr = 12, 0.02
    # oracle curve (on the GPU for speed; fp32, TF32 off)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = {k: v.clone().cuda() for k, v in sd0.items()}
    params = [v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k]
    opt = torch.optim.SGD(params, lr=lr, momentum=0.9)
    ref_curve = []
    for _ in range(steps):
        opt.zero_grad()
        loss = O.mscale_two_scale(O.Ctx(sd, training=True), images.cuda(), gts.cuda(), hcfg=hcfg)
        loss.backward()
        opt.step()
        ref_curve.append(float(loss))
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=True)
    net.load_state_dict(sd0)
    net = net.cuda().train()
    opt2 = torch.optim.SGD(net.parameters(), lr=lr, momentum=0.9)
    curve = []
    for _ in range(steps):
        opt2.zero_grad()
        loss = net({"images": images.cuda(), "gts": gts.cuda()})
        loss.backward()
        opt2.step()
        curve.append(float(loss))
    for a, b in zip(curve, ref_curve):
        assert abs(a - b) <= 0.08 * abs(b) + 0.02, (curve, ref_curve)
    drop_ref = ref_curve[0] - ref_curve[-1]
    assert drop_ref > 0.1, ref_curve                       # the oracle itself descends on this batch
    assert curve[0] - curve[-1] > 0.5 * drop_ref, (curve, ref_curve)


@pytest.mark.parametrize("use_graph", [False, True])
def test_backward_applies_upstream_gradient_and_accumulates(use_graph):
    """The autograd boundary (train.py:499-505): (k * loss).backward() publishes k * gradient (amp.scale_loss, loss /
    accumulation steps), live .grad tensors are accumulated into, dropped ones replaced, a foreign .grad tensor receives
    the step's contribution, and a forward without backward leaves param.grad alone."""
    O, B200SegModule = _mods()
    arch, hcfg = "ocrnet.HRNet_Mscale", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=use_graph)
    net.load_state_dict(sd0)
    net = net.cuda().train()
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    batch = {"images": images.cuda(), "gts": gts.cuda()}

    def flat():
        return torch.cat([p.grad.flatten() for p in net.parameters()]).clone()

    rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
    for _ in range(3 if use_graph else 1):          # eager warm-up, capture, replay
        net.zero_grad(set_to_none=True)
        net(batch).backward()
    g1 = flat()
    assert float(g1.norm()) > 0
    net.zero_grad(set_to_none=True)
    (net(batch) * 0.25).backward()                   # scaled loss
    assert rel(flat(), 0.25 * g1) <= 1e-5
    net(batch).backward()                            # live gradients: accumulate on top
    assert rel(flat(), 1.25 * g1) <= 1e-5
    before = flat()
    net(batch)                                       # forward only: nothing is published
    torch.cuda.synchronize()
    assert torch.equal(flat(), before)
    net.zero_grad(set_to_none=False)                 # in-place zeroing keeps the aliased views
    net(batch).backward()
    assert rel(flat(), g1) <= 1e-5
    names = [n for n, _ in net.named_parameters()]
    pieces = dict(zip(names, torch.split(g1, [p.numel() for p in net.parameters()])))
    p0 = net.get_parameter("ocr.cls_head.weight")    # a caller-owned gradient tensor
    own = torch.full_like(p0, 2.0)
    p0.grad = own
    (net(batch) * 2.0).backward()
    assert p0.grad is own
    assert rel(own, 2.0 + 2.0 * pieces["ocr.cls_head.weight"].view_as(p0)) <= 1e-5
    for n in ("backbone.conv1.weight", "scale_attn.conv0.weight", "ocr.aux_head.2.bias"):
        assert rel(net.get_parameter(n).grad.flatten(), 3.0 * pieces[n]) <= 1e-5, n     # 1 (previous) + 2 (this step)


def test_cuda_graph_replay_equals_eager():
    O, B200SegModule = _mods()
    hcfg = O.HRNET_W16_TEST
    arch = "ocrnet.HRNet_Mscale"
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    nets = []
    for use_graph in (False, True):
        net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=use_graph)
        net.load_state_dict(sd0)
        nets.append(net.cuda().train())
    opts = [torch.optim.SGD(n.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4) for n in nets]
    for step in range(4):
        images, gts = O.synth_batch(2, 64, 128, seed=100 + step)
        losses = []
        for net, opt in zip(nets, opts):
            opt.zero_grad()
            loss = net({"images": images.cuda(), "gts": gts.cuda()})
            loss.backward()
            opt.step()
            losses.append(float(loss))
        assert abs(losses[0] - losses[1]) <= 2e-3 * abs(losses[0]), (step, losses)


def test_train_step_is_bitwise_reproducible():
    """Two runs of one step on the same weights and batch: identical loss and gradients (fixed summation orders)."""
    O, B200SegModule = _mods()
    hcfg = O.HRNET_W16_TEST
    arch = "ocrnet.HRNet_Mscale"
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    images, gts = O.synth_batch(2, 64, 128, seed=7)
    runs = []
    for _ in range(2):
        net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=False)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        loss = net({"images": images.cuda(), "gts": gts.cuda()})
        loss.backward()
        runs.append((float(loss), {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}))
    assert runs[0][0] == runs[1][0], (runs[0][0], runs[1][0])
    assert runs[0][1].keys() == runs[1][1].keys()
    differ = [n for n in runs[0][1] if not torch.equal(runs[0][1][n], runs[1][1][n])]
    assert not differ, differ[:8]


def _condition_eval_weights(sd0):
    """Randomly initialised heads produce soft-region logits of magnitude ~150 and attention logits of ~1e3: both feed a
    softmax, so a 1 % bf16 difference in a logit changes a probability by e^1.5 and an eval comparison against ANY
    other arithmetic (the reference's own autocast path included) is meaningless. Scale the three softmax inputs to the
    O(1) range a trained network has; everything else keeps the synthetic weights."""
    for k, f in (("ocr.aux_head.2.weight", 0.02), ("ocr.aux_head.2.bias", 0.02),
                 ("ocr.ocr_distri_head.object_context_block.f_pixel.3.0.weight", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_pixel.3.0.bias", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_object.3.0.weight", 0.1),
                 ("ocr.ocr_distri_head.object_context_block.f_object.3.0.bias", 0.1)):
        if k in sd0:
            sd0[k] = sd0[k] * f


@pytest.mark.parametrize("arch,n_scales", [("ocrnet.HRNet_Mscale", None), ("ocrnet.HRNet_Mscale", [0.5, 1.0, 2.0]),
                                           ("ocrnet.HRNet", None), ("basic.HRNet", None),
                                           ("mscale.HRNet", None), ("mscale.HRNet", [0.5, 1.0, 2.0])])
def test_eval_forward_matches_oracle(arch, n_scales):
    """Eval mode (running-stat BN: no batch-statistics chaos) against the oracle with bf16-storage emulation: same dict
    keys as the reference (network/ocrnet.py:234-262,319-327), fp32 NCHW maps, argmax agreement."""
    O, B200SegModule = _mods()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    hcfg = O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    # non-trivial running statistics
    g = torch.Generator().manual_seed(9)
    for k in sd0:
        if k.endswith("running_mean"):
            sd0[k] = 0.1 * torch.randn(sd0[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd0[k] = 0.5 + torch.rand(sd0[k].shape, generator=g)
    _condition_eval_weights(sd0)
    images, _ = O.synth_batch(2, 64, 128, seed=5)
    sd = {k: v.clone().cuda() for k, v in sd0.items()}
    ctx = O.Ctx(sd, training=False, emulate_bf16=True)
    with torch.no_grad():
        if arch == "ocrnet.HRNet_Mscale":
            ref = O.mscale_nscale(ctx, images.cuda(), n_scales, hcfg=hcfg) if n_scales else \
                O.mscale_two_scale(ctx, images.cuda(), hcfg=hcfg)
        elif arch == "mscale.HRNet":
            ref = O.mscale_basic_nscale(ctx, images.cuda(), n_scales, hcfg=hcfg) if n_scales else \
                O.mscale_basic_two_scale(ctx, images.cuda(), hcfg=hcfg)
        elif arch == "ocrnet.HRNet":
            ref = O.ocrnet_forward(ctx, images.cuda(), hcfg=hcfg)
        else:
            ref = O.basic_forward(ctx, images.cuda(), hcfg=hcfg)
    net = B200SegModule(arch, 19, hcfg=hcfg, n_scales=n_scales)
    net.load_state_dict(sd0)
    net = net.cuda().eval()
    out = net({"images": images.cuda()})
    assert sorted(out.keys()) == sorted(ref.keys())
    for k in ref:
        a, b = out[k].double(), ref[k].double()
        assert a.shape == b.shape, (k, a.shape, b.shape)
        rel = float((a - b).norm() / (b.norm() + 1e-30))
        assert rel < 0.03, (k, rel)
    agree = float((out["pred"].argmax(1) == ref["pred"].argmax(1)).float().mean())
    assert agree > 0.97, agree


def test_eval_minibatch_device_tail_matches_host_scoring():
    """b200seg.evaltail.eval_minibatch (flip + two input scales, utils/trnval_utils.py:116-196) against the same loop
    written with torch ops on the module's own 'pred' outputs: identical class map and confusion matrix."""
    import torch.nn.functional as F
    O, B200SegModule = _mods()
    from b200seg.evaltail import eval_minibatch, iou_from_hist
    arch, hcfg = "ocrnet.HRNet", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    _condition_eval_weights(sd0)
    images, gts = O.synth_batch(2, 64, 128, seed=5)
    net = B200SegModule(arch, 19, hcfg=hcfg)
    net.load_state_dict(sd0)
    net = net.cuda().eval()
    im, gt = images.cuda(), gts.cuda()
    scales = (0.5, 1.0)
    res = eval_minibatch(net, im, gt, scales=scales, do_flip=True)
    out = 0.0
    with torch.no_grad():
        for flip in (1, 0):
            for s in scales:
                x = torch.flip(im, dims=[3]) if flip else im
                if s != 1.0:
                    x = F.interpolate(x, size=(round(64 * s), round(128 * s)), mode="bilinear", align_corners=False)
                p = net({"images": x})["pred"]
                if s != 1.0:
                    p = F.interpolate(p, size=(64, 128), mode="bilinear", align_corners=False)
                out = out + (torch.flip(p, dims=[3]) if flip else p)
    out = out / 4
    prob, arg = F.softmax(out, dim=1).max(1)
    agree = float((res["predictions"] == arg).float().mean())
    assert agree > 0.999, agree                                    # resize arithmetic differs in the last ulp only
    mask = gt < 19
    ref_hist = torch.bincount(19 * gt[mask] + arg[mask], minlength=361).view(19, 19)
    assert int((res["hist"] - ref_hist).abs().sum()) <= 4
    assert res["hist"].sum() == mask.sum()
    assert iou_from_hist(res["hist"]).shape == (19,)


def test_device_prefetcher_double_buffer_keeps_batches_intact():
    """b200seg.prefetch.DevicePrefetcher: batches arrive on the device unchanged and in order while a slow consumer runs on
    the compute stream (the copy of batch i+1 may only overwrite a slot after the step that used it has finished)."""
    from b200seg.prefetch import DevicePrefetcher
    g = torch.Generator().manual_seed(0)
    host = [{"images": torch.randn((1, 3, 64, 128), generator=g).pin_memory(),
             "gts": torch.randint(0, 19, (1, 64, 128), generator=g).pin_memory()} for _ in range(7)]
    big = torch.randn((4096, 4096), device="cuda")
    sums = []
    for i, b in enumerate(DevicePrefetcher(host)):
        assert b["images"].is_cuda and b["gts"].dtype == torch.long
        for _ in range(3):
            big = (big @ big).tanh_()                 # keep the compute stream busy after the batch was handed out
        sums.append((b["images"].double().sum() + b["gts"].double().sum()).clone())
    torch.cuda.synchronize()
    assert len(sums) == 7
    for i, s in enumerate(sums):
        want = host[i]["images"].double().sum() + host[i]["gts"].double().sum()
        assert abs(float(s) - float(want)) <= 1e-6 * abs(float(want)) + 1e-6, i


@pytest.mark.parametrize("n_scales", [None, [0.5, 1.0, 2.0]])
def test_eval_graph_replay_equals_eager(n_scales):
    """Eval mode: eager first call, captured second call, replays - identical maps, fresh output tensors, new weights and
    new inputs are picked up by the replay."""
    O, B200SegModule = _mods()
    arch, hcfg = "ocrnet.HRNet_Mscale", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    _condition_eval_weights(sd0)
    net = B200SegModule(arch, 19, hcfg=hcfg, n_scales=n_scales)
    net.load_state_dict(sd0)
    net = net.cuda().eval()
    ims = [O.synth_batch(2, 64, 128, seed=s)[0].cuda() for s in (5, 6)]
    eager = [net({"images": ims[0]})]                       # call 1: eager
    outs = [net({"images": ims[0]}), net({"images": ims[0]})]   # capture + replay
    for o in outs:
        assert sorted(o.keys()) == sorted(eager[0].keys())
        for k in o:
            assert torch.equal(o[k], eager[0][k]), k
    assert outs[0]["pred"].data_ptr() != outs[1]["pred"].data_ptr()
    ref_net = B200SegModule(arch, 19, hcfg=hcfg, n_scales=n_scales, use_cuda_graph=False)
    ref_net.load_state_dict(sd0)
    ref_net = ref_net.cuda().eval()
    with torch.no_grad():                                   # new weights + new input through the replay
        for p in list(net.parameters()) + list(ref_net.parameters()):
            p.mul_(1.01)
    a, b = net({"images": ims[1]}), ref_net({"images": ims[1]})
    for k in a:
        assert torch.equal(a[k], b[k]), k
