"""The launches that run once per training step around the network, over every architecture's real parameter table:
the end-of-step gradient fold (grad_fold), the gradient publish (publish_grads), the deferred BatchNorm running-statistics
update (bn_running_update), the weight repacking (pack_weights) and the optimizer (sgd_step through FusedSGD).

The tables are the module's own: the fold segments B200SegModule builds (the stem accumulating on the 16-channel padded
image), the pack table _repack builds (stem i_dst 16, o_pad = roundup8(o)), its flat BatchNorm running layout and its
parameters for FusedSGD. The fold table and the parameter list get two extra items, one of exactly one chunk and one
whose last chunk holds 3 elements (a second pack table holds two such items).
Bounds: the fold's plain additions and the packing are bit for bit against the same fp32 additions in the kernel's order
and one bf16 rounding; the multiply-adds (publish with accumulate, the running-statistics update, the SGD step), which
nvcc may contract to FMAs, are checked from the kernel's own previous state within one fp32 ulp of the float64 value of
each step's operand magnitudes. accum_f32 has no caller in the training step and is not tested here.
"""
import pytest

ARCHS = ("ocrnet.HRNet_Mscale", "ocrnet.HRNet", "basic.HRNet", "mscale.HRNet", "deepv3.DeepV3PlusW38",
         "mscale.DeepV3W38", "basic.HRNet_ASP", "mscale.HRNet_ASP")


def _torch():
    import torch
    from b200seg import raw
    return torch, raw


def _ulp32(x):
    torch, _ = _torch()
    _m, e = torch.frexp(x.abs().float().double())
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -149), torch.ldexp(torch.ones_like(x), e - 24))


def _within_ulp(got, r, mag, what, carried=0.0):
    """|got - r| <= one fp32 ulp of mag (float64 magnitude of the step's operands) plus the error carried in from
    earlier steps of the same launch."""
    err = (got.double() - r).abs()
    bad = int((err > _ulp32(mag) + carried).sum())
    assert bad == 0, "%s: %d elements off by more than one fp32 ulp (max %.3e)" % (what, bad, float(err.max()))


def _module(arch):
    """B200SegModule on the GPU with its device state, and the fold segments its constructor handed to grad_fold_table."""
    torch, raw = _torch()
    from b200seg.module import B200SegModule
    segs = []
    orig = raw.grad_fold_table

    def capture(s, dev):
        segs[:] = list(s)
        return orig(s, dev)
    raw.grad_fold_table = capture
    try:
        torch.manual_seed(0)
        net = B200SegModule(arch, 19).cuda()
        net._ensure_device_state()
    finally:
        raw.grad_fold_table = orig
    return net, segs


def _fold_index(segs, total):
    """For every dst element of the segments: the accumulator element grad_fold reads."""
    torch, _ = _torch()
    src = torch.full((total,), -1, dtype=torch.int64, device="cuda")
    for off, soff, cout, cin, taps, scin in segs:
        co = torch.arange(cout, device="cuda").view(-1, 1, 1)
        ci = torch.arange(cin, device="cuda").view(1, -1, 1)
        t = torch.arange(taps, device="cuda").view(1, 1, -1)
        src[off:off + cout * cin * taps] = (soff + (co * taps + t) * scin + ci).reshape(-1)
    return src


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ARCHS)
def test_fold_publish_running_update_and_pack(arch):
    torch, raw = _torch()
    net, segs = _module(arch)
    chunk = raw.lib().b200seg_grad_fold_chunk()
    total = net._step_flat.numel()
    acc_len = net._acc_hi.numel()
    # two extra vector segments behind everything: one chunk exactly, one chunk + 3 (a last chunk of 3 elements)
    extra = [(total, acc_len, 1, chunk, 1, chunk), (total + chunk, acc_len + chunk, 1, chunk + 3, 1, chunk + 3)]
    segs = segs + extra
    n_dst, n_acc = total + 2 * chunk + 3, acc_len + 2 * chunk + 3
    table = raw.grad_fold_table(segs, "cuda")
    idx = _fold_index(segs, n_dst)
    used = idx >= 0
    g = torch.Generator(device="cuda").manual_seed(1)
    for overwrite, with_b, clear in ((False, False, False), (True, True, False), (False, True, True)):
        a = torch.randn(n_acc, generator=g, device="cuda")
        b = torch.randn(n_acc, generator=g, device="cuda") if with_b else None
        dst = torch.randn(n_dst, generator=g, device="cuda")
        a0, b0, d0 = a.clone(), (b.clone() if with_b else None), dst.clone()
        raw.grad_fold(dst, a, b, table, clear=clear, overwrite=overwrite)
        torch.cuda.synchronize()
        want = torch.zeros_like(d0) if overwrite else d0.clone()
        want[used] = want[used] + a0[idx[used]]
        if with_b:
            want[used] = want[used] + b0[idx[used]]
        what = "%s grad_fold overwrite=%d acc_b=%d clear=%d" % (arch, overwrite, with_b, clear)
        assert torch.equal(dst[used].view(torch.int32), want[used].view(torch.int32)), what
        assert torch.equal(dst[~used], d0[~used]), what + ": padding written"
        read = torch.zeros(n_acc, dtype=torch.bool, device="cuda")
        read[idx[used]] = True
        for acc, acc0 in ((a, a0), (b, b0)):
            if acc is None:
                continue
            if clear:
                assert bool((acc[read] == 0).all()) and torch.equal(acc[~read], acc0[~read]), what + ": clearing"
            else:
                assert torch.equal(acc, acc0), what + ": accumulator changed"

    # publish_grads over the flat gradient: dst = (accumulate ? dst : 0) + (*scale_dev * scale_const) * src
    src = torch.randn(total, generator=g, device="cuda")
    for accumulate, sdev in ((False, None), (True, torch.tensor([0.37], device="cuda")), (True, None),
                             (False, torch.tensor([3.0], device="cuda"))):
        dst = torch.randn(total, generator=g, device="cuda")
        d0 = dst.clone()
        raw.publish_grads(dst, src, sdev, 0.5, accumulate=accumulate)
        torch.cuda.synchronize()
        sc = (sdev if sdev is not None else torch.ones(1, device="cuda")) * torch.tensor([0.5], device="cuda")
        prod = sc.double() * src.double()
        what = "%s publish_grads accumulate=%d scale_dev=%d" % (arch, accumulate, sdev is not None)
        if not accumulate:
            assert torch.equal(dst, (sc * src) + 0.0), what
        else:
            _within_ulp(dst, d0.double() + prod, d0.double().abs() + prod.abs(), what)

    # bn_running_update over the flat running layout, one and two passes
    run = net._run_flat
    n_layers = net._nbt_flat.numel()
    m = torch.tensor(0.1, dtype=torch.float32)
    om = (1.0 - m).double()
    for passes in (1, 2):
        r0 = torch.rand(run.numel(), generator=g, device="cuda") * 2 - 0.5
        b0, b1 = torch.randn(run.numel(), generator=g, device="cuda"), torch.randn(run.numel(), generator=g, device="cuda")
        run.copy_(r0)
        nbt0 = net._nbt_flat.clone()
        raw.bn_running_update(run, b0, b1 if passes == 2 else None, 0.1, net._nbt_flat, passes)
        torch.cuda.synchronize()
        md = m.double()
        r1 = om * r0.double() + md * b0.double()
        mag = om * r0.double().abs() + md * b0.double().abs()
        carried = 0.0
        if passes == 2:
            # the intermediate is not observable: the first step's ulp reaches the result scaled by (1 - m)
            carried = om * _ulp32(mag)
            mag = om * r1.abs() + md * b1.double().abs()
            r1 = om * r1 + md * b1.double()
        _within_ulp(run, r1, mag, "%s bn_running_update passes=%d" % (arch, passes), carried)
        assert torch.equal(net._nbt_flat, nbt0 + passes), arch
        assert n_layers > 0

    # pack_weights: the module's own pack table (B200SegModule._repack), read back item by item, plus a table of one
    # item of exactly one chunk and one of a chunk + 3 elements
    import numpy as np
    pchunk = raw.lib().b200seg_pack_chunk()
    net._repack()
    own = net._pack_table
    by_ptr = {p.data_ptr(): p.detach() for _n, p in net.named_parameters() if p.dim() == 4}
    outs = {}
    for w_f, w_d in net._packed.values():
        outs[w_f.data_ptr()], outs[w_d.data_ptr()] = w_f, w_d
    fields = np.dtype([("w", "<u8"), ("f", "<u8"), ("d", "<u8"), ("o", "<i4"), ("i", "<i4"), ("i_dst", "<i4"),
                       ("k", "<i4"), ("o_pad", "<i4"), ("r", "<i4")])
    items = own["items"].cpu().numpy().view(fields)
    entries = [(by_ptr[int(it["w"])], outs[int(it["f"])], outs[int(it["d"])]) for it in items]
    assert len(entries) == len(by_ptr)
    extra = []
    for shape in ((16, pchunk // 16, 1, 1), (1, pchunk + 3, 1, 1)):
        o, i = shape[0], shape[1]
        extra.append((torch.randn(shape, generator=g, device="cuda"),
                      torch.empty((o, 1, i), dtype=torch.bfloat16, device="cuda"),
                      torch.empty((i, 1, (o + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")))
    for which in (1, 2, 3):
        for tab, ents in ((own, entries), (raw.pack_table(extra, "cuda"), extra)):
            for _w, wf, wd in ents:
                wf.fill_(float("nan"))
                wd.fill_(float("nan"))
            raw.pack_weights(tab, which)
            torch.cuda.synchronize()
            for w, wf, wd in ents:
                o, i, k, _ = w.shape
                wb = w.to(torch.bfloat16)
                what = "%s pack_weights which=%d %s" % (arch, which, tuple(w.shape))
                assert wf.shape[2] == (16 if i == 3 else i) and wd.shape[2] == (o + 7) // 8 * 8, what
                f_want = torch.full_like(wf, float("nan"))
                if which & 1:
                    f_want[:, :, :i] = wb.permute(0, 2, 3, 1).reshape(o, k * k, i)
                d_want = torch.full_like(wd, float("nan"))
                if which & 2:
                    d_want[:i, :, :o] = wb.flip(2, 3).permute(1, 2, 3, 0).reshape(i, k * k, o)
                assert torch.equal(wf.view(torch.int16), f_want.view(torch.int16)), what + ": forward operand"
                assert torch.equal(wd.view(torch.int16), d_want.view(torch.int16)), what + ": data-gradient operand"


def _sgd_reference(w, grad, buf, lr, momentum, dampening, weight_decay, nesterov, fresh):
    """One torch.optim.SGD step in float64 from the kernel's fp32 state (w, buf) with the kernel's fp32 constants ->
    (param, buffer) and, for each, (operand magnitude, error carried in from the earlier multiply-adds of the step),
    one fp32 ulp of magnitude per multiply-add."""
    import numpy as np
    f = lambda x: float(np.float32(x))          # noqa: E731
    lr, m, wd, od = f(lr), f(momentum), f(weight_decay), f(np.float32(1.0) - np.float32(dampening))
    d = grad.double() + wd * w.double()
    dmag = grad.double().abs() + wd * w.double().abs()
    d_err = _ulp32(dmag)
    b = None
    if m != 0.0:
        if fresh:                               # b = d: the rounding of d is the buffer's one ulp
            b, bmag, b_carry = d, dmag, 0.0 * d_err
        else:
            b = m * buf.double() + od * d
            bmag = m * buf.double().abs() + od * dmag
            b_carry = od * d_err
        b_err = _ulp32(bmag) + b_carry
        if nesterov:
            step, s_err = d + m * b, _ulp32(dmag + m * b.abs()) + d_err + m * b_err
        else:
            step, s_err = b, b_err
    else:
        step, s_err = d, d_err
    p = w.double() - lr * step
    out = (p, w.double().abs() + lr * step.abs(), lr * s_err)
    return out, ((b, bmag, b_carry) if b is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("cfg", ["reference", "no_momentum", "nesterov", "dampening_late_param"])
def test_fused_sgd_against_float64_over_the_parameter_table(cfg, arch):
    """FusedSGD over the architecture's parameters plus one of one chunk and one of a chunk + 3 elements, step by
    step from the kernel's own previous state. dampening_late_param: one parameter gets its first gradient at step 2,
    when the others already hold momentum buffers; like torch.optim.SGD its buffer must start at that gradient."""
    torch, raw = _torch()
    from b200seg.module import B200SegModule
    from b200seg.optim import FusedSGD
    torch.manual_seed(0)
    net = B200SegModule(arch, 19)
    chunk = raw.lib().b200seg_sgd_chunk()
    ps = [p.detach().clone().cuda().requires_grad_(True) for p in net.parameters()]
    ps += [torch.randn(chunk, device="cuda").requires_grad_(True), torch.randn(chunk + 3, device="cuda").requires_grad_(True)]
    hp = dict(reference=dict(lr=0.01, momentum=0.9, weight_decay=1e-4),
              no_momentum=dict(lr=0.01, momentum=0.0, weight_decay=1e-4),
              nesterov=dict(lr=0.01, momentum=0.9, weight_decay=1e-4, nesterov=True),
              dampening_late_param=dict(lr=0.01, momentum=0.9, dampening=0.5, weight_decay=1e-4))[cfg]
    lr, mom, damp, wd, nest = hp["lr"], hp["momentum"], hp.get("dampening", 0.0), hp["weight_decay"], hp.get("nesterov", False)
    opt = FusedSGD(ps, **hp)
    late = ps[-1] if cfg == "dampening_late_param" else None
    g = torch.Generator(device="cuda").manual_seed(2)
    seen = set()
    for step in range(4):
        for p in ps:
            p.grad = None if (p is late and step == 0) else torch.randn(p.shape, generator=g, device="cuda")
        live = [p for p in ps if p.grad is not None]
        before = {id(p): (p.detach().clone(), opt.state[p]["momentum_buffer"].clone()
                          if "momentum_buffer" in opt.state.get(p, {}) else None) for p in live}
        opt.step()
        torch.cuda.synchronize()
        for k, p in enumerate(live):
            p0, b0 = before[id(p)]
            fresh = id(p) not in seen
            (r, rmag, r_carry), bref = _sgd_reference(p0, p.grad, b0, lr, mom, damp, wd, nest, fresh)
            what = "%s %s step %d parameter %d (%s)" % (arch, cfg, step, k, tuple(p.shape))
            if bref is not None:
                b, bmag, b_carry = bref
                _within_ulp(opt.state[p]["momentum_buffer"], b, bmag, what + " buffer", b_carry)
            _within_ulp(p.detach(), r, rmag, what, r_carry)
            seen.add(id(p))
