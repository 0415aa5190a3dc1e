"""The plane-ordered weight image of the halo-tile convolution (include/b200seg.h, b200seg_conv2d_planes_elems).

The image only changes where the kernel's producer copies the weights from: the same bytes land at the same shared-memory
addresses and the MMAs, tiling and summation order stay those of the TMA path. So every launch must give bitwise the same
outputs and statistics with and without the image, and the plan query must not depend on it.

  * host only: the plan of every halo configuration key of the traced programs is the same with the image set and unset;
    a misaligned or undersized image is refused;
  * GPU: the pack launch writes the image as a PyTorch restatement of the layout (forward and data gradient, padded
    rows and channels zero); every halo configuration key of tests/test_gpu_conv_classes.py runs bitwise identically
    with and without it (forward with statistics, forward with the affine epilogue, data gradient, both shared-memory
    reserves); a W16 two-scale training step with images equals the one without, bit for bit."""
import ctypes

import pytest
import torch

from b200seg import _lib
import test_gpu_conv_classes as classes

E_BADARG = -1
HALO_CASES = [c for c in classes.CASES if c[0] in ("fwd", "dgrad") and c[3][0] == "halo"]


def _plan(d, which):
    out = (ctypes.c_int32 * 13)()
    assert _lib.lib().b200seg_conv2d_plan_info(ctypes.byref(d), which | _lib.PLAN_WINDOW, out) == 0
    return list(out)


def _rows(d, which):
    rows = ctypes.c_int32(0)
    n = _lib.lib().b200seg_conv2d_planes_elems(ctypes.byref(d), which, ctypes.byref(rows))
    return n, rows.value


def test_halo_cases_exist():
    assert len(HALO_CASES) >= 20


@pytest.mark.parametrize("case", HALO_CASES, ids=classes._case_id)
def test_plan_query_ignores_the_image(case):
    entry, shape, res, _key = case
    which = 0 if entry == "fwd" else 1
    with classes.smem_reserve(res):
        d = classes._desc(shape, emit_stats=int(entry == "fwd"))
        n, rows = _rows(d, which)
        assert n > 0 and rows > 0
        plain = _plan(d, which)
        d.w_planes, d.w_planes_rows = 4096, rows
        assert _plan(d, which) == plain
        # the widest tiling of the plan fits the image's rows
        assert plain[1] * plain[2] <= rows


def test_image_only_for_halo_launches():
    d = classes._desc((1, 64, 64, 96, 96, 3, 2))          # stride 2: per-tap kernel
    assert _rows(d, 0) == (0, 0)
    d = classes._desc((1, 64, 64, 96, 96, 1, 1))          # 1x1
    assert _rows(d, 0) == (0, 0)
    d = classes._desc((1, 64, 64, 720, 512, 3, 1))
    n, rows = _rows(d, 0)
    assert rows >= 512 and n == 9 * 720 * rows
    n, rows = _rows(d, 1)                                  # data gradient: Cout 720, Cin 512
    assert rows >= 720 and n == 9 * 512 * rows


def test_misaligned_or_undersized_image_is_refused():
    L = _lib.lib()
    d = classes._desc((1, 256, 512, 720, 512, 3, 1))
    _n, rows = _rows(d, 0)
    fake = 1 << 20            # refused before anything is read or launched
    for ptr, r in ((fake + 8, rows), (fake, 256)):
        d.w_planes, d.w_planes_rows = ptr, r
        assert L.b200seg_conv2d_fwd(ctypes.byref(d), fake, fake, None, fake, None, None, None) == E_BADARG
        dd = classes._desc((1, 256, 512, 720, 512, 3, 1))
        _n, rows_d = _rows(dd, 1)
        dd.w_planes, dd.w_planes_rows = ptr, (rows_d if r == rows else 256)
        assert L.b200seg_conv2d_dgrad(ctypes.byref(dd), fake, 512, fake, None, 0, fake, 720, None) == E_BADARG


# ------------------------------------------------------------------------------------------------------------ GPU part
def _restate(w, rows_f, rows_d):
    """PyTorch restatement of both images of an OIHW fp32 3x3 weight."""
    o, i, _, _ = w.shape
    wb = w.to(torch.bfloat16)
    w_f = wb.permute(0, 2, 3, 1).reshape(o, 9, i)                       # [O][9][I]
    o8 = (o + 7) // 8 * 8
    w_d = torch.zeros((i, 9, o8), dtype=torch.bfloat16, device=w.device)
    w_d[:, :, :o] = wb.permute(1, 2, 3, 0).reshape(i, 9, o).flip(1)      # [I][9 flipped][O up to 8]
    img_f = torch.zeros((9, (i + 15) // 16 * 2, rows_f, 8), dtype=torch.bfloat16, device=w.device)
    img_f[:, :i // 8, :o] = w_f.view(o, 9, i // 8, 8).permute(1, 2, 0, 3)
    img_d = torch.zeros((9, (o8 + 15) // 16 * 2, rows_d, 8), dtype=torch.bfloat16, device=w.device)
    img_d[:, :o8 // 8, :i] = w_d.view(i, 9, o8 // 8, 8).permute(1, 2, 0, 3)
    return w_f, w_d, img_f, img_d


def _packed(w):
    """(w_f, w_d, image fwd, image dgrad) of an OIHW fp32 3x3 weight through the model's single pack launch."""
    from b200seg import raw
    o, i, _, _ = w.shape
    w_f = torch.zeros((o, 9, i), dtype=torch.bfloat16, device="cuda")
    w_d = torch.zeros((i, 9, (o + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")
    img_f, img_d = raw.planes_image(w.shape, 0, "cuda"), raw.planes_image(w.shape, 1, "cuda")
    raw.pack_weights(raw.pack_table([(w, w_f, w_d, img_f, img_d)], "cuda"), 3)
    return w_f, w_d, img_f, img_d


@pytest.mark.gpu
@pytest.mark.parametrize("o,i", [(48, 48), (96, 96), (192, 192), (384, 384), (256, 512), (512, 720), (720, 512),
                                 (24, 256), (96, 48)])
def test_pack_writes_the_image_layout(o, i):
    g = torch.Generator(device="cuda").manual_seed(o * 1000 + i)
    w = torch.randn((o, i, 3, 3), device="cuda", generator=g)
    w_f, w_d, img_f, img_d = _packed(w)
    assert (img_f is None) == (o % 16 != 0)
    ref_f, ref_d, ref_img_f, ref_img_d = _restate(w, img_f.shape[2] if img_f is not None else (o + 15) // 16 * 16,
                                                  img_d.shape[2] if img_d is not None else (i + 15) // 16 * 16)
    assert torch.equal(w_f, ref_f) and torch.equal(w_d, ref_d)
    if img_f is not None:
        assert torch.equal(img_f.view(torch.int16), ref_img_f.view(torch.int16))
    if img_d is not None:
        assert torch.equal(img_d.view(torch.int16), ref_img_d.view(torch.int16))
    if img_f is None:
        return
    # one pack table item with images next to one without: the latter's operands are still written
    from b200seg import raw
    w2 = torch.randn((32, 16, 3, 3), device="cuda", generator=g)
    f2 = torch.zeros((32, 9, 16), dtype=torch.bfloat16, device="cuda")
    d2 = torch.zeros((16, 9, 32), dtype=torch.bfloat16, device="cuda")
    img_f[:] = 0
    raw.pack_weights(raw.pack_table([(w, w_f, w_d, img_f, None), (w2, f2, d2)], "cuda"), 1)
    assert torch.equal(img_f.view(torch.int16), ref_img_f.view(torch.int16))
    assert torch.equal(f2, _restate(w2, 32, 16)[0])


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("case", HALO_CASES, ids=classes._case_id)
def test_outputs_identical_with_and_without_image(case):
    from b200seg import raw
    entry, shape, res, _key = case
    n, h, w, cin, cout, k, s, _dil = classes._shape8(shape)
    g = torch.Generator(device="cuda").manual_seed(classes._seed(case))
    wt = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5
    w_f, w_d, img_f, img_d = _packed(wt)
    with classes.smem_reserve(res):
        if entry == "fwd":
            x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(torch.bfloat16)
            outs = []
            for img in (None, img_f):
                y, (st, grid, cpad) = raw.conv2d_fwd(x, w_f, emit_stats=True, planes=img)
                scale = torch.rand(cout, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) + 0.5
                shift = torch.linspace(-0.1, 0.1, cout, device="cuda")
                z = raw.conv2d_fwd_affine(x, w_f, scale, shift, True, addend=y, planes=img)
                torch.cuda.synchronize()
                outs.append((y, st[:grid * 2 * cpad], z))
            for a, b, what in zip(outs[0], outs[1], ("output", "statistics partials", "affine output")):
                assert torch.equal(_bits(a), _bits(b)), what
        else:
            cpad = (cout + 7) // 8 * 8
            dy = torch.zeros((n, h, w, cpad), device="cuda", dtype=torch.bfloat16)
            dy[..., :cout] = torch.randn((n, h, w, cout), device="cuda", generator=g).to(torch.bfloat16)
            add = torch.randn((n, h, w, cin), device="cuda", generator=g).to(torch.bfloat16)
            outs = []
            for img in (None, img_d):
                dx = raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), 3, 1, planes=img)
                dx2 = add.clone()
                raw.conv2d_dgrad(dy, w_d, (n, h, w, cin), 3, 1, addend=dx2, out=dx2, planes=img)
                torch.cuda.synchronize()
                outs.append((dx, dx2))
            for a, b, what in zip(outs[0], outs[1], ("data gradient", "accumulated data gradient")):
                assert torch.equal(_bits(a), _bits(b)), what


@pytest.mark.gpu
def test_two_scale_step_identical_with_and_without_images(monkeypatch):
    """ocrnet.HRNet_Mscale, W16 test widths: two eager SGD steps with the images equal those without, bitwise."""
    from oracle import seg_oracle as O
    from b200seg import raw
    from b200seg.module import B200SegModule
    hcfg = O.HRNET_W16_TEST
    arch = "ocrnet.HRNet_Mscale"
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0
    results = []
    planes_image = raw.planes_image
    for with_images in (True, False):
        monkeypatch.setattr(raw, "planes_image", planes_image if with_images else (lambda *a, **k: None))
        net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=False)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
        losses = []
        for step in range(2):
            images, gts = O.synth_batch(2, 64, 128, seed=100 + step)
            opt.zero_grad()
            loss = net({"images": images.cuda(), "gts": gts.cuda()})
            loss.backward()
            opt.step()
            losses.append(loss.detach().clone())
        assert bool(net._planes) == with_images
        results.append((losses, {n: p.grad.clone() for n, p in net.named_parameters()},
                        {n: p.detach().clone() for n, p in net.named_parameters()}))
    (l0, g0, p0), (l1, g1, p1) = results
    assert all(torch.equal(a, b) for a, b in zip(l0, l1)), (l0, l1)
    assert all(torch.equal(g0[n], g1[n]) for n in g0), [n for n in g0 if not torch.equal(g0[n], g1[n])][:5]
    assert all(torch.equal(p0[n], p1[n]) for n in p0)
