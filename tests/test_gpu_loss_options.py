"""Op-level parity of the two loss options through the C ABI: the image-weighted cross-entropy of --img_wt_loss
(ImageBasedCrossEntropyLoss2d, loss/utils.py:70-118) and RMI on the OCR auxiliary head (--ocr_aux_loss_rmi,
network/ocrnet.py:116,302-303).

Class counts are compared exactly with torch.bincount and the class weights bit for bit with an fp32 restatement.
Losses and logit gradients are compared with float64 autograd on the same fp32 logits: 2e-5 relative on the
cross-entropy loss, 1e-4 on RMI, 2^-7 of the tensor scale on bf16 gradients (2^-6 where RMI adds its fp64 solve).
Every launch runs twice and must give identical bits."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

TOL = 2.0 ** -7


def _raw():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from b200seg import raw
    return raw


def close(a, b, tol, what=""):
    a, b = a.double(), b.double()
    scale = b.abs().max().item() + 1e-12
    err = (a - b).abs().max().item()
    assert err <= tol * scale, "%s max err %.3e vs scale %.3e (tol %.1e)" % (what, err, scale, tol)


def _labels(case, n=2, H=64, W=96, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gts = torch.randint(0, 19, (n, H, W), generator=g, device="cuda")
    gts[:, :5] = 255
    gts[0, 20:40, 30:70] = 3
    if case == "mixed":          # image 1: classes 0-4 only, class 18 absent from the whole batch
        gts[1] = torch.where(gts[1] != 255, gts[1] % 5, gts[1])
        gts[0] = torch.where(gts[0] == 18, torch.full_like(gts[0], 17), gts[0])
    elif case == "full":         # one class fills the whole crop of image 1
        gts[1] = 7
    elif case == "empty":        # image 1 has no valid pixel
        gts[1] = 255
    return gts


def _restated_weights(gts, ub, half):
    import _img_wt_oracle as W
    w = W.img_wt_class_weights(gts, ub)
    return w.half().float() if half else w


@pytest.mark.parametrize("case", ["mixed", "full", "empty"])
@pytest.mark.parametrize("ub,half", [(1.0, False), (2.5, False), (2.5, True), (1.3, True)])
def test_label_histogram_and_class_weights(case, ub, half):
    raw = _raw()
    gts = _labels(case)
    n = gts.shape[0]
    outs = [raw.label_class_weights(gts, ub, half) for _ in range(2)]
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))       # bits: the empty case holds NaN
    counts, weights, coef, scale = outs[0]
    for i in range(n):
        ref = torch.bincount(gts[i][gts[i] < 19], minlength=19)
        assert torch.equal(counts[i].long(), ref), i
    want = _restated_weights(gts, ub, half)
    assert torch.equal(weights.view(torch.int32), want.view(torch.int32)), (weights, want)
    den = (want.double()[None] * counts.double()).sum(1)
    for i in range(n):
        if den[i] == 0:
            assert torch.isnan(coef[i]).all()
        else:
            close(coef[i], want.double() / den[i], 1e-7, "coef")
    assert math.isnan(float(scale)) == (case == "empty")
    if case != "empty":
        assert float(scale) == 1.0


def _setup(two_scale, n=2, H=64, W=96):
    hq, wq = H // 4, W // 4
    hm, wm, hl, wl = (H // 2, W // 2, H // 8, W // 8) if two_scale else (0, 0, 0, 0)
    g = torch.Generator(device="cuda").manual_seed(1)
    mk = lambda *s: torch.randn(s, generator=g, device="cuda")
    t = dict(hi_cls=torch.zeros((n, hq, wq, 20), device="cuda"), hi_aux=torch.zeros((n, hq, wq, 20), device="cuda"))
    t["hi_cls"][..., :19], t["hi_aux"][..., :19] = mk(n, hq, wq, 19) * 2, mk(n, hq, wq, 19) * 2
    if two_scale:
        t["lo_cls"], t["lo_aux"] = torch.zeros((n, hl, wl, 20), device="cuda"), torch.zeros((n, hl, wl, 20), device="cuda")
        t["lo_cls"][..., :19], t["lo_aux"][..., :19] = mk(n, hl, wl, 19) * 2, mk(n, hl, wl, 19) * 2
        t["lo_attn"] = mk(n, hl, wl, 1).contiguous()
    return (hq, wq, hm, wm, hl, wl), t


def _fp64_graph(t, two_scale, H, W):
    """Leaves (float64, NCHW) and the blended predictions of MscaleOCR.two_scale_forward / OCRNet.forward."""
    nchw = lambda x: x.permute(0, 3, 1, 2).contiguous().double().requires_grad_(True)
    up = lambda x, size: F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    leaves = [nchw(t["hi_cls"][..., :19]), nchw(t["hi_aux"][..., :19])]
    if not two_scale:
        return leaves, dict(joint=up(leaves[0], (H, W)), joint_aux=up(leaves[1], (H, W)))
    hm, wm = H // 2, W // 2
    leaves += [nchw(t["lo_cls"][..., :19]), nchw(t["lo_aux"][..., :19]), nchw(t["lo_attn"])]
    a = up(torch.sigmoid(leaves[4]), (hm, wm))
    a_up = up(a, (H, W))
    lo_up = up(leaves[2], (hm, wm))
    return leaves, dict(joint=up(a * lo_up, (H, W)) + (1 - a_up) * up(leaves[0], (H, W)),
                        joint_aux=up(a * up(leaves[3], (hm, wm)), (H, W)) + (1 - a_up) * up(leaves[1], (H, W)),
                        sup_lo=up(lo_up, (H, W)), sup_hi=up(leaves[0], (H, W)))


def _run_twice(fn):
    a, b = fn(), fn()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                               y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))
    return a


def _check_grads(raw, d, t, leaves, g_hi, g_lo, g_sup, two_scale, tol, tag):
    d_cls, d_aux = _run_twice(lambda: raw.mscale_hi_bwd(d, g_hi))
    close(d_cls[..., :19], leaves[0].grad.permute(0, 2, 3, 1), tol, "d hi cls " + tag)
    close(d_aux[..., :19], leaves[1].grad.permute(0, 2, 3, 1), tol, "d hi aux " + tag)
    outs = [d_cls, d_aux]
    if two_scale:
        dl = _run_twice(lambda: raw.mscale_lo_bwd(d, g_lo, g_sup, t["lo_cls"], t["lo_aux"], t["lo_attn"], t["mid"]))
        for k, (got, leaf) in enumerate(zip(dl, leaves[2:])):
            close(got[..., :leaf.shape[1]], leaf.grad.permute(0, 2, 3, 1), tol, "d lo %d %s" % (k, tag))
        outs += list(dl)
    return outs


@pytest.mark.parametrize("case", ["mixed", "full", "empty"])
@pytest.mark.parametrize("two_scale,sup,ub,half", [(True, 0.0, 2.5, False), (True, 0.05, 1.0, True),
                                                   (False, 0.0, 2.0, True)])
def test_image_weighted_ce_fwd_bwd(case, two_scale, sup, ub, half):
    import _img_wt_oracle
    raw = _raw()
    n, H, W = 2, 64, 96
    (hq, wq, hm, wm, hl, wl), t = _setup(two_scale, n, H, W)
    gts = _labels(case, n, H, W)
    d = raw.mscale_desc(n, H, W, hq, wq, hm, wm, hl, wl, 2, 1.0, 0.4, sup)
    leaves, p = _fp64_graph(t, two_scale, H, W)
    crit = _img_wt_oracle.criterion_img_wt(upper_bound=ub, batch_weights=False, fp16=half)
    ref = 0.4 * crit(p["joint_aux"], gts) + crit(p["joint"], gts)
    if sup:
        ref = ref + sup * crit(p["sup_lo"], gts) + sup * crit(p["sup_hi"], gts)
    ref.backward()
    t["mid"], mid_sup = raw.mscale_mid_fwd(d, t["lo_cls"], t["lo_aux"], t["lo_attn"]) if two_scale else (None, None)
    _, _, coef, scale = raw.label_class_weights(gts, ub, half)
    loss, g_hi, g_lo, g_sup = _run_twice(lambda: raw.mscale_loss_fwd(d, gts, scale, t["hi_cls"], t["hi_aux"], t["mid"],
                                                                     mid_sup, class_coef=coef))
    if case == "empty":
        assert math.isnan(float(loss[0])) and math.isnan(float(ref))
    else:
        assert abs(float(loss[0]) - float(ref)) <= 2e-5 * abs(float(ref)), (float(loss[0]), float(ref))
    outs = _check_grads(raw, d, t, leaves, g_hi, g_lo, g_sup, two_scale, TOL, "img_wt")
    if case == "empty":
        for o in outs:
            assert float(o[1].float().abs().max()) == 0.0          # the all-ignored image gets no gradient
            assert float(o[0].float().abs().max()) > 0.0


@pytest.mark.parametrize("two_scale,sup", [(True, 0.0), (True, 0.05), (False, 0.0)])
def test_rmi_on_auxiliary_head_fwd_bwd(two_scale, sup):
    """RMILoss with cfg.LOSS.OCR_AUX_RMI: the auxiliary term is 0.4 * (0.5 BCE + 0.5 RMI) of joint_aux."""
    from oracle import seg_oracle as O
    raw = _raw()
    n, H, W = 2, 64, 96
    (hq, wq, hm, wm, hl, wl), t = _setup(two_scale, n, H, W)
    gts = _labels("mixed", n, H, W)
    d = raw.mscale_desc(n, H, W, hq, wq, hm, wm, hl, wl, 2, 1.0, 0.4, sup, loss_kind=1)
    leaves, p = _fp64_graph(t, two_scale, H, W)
    crit = lambda x, do_rmi: O.rmi_loss(x, gts, do_rmi=do_rmi)
    ref = 0.4 * crit(p["joint_aux"], True) + crit(p["joint"], True)
    if sup:
        ref = ref + sup * crit(p["sup_lo"], False) + sup * crit(p["sup_hi"], False)
    ref.backward()
    with torch.no_grad():
        ja = p["joint_aux"].detach()
        aux_rmi_ref = 0.4 * (O.rmi_loss(ja, gts, do_rmi=True) - 0.5 * O.rmi_loss(ja, gts, do_rmi=False))
    t["mid"], mid_sup = raw.mscale_mid_fwd(d, t["lo_cls"], t["lo_aux"], t["lo_attn"]) if two_scale else (None, None)
    inv = raw.count_valid(gts, plus_one=True)

    def fwd():
        pr, la = raw.rmi_pool(d, gts, t["hi_cls"], t["mid"])
        pr_aux = raw.rmi_pool_aux(d, gts, t["hi_aux"], t["mid"])
        dpr, terms = raw.rmi_solve_grad(d, pr, la, d.w_head0)
        dpr_aux, terms_aux = raw.rmi_solve_grad(d, pr_aux, la, d.w_head1)
        out = raw.mscale_loss_fwd(d, gts, inv, t["hi_cls"], t["hi_aux"], t["mid"], mid_sup, dpr, terms,
                                  rmi_dpr_aux=dpr_aux, rmi_terms_aux=terms_aux)
        return (pr_aux, dpr_aux, terms_aux) + tuple(out)

    _, _, _, loss, g_hi, g_lo, g_sup = _run_twice(fwd)
    assert abs(float(loss[6]) - float(aux_rmi_ref)) <= 1e-4 * abs(float(aux_rmi_ref)) + 1e-6, \
        (float(loss[6]), float(aux_rmi_ref))
    assert abs(float(loss[0]) - float(ref)) <= 1e-4 * abs(float(ref)), (float(loss[0]), float(ref))
    _check_grads(raw, d, t, leaves, g_hi, g_lo, g_sup, two_scale, 2 * TOL, "aux rmi")


def test_loss_fwd_ex_without_options_equals_loss_fwd():
    """b200seg_mscale_loss_fwd_ex with no option is b200seg_mscale_loss_fwd, bit for bit."""
    import ctypes
    from b200seg import _lib
    raw = _raw()
    n, H, W = 2, 64, 96
    (hq, wq, hm, wm, hl, wl), t = _setup(True, n, H, W)
    gts = _labels("mixed", n, H, W)
    d = raw.mscale_desc(n, H, W, hq, wq, hm, wm, hl, wl, 2, 1.0, 0.4, 0.05)
    mid, mid_sup = raw.mscale_mid_fwd(d, t["lo_cls"], t["lo_aux"], t["lo_attn"])
    inv = raw.count_valid(gts)
    loss, g_hi, g_lo, g_sup = raw.mscale_loss_fwd(d, gts, inv, t["hi_cls"], t["hi_aux"], mid, mid_sup)
    L = _lib.lib()
    nb = L.b200seg_mscale_loss_blocks(ctypes.byref(d))
    bufs = [torch.empty_like(x) for x in (g_hi, g_lo, g_sup)]
    ws, loss2 = torch.empty(nb * 4, device="cuda"), torch.zeros(8, device="cuda")
    p = raw.ptr
    rc = L.b200seg_mscale_loss_fwd_ex(ctypes.byref(d), p(gts), p(inv), None, p(t["hi_cls"]), p(t["hi_aux"]), p(mid),
                                      p(mid_sup), p(bufs[0]), p(bufs[1]), p(bufs[2]), p(ws), p(loss2), None, None, 0,
                                      None, None, 0, raw.stream_ptr())
    assert rc == 0
    assert torch.equal(loss, loss2)
    for a, b in zip((g_hi, g_lo, g_sup), bufs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
