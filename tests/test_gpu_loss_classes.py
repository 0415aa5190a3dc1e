"""Every configuration of the loss launches of the training step (tools/loss_classes.py) checked against float64.

ROWS holds, per configuration key the traced training steps reach (every architecture under CE, RMI and the
image-weighted CE with and without binary16 weights, the two-scale architectures with supervision, RMI on the OCR
auxiliary head), the smallest shape found that keeps the key: a launch of one C ABI entry point with its arguments in
ABI order, PTR marking the operands that are present; an optional third element names the data of an edge row.
tests/test_loss_plans.py checks on the CPU that the rows cover every key of the programs. Edge rows no traced program
reaches follow: a batch whose labels are all ignored (CE loss NaN like the reference's 0/0), an image without a valid
pixel under the image-weighted CE (loss_scale NaN), non-integer ratios at every level, the smallest RMI crop (12x12:
most of the 48 moment chunks are empty), RMI crops with H % 4 = 1, 2 and 3, a crop labelled with one class (zero label
covariance) and logits near +-30 (saturated softmax and BCE).

Every reference is computed in float64 from exactly the inputs the kernel read (A = the same operation on |inputs|,
the interpolation matrices are test_gpu_ew_classes._interp, PyTorch's align_corners=False rule):
  * count_valid: the count exactly, inv_count bit for bit against fp32 1 / float32(count [+ 1]);
  * label_class_weights: counts exactly, weights bit for bit against the fp32 restatement of tests/_img_wt_oracle.py,
    coef bit for bit against one rounding of the float64 w / sum_c w[c] count[c]. That denominator is exact in float64:
    every w is an fp32 value in [1, upper_bound + 1], hence a multiple of 2^-23, so every product and partial sum of
    w[c] count[c] is a multiple of 2^-23 below (upper_bound + 1) N for an image of N pixels: an integer number of
    2^-23 units below 2^53 while (upper_bound + 1) N < 2^30 (300M pixels at upper_bound 2.5), which fp64 holds exactly;
    loss_scale is 1, or NaN for a batch with an image without a valid pixel;
  * mscale_mid_fwd: sigmoid and interpolation in float64, |out - r| <= EW_REL * A;
  * mscale_loss_fwd(_ex) (plain, weighted and auxiliary-RMI instantiations): the joint logits, log-softmax / BCE terms
    and gradient rows Ghi, Glo and Gsup from the kernel's fp32 hi, mid, mid_sup, class_coef and rmi_dpr; bf16 rows
    follow the bf16 rules of test_gpu_ew_classes (one ulp plus EW_REL * A, a cap on the share of mismatches); the
    gradient channels of ignored pixels are exactly 0; loss_out[0..6] within STAT_REL of the sum of magnitudes;
  * mscale_hi_bwd, mscale_lo_bwd (dmid_ws of mid_bwd included): the transposed float64 interpolation matrices applied to
    the kernel's own bf16 gradient rows, the product rule and sigmoid' in float64; lo_bwd's second stage reads the
    kernel's own dmid_ws;
  * rmi_pool(_aux): float64 average pooling (4 / 4, pad 2, divisor 16) of sigmoid(joint) * mask + 1e-6 and
    onehot * mask;
  * rmi_solve_grad: rmi_lower_bound (loss/rmi.py) restated in float64 from the kernel's pooled maps, rmi_terms and dpr
    by autograd; the restatement is pinned to oracle.seg_oracle.rmi_loss once (test_rmi_restatement_matches_oracle).
    Bound: the fp32 rounding of the output plus RMI_ALLOW of the largest |reference| of the tensor, for the fp64 solve
    of an ill-conditioned system (G ~ 1 / alpha).
Outputs go into a NaN-filled buffer with a NaN guard behind it: nothing outside the output may change and everything in
it must be finite (partial_ws, dmid_ws, the RMI workspace and G included, and the zero padding: channels 19..31 of d_cls
/ d_aux, the auxiliary half of the mid rows with one head, channel 39). Unused input channels hold NaN. Every launch runs
twice and must give the same bits.

Largest values observed on one H100 80GB HBM3 (700 W power limit) over the 85 rows, which run in 17 s there
(headroom = bound / observed):
  |out - r| / (ulp_bf16(r) + EW_REL * A), every bf16 output   0.4998 (2x: the bf16 rounding itself)
  fp32 arithmetic error / A (EW_REL 2^-18 = 3.8e-6)          loss_fwd Ghi 9.7e-7 (3.9x), mid_fwd 3.0e-7, rmi_pool
                                                              2.9e-7, Glo 2.6e-7, lo_bwd 1.1e-7, mid_bwd 1.0e-7 (13x and
                                                              more), hi_bwd 1.2e-8
  share of bf16 outputs != round_bf16(r)                      0.021 % (Glo of the saturated auxiliary-RMI row, 47x)
  loss_out / sum of magnitudes (STAT_REL 1e-5)                5.4e-8 (186x)
  RMI fp64 allowance (RMI_ALLOW 2^-20 = 9.5e-7)               dpr 3.4e-7 of its largest value (2.8x) on the 12x12 crop,
                                                              where 4 positions estimate a 9 x 9 covariance and the
                                                              alpha = 5e-4 regularisation makes G ~ 1 / alpha; rmi_terms
                                                              are the fp32 rounding of the reference on every row
The 20 composed rows (test_composed_loss_step_against_float64_autograd, one per geometry and criterion, described above
their runner) on the same card: err / bound 0.485 (2.1x; the attention logit 0.196), loss 1.2e-7 of its value (170x).

Substituted kernel errors, each built into the library in turn and run against this file on the H100 (rows failed of
the 85 per-launch rows + of the 20 composed rows):
  hi_bwd_kernel reading head 1 from acc[c + 2]                 3 + 8  (every two-head hi_bwd row and composed row)
  loss_finalize_kernel skipping the last partial block         36 + 20
  rmi_moments_kernel dropping its last chunk                   6 + 8
  mid_bwd_kernel dropping the supervised dS term               4 + 10 (every supervised lo_bwd row)
  lo_bwd_kernel applying s * s instead of s * (1 - s)          7 + 10 (every lo_bwd row)
  adj_range's upper bound one fine pixel short                 14 + 20
  sgd_step_kernel using first_step for every block             24 of the 32 FusedSGD rows of tests/test_gpu_bookkeeping.py
                                                               (all but momentum 0, where no buffer is read)
"""
import ctypes
import math
import zlib

import pytest

import test_gpu_ew_classes as ew
from test_gpu_ew_classes import Buf, PTR, EW_REL, STAT_REL, _interp, _resample, _twice, _note

RMI_ALLOW = 2.0 ** -20
NC = 19
IGN = 255


# ------------------------------------------------------------------------------------------------------------ rows
def ms(n, h, w, hq, wq, hm=0, wm=0, hl=0, wl=0, nheads=1, sup_wt=0.0, kind=0):
    return ("ms", n, h, w, hq, wq, hm, wm, hl, wl, nheads, float(sup_wt), IGN, kind)


def geo(n, h, w, rh, rl=None, nheads=1, sup=False, kind=0):
    """One scale (rl None) or two: mid grid H / 2, lo maps at mid / rl."""
    if rl is None:
        return ms(n, h, w, h // rh, w // rh, nheads=nheads, kind=kind)
    hm, wm = h // 2, w // 2
    return ms(n, h, w, h // rh, w // rh, hm, wm, hm // rl, wm // rl, nheads, 0.05 if sup else 0.0, kind)


def _p(x):
    return PTR if x else None


def loss_fwd_row(d, variant="plain", case=None):
    """variant plain | wt | aux_rmi; the RMI terms are present with loss_kind 1."""
    two, sup, heads, rmi = d[6] > 0, d[11] != 0.0, d[10], d[13] == 1
    common = (_p(heads > 1), _p(two), _p(two and sup), PTR, _p(two), _p(two and sup), PTR, PTR, _p(rmi), _p(rmi),
              d[1] * NC if rmi else 0)
    if variant == "plain":
        row = ("mscale_loss_fwd", (d, PTR, PTR, PTR) + common + (0,))
    else:
        aux = variant == "aux_rmi"
        row = ("mscale_loss_fwd_ex", (d, PTR, PTR, _p(variant == "wt"), PTR) + common +
               (_p(aux), _p(aux), d[1] * NC if aux else 0, 0))
    return row + ((case,) if case else ())


def mid_fwd_row(d):
    return ("mscale_mid_fwd", (d, PTR, _p(d[10] > 1), PTR, PTR, _p(d[11] != 0.0), 0))


def hi_bwd_row(d):
    return ("mscale_hi_bwd", (d, PTR, PTR, _p(d[10] > 1), 0))


def lo_bwd_row(d):
    two = d[10] > 1
    return ("mscale_lo_bwd", (d, PTR, _p(d[11] != 0.0), PTR, _p(two), PTR, PTR, PTR, PTR, _p(two), PTR, 0))


def rmi_pool_row(d, aux=False):
    if aux:
        return ("rmi_pool_aux", (d, PTR, PTR, _p(d[6] > 0), PTR, 0))
    return ("rmi_pool", (d, PTR, PTR, _p(d[6] > 0), PTR, PTR, 0))


def rmi_solve_row(n, h, w, case=None):
    row = ("rmi_solve_grad", (n, h, w, PTR, PTR, 0.5 / (n * 9.0), PTR, 0, PTR, PTR, PTR, 0))
    return row + ((case,) if case else ())


def _loss_rows():
    rows = []
    # traced: every (hi ratio, mid / lo ratio, heads) of the eight architectures; loss_fwd on a capped grid
    archs = [(4, 4, 2), (4, None, 2), (4, None, 1), (4, 4, 1), (2, None, 1), (2, 2, 1)]
    for rh, rl, heads in archs:
        for sup in ((False, True) if rl else (False,)):
            d_ce = geo(1, 512, 544, rh, rl, heads, sup)
            d_rmi = geo(1, 512, 544, rh, rl, heads, sup, kind=1)
            rows += [loss_fwd_row(d_ce), loss_fwd_row(d_rmi), loss_fwd_row(d_ce, "wt")]
            if heads > 1:
                rows.append(loss_fwd_row(d_rmi, "aux_rmi"))
            if rl:
                rows.append(mid_fwd_row(geo(1, 64, 96, rh, rl, heads, sup)))
                rows.append(lo_bwd_row(geo(1, 1040, 1040, rh, rl, heads, sup)))
        rows.append(hi_bwd_row(geo(1, 1040, 1040, rh, rl, heads) if rh == 2 else geo(1, 64, 96, rh, rl, heads)))
        rows.append(rmi_pool_row(geo(1, 48, 64, rh, rl, heads, kind=1)))
        if heads > 1:
            rows.append(rmi_pool_row(geo(1, 48, 64, rh, rl, heads, kind=1), aux=True))
    rows += [("count_valid", (PTR, 736 * 736, IGN, 0, PTR, PTR, 0)), ("count_valid", (PTR, 736 * 736, IGN, 1, PTR, PTR, 0)),
             ("label_class_weights", (PTR, 1, 1040 * 1040, 1.0, 0, PTR, PTR, PTR, PTR, 0)),
             ("label_class_weights", (PTR, 1, 1040 * 1040, 2.5, 1, PTR, PTR, PTR, PTR, 0)),
             rmi_solve_row(1, 700, 700)]
    # edges
    frac = ms(2, 50, 70, 13, 18, 25, 35, 7, 9, 2, 0.05, 0)
    frac_rmi = frac[:13] + (1,)
    rows += [("count_valid", (PTR, 2 * 40 * 48, IGN, 0, PTR, PTR, 0), "ignored_image"),
             ("label_class_weights", (PTR, 2, 40 * 48, 1.0, 0, PTR, PTR, PTR, PTR, 0), "ignored_image"),
             loss_fwd_row(geo(2, 40, 48, 4, 4, 2, True), "plain", "all_ignored"),
             loss_fwd_row(geo(2, 40, 48, 4, 4, 2, True), "wt", "ignored_image"),
             loss_fwd_row(frac), loss_fwd_row(frac, "wt"), loss_fwd_row(frac_rmi), loss_fwd_row(frac_rmi, "aux_rmi"),
             mid_fwd_row(frac), hi_bwd_row(frac), lo_bwd_row(frac), rmi_pool_row(frac_rmi),
             rmi_pool_row(frac_rmi, aux=True),
             loss_fwd_row(geo(1, 32, 48, 4, 4, 2, True), "plain", "saturated"),
             loss_fwd_row(geo(1, 32, 48, 4, 4, 2, True, kind=1), "aux_rmi", "saturated"),
             rmi_pool_row(ms(1, 12, 12, 3, 3, kind=1)), rmi_solve_row(2, 12, 12)]
    for h in (49, 50, 51):
        rows += [rmi_pool_row(ms(1, h, 52, h // 4, 13, kind=1)), rmi_solve_row(2, h, 52)]
    rows.append(rmi_solve_row(2, 48, 64, "one_class"))
    return rows


ROWS = _loss_rows()


def row_id(row):
    return "%s-%08x%s" % (row[0], zlib.crc32(repr(row[1]).encode()), "-" + row[2] if len(row) > 2 else "")


# ------------------------------------------------------------------------------------------------------- GPU helpers
def _torch():
    import torch
    return torch


def _desc(t):
    from b200seg import _lib
    _m, n, h, w, hq, wq, hm, wm, hl, wl, nheads, sup_wt, ign, kind = t
    d = _lib.MscaleDesc()
    d.n, d.h, d.w, d.hq, d.wq, d.hm, d.wm, d.hl, d.wl = n, h, w, hq, wq, hm, wm, hl, wl
    d.nheads, d.w_head0, d.w_head1, d.sup_wt, d.ignore_index, d.loss_kind = nheads, 1.0, 0.4, sup_wt, ign, kind
    return d


def _rng(row):
    torch = _torch()
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(row_id(row).encode()))


def _case(row):
    return row[2] if len(row) > 2 else None


def _labels(g, n, h, w, case=None, one_class=None):
    torch = _torch()
    lab = torch.randint(0, NC, (n, h, w), generator=g, device="cuda", dtype=torch.int64)
    if one_class is not None:
        lab.fill_(one_class)
    drop = torch.rand((n, h, w), generator=g, device="cuda") < 0.1
    lab = torch.where(drop, torch.full_like(lab, IGN), lab)
    if case == "all_ignored":
        lab.fill_(IGN)
    elif case == "ignored_image":
        lab[-1].fill_(IGN)
    return lab.contiguous()


def _logits(g, rows, width, scale=2.0, case=None):
    """fp32 [rows, width] with NaN in column 19 (and 39) that no kernel may read."""
    torch = _torch()
    x = scale * torch.randn((rows, width), generator=g, device="cuda", dtype=torch.float64)
    if case == "saturated":
        x = 30.0 * torch.sign(x) + 0.5 * x.clamp(-1, 1)
    x = x.float()
    x[:, NC::20] = float("nan")
    return x.contiguous()


def _mid_input(g, rows, case=None):
    """mid rows [rows, 40]: A4 * cls4 (19), A4 * aux4 (19), A4 in (0, 1), NaN."""
    torch = _torch()
    m = _logits(g, rows, 20, case=case).repeat(1, 2)
    m[:, NC:2 * NC] = _logits(g, rows, 20, case=case)[:, :NC]
    m[:, 38] = torch.rand((rows,), generator=g, device="cuda")
    m[:, 39] = float("nan")
    return m.contiguous()


def _bf16_rows(g, rows, width, scale=1e-3):
    torch = _torch()
    return (scale * torch.randn((rows, width), generator=g, device="cuda", dtype=torch.float64)).to(torch.bfloat16)


class DBuf(Buf):
    """float64 output buffer (NaN-filled, checked through its 64-bit pattern)."""

    def check(self, what):
        torch = _torch()
        assert bool(torch.isfinite(self.v).all()), "%s: non-finite or unwritten output element" % what
        nan = torch.full((1,), float("nan"), dtype=torch.float64, device="cuda").view(torch.int64)
        outside = torch.ones(self.flat.shape, dtype=torch.bool, device="cuda")
        rows, ld = self.v.shape[0], self.v.stride(0)
        outside[: rows * ld].view(rows, ld)[:, : self.c] = False
        assert int((self.flat.view(torch.int64)[outside] != nan).sum()) == 0, "%s: written outside" % what


class IBuf(Buf):
    """Integer output buffer: filled with -1 (and a -1 guard) instead of NaN."""

    def __init__(self, rows, c, dtype):
        torch = _torch()
        self.flat = torch.full((rows * c + 4096,), -1, dtype=dtype, device="cuda")
        self.v = self.flat[: rows * c].view(rows, c)
        self.c = c

    def check(self, what):
        assert int((self.flat[self.v.numel():] != -1).sum()) == 0, "%s: written past the output" % what


def _check_f32(out, r, A, what, kind, rel=EW_REL):
    torch = _torch()
    assert bool(torch.isfinite(out).all()), "%s: non-finite output" % what
    e = float(((out.double() - r).abs() / A.clamp_min(1e-300)).max())
    _note(kind + " err/A", e, what)
    assert e <= rel, "%s: error %.3e of A, bound %.1e" % (what, e, rel)


def _ulp32(r):
    torch = _torch()
    _m, e = torch.frexp(r)
    return torch.where(r == 0, torch.zeros_like(r), torch.ldexp(torch.ones_like(r), e - 24))


# --------------------------------------------------------------------------------------------- counts and weights
def _run_count_valid(row):
    import numpy as np
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    total, plus = a[1], a[3]
    n = 2 if _case(row) else 1
    lab = _labels(_rng(row), n, 1, total // n, _case(row)).view(-1)
    outs, _ = _twice(name, a, {0: lab}, lambda: ({4: IBuf(1, 1, torch.int64), 5: Buf(1, 1, 1, torch.float32)}, {}))
    cnt = int((lab != IGN).sum())
    assert int(outs[4].v.item()) == cnt, tag
    want = np.float32(1.0) / (np.float32(cnt) + np.float32(1.0 if plus else 0.0))
    assert outs[5].v.cpu().numpy().view(np.uint32)[0, 0] == np.array([want], np.float32).view(np.uint32)[0], tag
    outs[4].check(tag)
    outs[5].check(tag)


def _img_wt_weights(lab, ub, half):
    import _img_wt_oracle as W
    w = W.img_wt_class_weights(lab, ub).float()
    return w.half().float() if half else w


def _run_label_class_weights(row):
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    n, per, ub, half = a[1], a[2], a[3], a[4]
    lab = _labels(_rng(row), n, 1, per, _case(row))

    def outs():
        o = {5: IBuf(n, NC, torch.int32), 6: Buf(1, NC, NC, torch.float32), 7: Buf(n, NC, NC, torch.float32),
             8: Buf(1, 1, 1, torch.float32)}
        return o, {}
    got, _ = _twice(name, a, {0: lab}, outs)
    counts = torch.stack([torch.bincount(lab[i][lab[i] != IGN], minlength=NC) for i in range(n)])
    assert torch.equal(got[5].v.long(), counts), "%s: class counts" % tag
    w = _img_wt_weights(lab, ub, half)
    assert torch.equal(got[6].v.view(-1).view(torch.int32), w.view(torch.int32)), "%s: class weights" % tag
    den = (w.double()[None] * counts.double()).sum(1, keepdim=True)
    coef = (w.double()[None] / den).float()
    empty = (den == 0).view(-1)
    assert torch.equal(got[7].v[~empty].view(torch.int32), coef[~empty].view(torch.int32)), "%s: coef" % tag
    assert bool(torch.isnan(got[7].v[empty]).all()), tag
    scale = float(got[8].v.item())
    assert (scale != scale) if bool(empty.any()) else scale == 1.0, "%s: loss_scale %r" % (tag, scale)
    got[8].v.copy_(torch.nan_to_num(got[8].v, nan=0.0))
    for k in (5, 6, 8):
        got[k].check(tag)
    got[7].flat[: n * NC] = torch.nan_to_num(got[7].flat[: n * NC], nan=0.0)
    got[7].check(tag)


# ------------------------------------------------------------------------------------------------------- mid / loss
def _up(x, n, h, w, H, W):
    return _resample(x, n, h, w, H, W)


def _run_mid_fwd(row):
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    d = a[0]
    n, hm, wm, hl, wl, heads, sup = d[1], d[6], d[7], d[8], d[9], d[10], d[11] != 0.0
    g = _rng(row)
    lc, lx, la = _logits(g, n * hl * wl, 20), _logits(g, n * hl * wl, 20), _logits(g, n * hl * wl, 1)
    la[:] = torch.randn(la.shape, generator=g, device="cuda")
    ins = {0: _desc(d), 1: lc, 3: la}
    if heads > 1:
        ins[2] = lx

    def outs():
        o = {4: Buf(n * hm * wm, 40, 40, torch.float32)}
        if sup:
            o[5] = Buf(n * hm * wm, NC, 20, torch.float32)     # channel 19 is not written
        return o, {}
    got, _ = _twice(name, a, ins, outs)
    A4 = _up(torch.sigmoid(la.double()), n, hl, wl, hm, wm)
    C4 = _up(lc.double()[:, :NC], n, hl, wl, hm, wm)
    C4a = _up(lc.double()[:, :NC].abs(), n, hl, wl, hm, wm)
    r = torch.zeros((n * hm * wm, 40), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    r[:, :NC], A[:, :NC] = A4 * C4, A4 * C4a
    if heads > 1:
        X4 = _up(lx.double()[:, :NC], n, hl, wl, hm, wm)
        r[:, NC:2 * NC], A[:, NC:2 * NC] = A4 * X4, A4 * _up(lx.double()[:, :NC].abs(), n, hl, wl, hm, wm)
    r[:, 38:39], A[:, 38:39] = A4, A4
    got[4].check(tag)
    _check_f32(got[4].v, r, A, tag, "mid_fwd")
    if sup:
        got[5].check(tag)
        _check_f32(got[5].v, C4, C4a, tag + " mid_sup", "mid_fwd")


PLAIN = ["desc", "labels", "inv", "hi_cls", "hi_aux", "mid", "mid_sup", "g_hi", "g_lo", "g_sup", "ws", "loss", "dpr",
         "terms", "n_terms", "stream"]
EX = ["desc", "labels", "inv", "coef", "hi_cls", "hi_aux", "mid", "mid_sup", "g_hi", "g_lo", "g_sup", "ws", "loss",
      "dpr", "terms", "n_terms", "dpr_aux", "terms_aux", "n_aux", "stream"]


def _ce(J, lab, valid, coef):
    """float64 CE of J [P, 19]: (nll [P], grad (softmax - onehot) * coef, 0 where invalid)."""
    torch = _torch()
    y = torch.where(valid, lab, torch.zeros_like(lab))
    ls = torch.log_softmax(J, 1)
    oh = torch.nn.functional.one_hot(y, NC).double()
    nll = torch.where(valid, -ls.gather(1, y[:, None])[:, 0], torch.zeros_like(ls[:, 0]))
    grad = torch.where(valid[:, None], (ls.exp() - oh) * coef[:, None], torch.zeros_like(J))
    return nll, grad, ls.exp()


def _bce(J, lab, valid, coef):
    torch = _torch()
    y = torch.nn.functional.one_hot(torch.where(valid, lab, torch.zeros_like(lab)), NC).double()
    sp = J.clamp_min(0) - J * y + torch.log1p(torch.exp(-J.abs()))
    loss = torch.where(valid, sp.sum(1), torch.zeros_like(sp[:, 0]))
    P = torch.sigmoid(J)
    grad = torch.where(valid[:, None], (P - y) * coef[:, None], torch.zeros_like(J))
    return loss, grad, P


def _run_loss_fwd(row):
    import numpy as np
    torch = _torch()
    from b200seg import _lib
    name, a = row[0], row[1]
    tag, case = row_id(row), _case(row)
    names = PLAIN if name == "mscale_loss_fwd" else EX
    arg = {k: a[i] for i, k in enumerate(names)}
    idx = {k: i for i, k in enumerate(names)}
    d = arg["desc"]
    n, H, W, hq, wq, hm, wm, heads, sup_wt, kind = d[1], d[2], d[3], d[4], d[5], d[6], d[7], d[10], d[11], d[13]
    two, rmi, wt, aux_rmi = hm > 0, kind == 1, arg.get("coef") is not None, arg.get("dpr_aux") is not None
    desc = _desc(d)
    P = n * H * W
    Hp, Wp = H // 4 + 1, W // 4 + 1
    g = _rng(row)
    lab = _labels(g, n, H, W, case)
    valid = (lab != IGN).view(-1)
    labv = lab.view(-1)
    ins = {0: desc, idx["labels"]: lab}
    hi = _logits(g, n * hq * wq, 20, case=case)
    hx = _logits(g, n * hq * wq, 20, case=case)
    ins[idx["hi_cls"]] = hi
    if heads > 1:
        ins[idx["hi_aux"]] = hx
    if two:
        mid = _mid_input(g, n * hm * wm, case)
        ins[idx["mid"]] = mid
        if sup_wt != 0.0:
            msup = _logits(g, n * hm * wm, 20, case=case)
            ins[idx["mid_sup"]] = msup
    cnt = int(valid.sum())
    if wt:
        w = _img_wt_weights(lab, 1.0, False)
        counts = torch.stack([torch.bincount(lab[i][lab[i] != IGN], minlength=NC) for i in range(n)]).double()
        den = (w.double()[None] * counts).sum(1, keepdim=True)
        coef = torch.where(den > 0, w.double()[None] / den, torch.full_like(den, float("nan"))).float()
        ins[idx["coef"]] = coef.contiguous()
        inv = torch.tensor([float("nan") if bool((den == 0).any()) else 1.0], device="cuda")
        icnt = 1.0
    else:
        inv = (1.0 / (torch.tensor([float(cnt)], device="cuda") + (1.0 if rmi else 0.0))).float()
        icnt = float(inv.item())
    ins[idx["inv"]] = inv
    if rmi:
        dpr = (0.05 * torch.randn((n * Hp * Wp, 20), generator=g, device="cuda")).float()
        terms = torch.randn((n * NC,), generator=g, device="cuda").float()
        ins[idx["dpr"]], ins[idx["terms"]] = dpr, terms
    if aux_rmi:
        dpr_a = (0.05 * torch.randn((n * Hp * Wp, 20), generator=g, device="cuda")).float()
        terms_a = torch.randn((n * NC,), generator=g, device="cuda").float()
        ins[idx["dpr_aux"]], ins[idx["terms_aux"]] = dpr_a, terms_a
    nb = _lib.lib().b200seg_mscale_loss_blocks(ctypes.byref(desc))

    def outs():
        o = {idx["g_hi"]: Buf(P, 40, 40, torch.bfloat16), idx["ws"]: Buf(nb * 4, 1, 1, torch.float32),
             idx["loss"]: Buf(1, 7, 7, torch.float32)}
        if two:
            o[idx["g_lo"]] = Buf(P, 40, 40, torch.bfloat16)
            if sup_wt != 0.0:
                o[idx["g_sup"]] = Buf(P, 40, 40, torch.bfloat16)
        return o, {}
    got, _ = _twice(name, a, ins, outs)

    # float64 reference from the kernel's inputs
    hcd = _up(hi.double()[:, :NC], n, hq, wq, H, W)
    hca = _up(hi.double()[:, :NC].abs(), n, hq, wq, H, W)
    had = _up(hx.double()[:, :NC], n, hq, wq, H, W) if heads > 1 else torch.zeros_like(hcd)
    haa = _up(hx.double()[:, :NC].abs(), n, hq, wq, H, W) if heads > 1 else torch.zeros_like(hcd)
    if two:
        Mu = _up(mid.double()[:, :39], n, hm, wm, H, W)
        Ma = _up(mid.double()[:, :39].abs(), n, hm, wm, H, W)
        oma = 1.0 - Mu[:, 38]
        Jc, Ja = Mu[:, :NC] + oma[:, None] * hcd, Mu[:, NC:2 * NC] + oma[:, None] * had
        Jca, Jaa = Ma[:, :NC] + oma.abs()[:, None] * hca, Ma[:, NC:2 * NC] + oma.abs()[:, None] * haa
    else:
        oma = torch.ones((P,), dtype=torch.float64, device="cuda")
        Jc, Ja, Jca, Jaa = hcd, had, hca, haa
    if wt:
        pw = torch.where(valid, coef.double()[torch.arange(n, device="cuda").repeat_interleave(H * W),
                                                labv.clamp(0, NC - 1)], torch.zeros_like(oma))
    else:
        pw = torch.ones_like(oma)
    ones = torch.ones_like(oma)
    stats = [0.0] * 4
    w0, w1 = (0.5 if rmi else 1.0), (0.2 if aux_rmi else 0.4)
    sup_wt = float(np.float32(sup_wt))

    def head(J, Jabs, wgt, bce, dp):
        f = _bce if bce else _ce
        cw = torch.where(valid, ones * wgt * icnt * pw, torch.zeros_like(ones))     # 1 / 0 never reaches a gradient
        loss, gr, Pr = f(J, labv, valid, cw)
        A = cw.abs()[:, None] * (1.0 + Jabs.max(1, keepdim=True).values)
        if dp is not None:
            cell = ((torch.arange(n, device="cuda").repeat_interleave(H * W) * Hp +
                     (torch.arange(H, device="cuda").repeat_interleave(W).repeat(n) + 2) // 4) * Wp +
                    (torch.arange(W, device="cuda").repeat(n * H) + 2) // 4)
            dpc = dp.double()[cell, :NC]
            gr = gr + torch.where(valid[:, None], dpc * 0.0625 * Pr * (1 - Pr), torch.zeros_like(gr))
            A = A + dpc.abs() * 0.0625 * 0.25
        return (loss * pw).sum(), gr, A
    stats[0], gc, Ac = head(Jc, Jca, w0, rmi, dpr if rmi else None)
    if heads > 1:
        stats[1], ga, Aa = head(Ja, Jaa, w1, rmi, dpr_a if aux_rmi else None)
    else:
        ga, Aa = torch.zeros_like(gc), torch.zeros_like(gc)
    ghi = torch.zeros((P, 40), dtype=torch.float64, device="cuda")
    Ahi = torch.zeros_like(ghi)
    ghi[:, :NC], ghi[:, NC:2 * NC] = oma[:, None] * gc, oma[:, None] * ga
    Ahi[:, :NC], Ahi[:, NC:2 * NC] = oma.abs()[:, None] * Ac, oma.abs()[:, None] * Aa
    ghi[:, 39], Ahi[:, 39] = oma, (Ma[:, 38] + 1.0 if two else ones)
    if sup_wt != 0.0:
        s3, Sh, Ash = head(hcd, hca, sup_wt, rmi, None)
        stats[3] = s3
        ghi[:, :NC] += Sh
        Ahi[:, :NC] += Ash
    if two:
        glo = torch.zeros((P, 40), dtype=torch.float64, device="cuda")
        Alo = torch.zeros_like(glo)
        glo[:, :NC], glo[:, NC:2 * NC], Alo[:, :NC], Alo[:, NC:2 * NC] = gc, ga, Ac, Aa
        glo[:, 38] = -(hcd * gc + had * ga).sum(1)
        Alo[:, 38] = (hca * (gc.abs() + Ac) + haa * (ga.abs() + Aa)).sum(1)
        _check_rows(got[idx["g_lo"]], glo, Alo, valid, 39, tag + " Glo", "loss_fwd Glo")
        if sup_wt != 0.0:
            Su = _up(msup.double()[:, :NC], n, hm, wm, H, W)
            Sa = _up(msup.double()[:, :NC].abs(), n, hm, wm, H, W)
            s2, Sl, Asl = head(Su, Sa, sup_wt, rmi, None)
            stats[2] = s2
            gs = torch.zeros((P, 40), dtype=torch.float64, device="cuda")
            As = torch.zeros_like(gs)
            gs[:, :NC], As[:, :NC] = Sl, Asl
            _check_rows(got[idx["g_sup"]], gs, As, valid, 40, tag + " Gsup", "loss_fwd Gsup")
    _check_rows(got[idx["g_hi"]], ghi, Ahi, valid, 38, tag + " Ghi", "loss_fwd Ghi")
    got[idx["ws"]].check(tag + " partial_ws")
    # loss vector: t_k are the sums of the pointwise terms over valid pixels (weighted by pw for the image-weighted
    # CE), every term >= 0, so the sums of magnitudes are the sums themselves (plus |rmi_terms|)
    t = [float(x) for x in stats]
    r = [float(terms.double().sum()) if rmi else 0.0, float(terms_a.double().sum()) if aux_rmi else 0.0]
    ra = [float(terms.double().abs().sum()) if rmi else 0.0, float(terms_a.double().abs().sum()) if aux_rmi else 0.0]
    ic = float(inv.item())
    lin = ic * (w0 * t[0] + (w1 * t[1] if heads > 1 else 0.0) + sup_wt * (t[2] + t[3])) if t != [0.0] * 4 or \
        math.isfinite(ic) else float("nan")
    want = [lin + r[0] + r[1]] + [ic * tk for tk in t] + r
    mag = [abs(lin) + ra[0] + ra[1]] + [abs(ic * tk) for tk in t] + ra
    out = got[idx["loss"]].v.view(-1).double().tolist()
    for k in range(7):
        if want[k] != want[k]:
            assert out[k] != out[k], "%s: loss_out[%d] = %r, want NaN" % (tag, k, out[k])
            continue
        e = abs(out[k] - want[k]) / max(mag[k], 1e-30)
        _note("loss_out sum/mag", e, tag)
        assert e <= STAT_REL, "%s: loss_out[%d] %r vs %r" % (tag, k, out[k], want[k])
    got[idx["loss"]].v.copy_(torch.nan_to_num(got[idx["loss"]].v, nan=0.0))
    got[idx["loss"]].check(tag + " loss_out")


def _check_rows(buf, r, A, valid, grad_cols, what, kind):
    """bf16 gradient rows against float64; gradient channels [0, grad_cols) of ignored pixels exactly 0."""
    torch = _torch()
    buf.check(what)
    out = buf.v
    bad = int((out[~valid, :grad_cols].float() != 0).sum())
    assert bad == 0, "%s: %d nonzero gradients at ignored pixels" % (what, bad)
    # outputs below the fp32 resolution of their own arithmetic (|r| <= EW_REL * A: saturated softmax / BCE terms, where
    # fp32 sigmoid(30) is 1) are held to the error bound only, not counted as bf16 mismatches
    tiny = r.abs() <= EW_REL * A
    err = (out.double() - r).abs()
    assert bool((err[tiny] <= (ew._ulp_bf16(r) + EW_REL * A)[tiny]).all()), "%s: error bound" % what
    ew._check_bf16(torch.where(tiny, r.to(torch.bfloat16), out), r, A, what, kind)


# ----------------------------------------------------------------------------------------------------- backward
def _adj(x, n, h, w, H, W):
    """Transpose of _resample: x [n * H * W, c] -> [n * h * w, c]."""
    torch = _torch()
    Uy, Ux = _interp(H, h), _interp(W, w)
    c = x.shape[1]
    t = torch.einsum("Yy,nYXc->nyXc", Uy, x.reshape(n, H, W, c))
    return torch.einsum("Xx,nyXc->nyxc", Ux, t).reshape(n * h * w, c)


def _run_hi_bwd(row):
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    d = a[0]
    n, H, W, hq, wq, heads = d[1], d[2], d[3], d[4], d[5], d[10]
    g = _rng(row)
    G = _bf16_rows(g, n * H * W, 40)

    def outs():
        o = {2: Buf(n * hq * wq, 32, 32, torch.bfloat16)}
        if heads > 1:
            o[3] = Buf(n * hq * wq, 32, 32, torch.bfloat16)
        return o, {}
    got, _ = _twice(name, a, {0: _desc(d), 1: G}, outs)
    Gd = G.double()
    for k, hd in ((2, 0), (3, 1)):
        if k not in got:
            continue
        r = torch.zeros((n * hq * wq, 32), dtype=torch.float64, device="cuda")
        A = torch.zeros_like(r)
        r[:, :NC] = _adj(Gd[:, hd * NC:(hd + 1) * NC], n, hq, wq, H, W)
        A[:, :NC] = _adj(Gd[:, hd * NC:(hd + 1) * NC].abs(), n, hq, wq, H, W)
        got[k].check(tag)
        ew._check_bf16(got[k].v, r, A, "%s head %d" % (tag, hd), "hi_bwd")


def _run_lo_bwd(row):
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    d = a[0]
    n, H, W, hm, wm, hl, wl, heads, sup = d[1], d[2], d[3], d[6], d[7], d[8], d[9], d[10], d[11] != 0.0
    g = _rng(row)
    Glo = _bf16_rows(g, n * H * W, 40)
    ins = {0: _desc(d), 1: Glo}
    if sup:
        Gs = _bf16_rows(g, n * H * W, 40)
        Gs[:, NC:] = 0
        ins[2] = Gs
    lc, lx = _logits(g, n * hl * wl, 20), _logits(g, n * hl * wl, 20)
    la = torch.randn((n * hl * wl,), generator=g, device="cuda").float()
    mid = _mid_input(g, n * hm * wm)
    ins.update({3: lc, 5: la, 6: mid})
    if heads > 1:
        ins[4] = lx

    def outs():
        o = {7: Buf(n * hm * wm, 40, 40, torch.float32), 8: Buf(n * hl * wl, 32, 32, torch.bfloat16),
             10: Buf(n * hl * wl, 8, 8, torch.bfloat16)}
        if heads > 1:
            o[9] = Buf(n * hl * wl, 32, 32, torch.bfloat16)
        return o, {}
    got, _ = _twice(name, a, ins, outs)
    dP = _adj(Glo.double(), n, hm, wm, H, W)
    dPa = _adj(Glo.double().abs(), n, hm, wm, H, W)
    A4 = mid.double()[:, 38:39]
    C4 = _up(lc.double()[:, :NC], n, hl, wl, hm, wm)
    C4a = _up(lc.double()[:, :NC].abs(), n, hl, wl, hm, wm)
    D = torch.zeros((n * hm * wm, 40), dtype=torch.float64, device="cuda")
    DA = torch.zeros_like(D)
    D[:, :NC], DA[:, :NC] = A4 * dP[:, :NC], A4 * dPa[:, :NC]
    if sup:
        D[:, :NC] += _adj(Gs.double()[:, :NC], n, hm, wm, H, W)
        DA[:, :NC] += _adj(Gs.double()[:, :NC].abs(), n, hm, wm, H, W)
    D[:, 38] = dP[:, 38] + (C4 * dP[:, :NC]).sum(1)
    DA[:, 38] = dPa[:, 38] + (C4a * dPa[:, :NC]).sum(1)
    if heads > 1:
        X4 = _up(lx.double()[:, :NC], n, hl, wl, hm, wm)
        X4a = _up(lx.double()[:, :NC].abs(), n, hl, wl, hm, wm)
        D[:, NC:2 * NC], DA[:, NC:2 * NC] = A4 * dP[:, NC:2 * NC], A4 * dPa[:, NC:2 * NC]
        D[:, 38] += (X4 * dP[:, NC:2 * NC]).sum(1)
        DA[:, 38] += (X4a * dPa[:, NC:2 * NC]).sum(1)
    got[7].check(tag + " dmid_ws")
    _check_f32(got[7].v, D, DA, tag + " dmid_ws", "mid_bwd")
    Dk = got[7].v.double()           # the second stage from the kernel's own dmid_ws
    for k, lo_ in ((8, 0), (9, NC)):
        if k not in got:
            continue
        r = torch.zeros((n * hl * wl, 32), dtype=torch.float64, device="cuda")
        A = torch.zeros_like(r)
        r[:, :NC] = _adj(Dk[:, lo_:lo_ + NC], n, hl, wl, hm, wm)
        A[:, :NC] = _adj(Dk[:, lo_:lo_ + NC].abs(), n, hl, wl, hm, wm)
        got[k].check(tag)
        ew._check_bf16(got[k].v, r, A, tag, "lo_bwd")
    s = torch.sigmoid(la.double())
    r = torch.zeros((n * hl * wl, 8), dtype=torch.float64, device="cuda")
    A = torch.zeros_like(r)
    r[:, 0] = _adj(Dk[:, 38:39], n, hl, wl, hm, wm)[:, 0] * s * (1 - s)
    A[:, 0] = _adj(Dk[:, 38:39].abs(), n, hl, wl, hm, wm)[:, 0] * s * (1 - s)
    got[10].check(tag)
    ew._check_bf16(got[10].v, r, A, tag + " d_attn", "lo_bwd")


# ---------------------------------------------------------------------------------------------------------- RMI
def _pool(x, n, H, W):
    """float64 avg_pool2d(4, 4, pad 2) of x [n * H * W, c] (zero padding, divisor 16) -> [n * Hp * Wp, c]."""
    torch = _torch()
    c = x.shape[1]
    t = x.reshape(n, H, W, c).permute(0, 3, 1, 2)
    p = torch.nn.functional.avg_pool2d(t, 4, 4, 2)
    return p.permute(0, 2, 3, 1).reshape(-1, c)


def _run_rmi_pool(row):
    torch = _torch()
    name, a = row[0], row[1]
    tag = row_id(row)
    d = a[0]
    n, H, W, hq, wq, hm, wm = d[1], d[2], d[3], d[4], d[5], d[6], d[7]
    aux = name == "rmi_pool_aux"
    Hp, Wp = H // 4 + 1, W // 4 + 1
    g = _rng(row)
    lab = _labels(g, n, H, W)
    hi = _logits(g, n * hq * wq, 20)
    ins = {0: _desc(d), 1: lab, 2: hi}
    if hm:
        mid = _mid_input(g, n * hm * wm)
        ins[3] = mid

    def outs():
        o = {4: Buf(n * Hp * Wp, 20, 20, torch.float32)}
        if not aux:
            o[5] = Buf(n * Hp * Wp, 20, 20, torch.float32)
        return o, {}
    got, _ = _twice(name, a, ins, outs)
    J = _up(hi.double()[:, :NC], n, hq, wq, H, W)
    if hm:
        Mu = _up(mid.double()[:, :39], n, hm, wm, H, W)
        hd = NC if aux else 0
        J = Mu[:, hd:hd + NC] + (1.0 - Mu[:, 38:39]) * J
    lv = lab.view(-1)
    valid = ((lv != IGN) & (lv >= 0) & (lv < NC)).double()[:, None]
    pr = _pool(torch.sigmoid(J) * valid + 1e-6, n, H, W)
    r = torch.zeros((n * Hp * Wp, 20), dtype=torch.float64, device="cuda")
    r[:, :NC] = pr
    got[4].check(tag)
    _check_f32(got[4].v, r, r.abs() + 1e-30, tag + " pr_pool", "rmi_pool")
    if not aux:
        oh = torch.nn.functional.one_hot(lv.clamp(0, NC - 1), NC).double() * valid
        r = torch.zeros_like(r)
        r[:, :NC] = _pool(oh, n, H, W)
        got[5].check(tag)
        _check_f32(got[5].v, r, r.abs() + 1e-30, tag + " la_pool", "rmi_pool")


def rmi_lower_bound(pr, la, n, Hp, Wp, radius=3, pos_alpha=5e-4):
    """rmi_lower_bound (loss/rmi.py) from pooled maps pr, la [n * Hp * Wp, 20] in float64: -> [n, 19] of
    sum_k log(diag(chol(appro + alpha I)) + 1e-8), the per (image, class) value before the mean and the / 9."""
    torch = _torch()
    pr = pr[:, :NC].reshape(n, Hp, Wp, NC).permute(0, 3, 1, 2)
    la = la[:, :NC].reshape(n, Hp, Wp, NC).permute(0, 3, 1, 2)
    nh, nw = Hp - (radius - 1), Wp - (radius - 1)
    la_v = torch.stack([la[:, :, y:y + nh, x:x + nw] for y in range(radius) for x in range(radius)], 2)
    pr_v = torch.stack([pr[:, :, y:y + nh, x:x + nw] for y in range(radius) for x in range(radius)], 2)
    la_v = la_v.reshape(n, NC, 9, -1)
    pr_v = pr_v.reshape(n, NC, 9, -1)
    eye = torch.eye(9, dtype=torch.float64, device=pr.device)[None, None]
    la_v = la_v - la_v.mean(3, keepdim=True)
    pr_v = pr_v - pr_v.mean(3, keepdim=True)
    la_cov = la_v @ la_v.transpose(2, 3)
    pr_cov = pr_v @ pr_v.transpose(2, 3)
    inv = torch.inverse(pr_cov + eye * pos_alpha)
    la_pr = la_v @ pr_v.transpose(2, 3)
    appro = la_cov - (la_pr @ inv) @ la_pr.transpose(-2, -1)
    chol = torch.linalg.cholesky(appro + eye * pos_alpha)
    return torch.log(torch.diagonal(chol, dim1=-2, dim2=-1) + 1e-8).sum(-1)


def _run_rmi_solve_grad(row):
    import numpy as np
    torch = _torch()
    from b200seg import _lib
    name, a = row[0], row[1]
    tag = row_id(row)
    n, H, W, scale = a[0], a[1], a[2], a[5]
    Hp, Wp = H // 4 + 1, W // 4 + 1
    g = _rng(row)
    lab = _labels(g, n, H, W, one_class=3 if _case(row) == "one_class" else None)
    logit = torch.randn((n * H * W, NC), generator=g, device="cuda", dtype=torch.float64) * 2
    valid = (lab.view(-1) != IGN).double()[:, None]
    pr = torch.zeros((n * Hp * Wp, 20), device="cuda")
    la = torch.zeros_like(pr)
    pr[:, :NC] = _pool(torch.sigmoid(logit) * valid + 1e-6, n, H, W).float()
    la[:, :NC] = _pool(torch.nn.functional.one_hot(lab.view(-1).clamp(0, NC - 1), NC).double() * valid, n, H, W).float()
    nbytes = _lib.lib().b200seg_rmi_ws_bytes(n)
    a = a[:7] + (nbytes,) + a[8:]

    def outs():
        return {6: DBuf(nbytes // 8, 1, 1, torch.float64), 8: DBuf(n * NC, 180, 180, torch.float64),
                9: Buf(n * NC, 1, 1, torch.float32), 10: Buf(n * Hp * Wp, 20, 20, torch.float32)}, {}
    got, _ = _twice(name, a, {3: pr, 4: la}, outs)
    for k in (6, 8, 9, 10):
        got[k].check(tag)
    sc = float(np.float32(scale))
    prd = pr.double().requires_grad_(True)
    with torch.enable_grad():
        terms = rmi_lower_bound(prd, la.double(), n, Hp, Wp) * sc
        terms.sum().backward()
    dpr = prd.grad
    for got_t, r, what in ((got[9].v.view(-1), terms.detach().view(-1), "rmi_terms"),
                           (got[10].v, dpr, "dpr")):
        r = r.double()
        e = float(((got_t.double() - r).abs() - _ulp32(r)).clamp_min(0).max()) / max(float(r.abs().max()), 1e-300)
        _note("rmi " + what + " fp64 error / max", e, tag)
        assert e <= RMI_ALLOW, "%s %s: error %.3e of the largest value, allowance %.1e" % (tag, what, e, RMI_ALLOW)


RUNNERS = {"count_valid": _run_count_valid, "label_class_weights": _run_label_class_weights,
           "mscale_mid_fwd": _run_mid_fwd, "mscale_loss_fwd": _run_loss_fwd, "mscale_loss_fwd_ex": _run_loss_fwd,
           "mscale_hi_bwd": _run_hi_bwd, "mscale_lo_bwd": _run_lo_bwd, "rmi_pool": _run_rmi_pool,
           "rmi_pool_aux": _run_rmi_pool, "rmi_solve_grad": _run_rmi_solve_grad}


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_loss_configuration_against_float64(row):
    RUNNERS[row[0]](row)


@pytest.mark.gpu
def test_rmi_restatement_matches_oracle():
    """rmi_lower_bound above, from pooled maps, against oracle.seg_oracle.rmi_loss on logits (the reference's
    RMILoss.forward_sigmoid): the RMI part of the loss agrees to float64 rounding."""
    torch = _torch()
    from oracle import seg_oracle as O
    g = torch.Generator(device="cuda").manual_seed(7)
    n, H, W = 2, 48, 64
    logits = 2 * torch.randn((n, NC, H, W), generator=g, device="cuda", dtype=torch.float64)
    lab = _labels(g, n, H, W)
    full = O.rmi_loss(logits, lab).double()
    bce = O.rmi_loss(logits, lab, do_rmi=False).double()
    valid = (lab.view(-1) != IGN).double()[:, None]
    lg = logits.permute(0, 2, 3, 1).reshape(-1, NC)
    pr = _pool(torch.sigmoid(lg) * valid + 1e-6, n, H, W).float().double()
    la = _pool(torch.nn.functional.one_hot(lab.view(-1).clamp(0, NC - 1), NC).double() * valid, n, H, W).float().double()
    mine = rmi_lower_bound(pr, la, n, H // 4 + 1, W // 4 + 1).mean(0).sum() / 9.0
    # the oracle pools in float64 from fp64 logits, then rounds per class to fp32
    assert abs(float(full - 0.5 * bce) - 0.5 * float(mine)) <= 1e-5 * abs(float(mine)) + 1e-7


# ------------------------------------------------------------------------------------------------- composed rows
# One row per geometry of the eight architectures (heads, hi ratio, one scale or two with the lo ratio) and criterion,
# at n = 2, 64 x 96, with supervision on the two-scale geometries: the step's own chain (count_valid or
# label_class_weights, mid_fwd, rmi_pool / rmi_solve_grad, loss_fwd, hi_bwd, lo_bwd) against float64 autograd of the
# reference formula on F.interpolate (the one test_gpu_ops.py states), with the criteria of oracle/seg_oracle.py and
# tests/_img_wt_oracle.py. Nothing here shares the kernels' 40-wide row layout, so a layout convention the launches
# agree on but the reference does not (where head 1 sits, which column carries dA or 1 - A) fails these rows.
# Bound per output: ulp_bf16(r) + COMPOSED_REL * (the pixel's largest |r|; the tensor's for the attention logit) +
# 2^-12 * (the tensor's largest |r|), for the bf16 gradient rows between the launches; the loss within COMPOSED_LOSS_REL.
COMPOSED_REL = 2.0 ** -7
COMPOSED_LOSS_REL = 2e-5
GEOMETRIES = [(2, 4, 4), (2, 4, None), (1, 4, None), (1, 4, 4), (1, 2, None), (1, 2, 2)]   # (heads, hi ratio, lo ratio)
COMPOSED = [(geo_, crit) for geo_ in GEOMETRIES for crit in ("ce", "rmi", "img_wt")] + \
    [(geo_, "rmi_aux") for geo_ in GEOMETRIES if geo_[0] > 1]


def composed_id(row):
    (heads, rh, rl), crit = row
    return "heads%d-hi%d-%s-%s" % (heads, rh, "lo%d" % rl if rl else "one_scale", crit)


def _check_composed(got, r, what, scale="pixel"):
    """scale 'pixel': the pixel's largest |r| (class gradients); 'tensor': the tensor's largest |r| (the attention
    logit's gradient, one channel that is a difference of the heads' products, so its size says nothing about the
    rounding of its terms)."""
    torch = _torch()
    got, r = got.double(), r.double()
    err = (got - r).abs()
    big = r.abs().amax(-1, keepdim=True) if scale == "pixel" else r.abs().max()
    bound = ew._ulp_bf16(r) + COMPOSED_REL * big + 2.0 ** -12 * float(r.abs().max())
    _note("composed err/bound", float((err / bound.clamp_min(1e-300)).max()), what)
    assert bool((err <= bound).all()), "%s: %d outputs off, max err %.3e" % (what, int((err > bound).sum()),
                                                                             float(err.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("row", COMPOSED, ids=composed_id)
def test_composed_loss_step_against_float64_autograd(row):
    torch = _torch()
    import torch.nn.functional as F
    from b200seg import raw
    from oracle import seg_oracle as O
    import _img_wt_oracle as W
    (heads, rh, rl), crit = row
    n, H, W_ = 2, 64, 96
    hq, wq = H // rh, W_ // rh
    two = rl is not None
    hm, wm = (H // 2, W_ // 2) if two else (0, 0)
    hl, wl = (hm // rl, wm // rl) if two else (0, 0)
    sup = 0.05 if two else 0.0
    rmi = crit.startswith("rmi")
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(composed_id(row).encode()))
    gts = _labels(g, n, H, W_)
    gts[:, 20:30, 40:50] = 3                                  # a coherent region: non-trivial label covariance

    def logits(h, w, c=NC):
        t = torch.zeros((n, h, w, 20 if c == NC else c), device="cuda")
        t[..., :c] = 2 * torch.randn((n, h, w, c), generator=g, device="cuda")
        return t.contiguous()
    hi = [logits(hq, wq) for _ in range(heads)]
    d = raw.mscale_desc(n, H, W_, hq, wq, hm, wm, hl, wl, heads, 1.0, 0.4, sup, 255, 1 if rmi else 0)
    # the step, as b200seg.model.train_loss runs it
    mid = mid_sup = None
    if two:
        lo = [logits(hl, wl) for _ in range(heads)]
        lo_attn = logits(hl, wl, 1)
        mid, mid_sup = raw.mscale_mid_fwd(d, lo[0], lo[1] if heads > 1 else None, lo_attn)
    coef = None
    if crit == "img_wt":
        _, _, coef, inv = raw.label_class_weights(gts, 1.0, False)
    else:
        inv = raw.count_valid(gts, 255, plus_one=rmi)
    dpr = terms = dpr_a = terms_a = None
    if rmi:
        pr, la = raw.rmi_pool(d, gts, hi[0], mid)
        dpr, terms = raw.rmi_solve_grad(d, pr, la, d.w_head0)
        if crit == "rmi_aux":
            dpr_a, terms_a = raw.rmi_solve_grad(d, raw.rmi_pool_aux(d, gts, hi[1], mid), la, d.w_head1)
    loss, g_hi, g_lo, g_sup = raw.mscale_loss_fwd(d, gts, inv, hi[0], hi[1] if heads > 1 else None, mid, mid_sup, dpr,
                                                  terms, coef, dpr_a, terms_a)
    d_cls, d_aux = raw.mscale_hi_bwd(d, g_hi)
    if two:
        dl_cls, dl_aux, dl_attn = raw.mscale_lo_bwd(d, g_lo, g_sup, lo[0], lo[1] if heads > 1 else None, lo_attn, mid)
    torch.cuda.synchronize()

    # the reference formula in float64 (network/ocrnet.py two_scale_forward, network/mscale.py, loss/*.py)
    leaf = lambda t, c=NC: t[..., :c].double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)   # noqa: E731
    up = lambda t, size: F.interpolate(t, size=size, mode="bilinear", align_corners=False)   # noqa: E731
    if crit == "ce":
        head0 = head1 = side = lambda t: O.ce_loss(t, gts)                # noqa: E731
    elif crit == "img_wt":
        wcrit = W.criterion_img_wt(1.0)
        head0 = head1 = side = lambda t: wcrit(t, gts)                    # noqa: E731
    else:
        head0 = lambda t: O.rmi_loss(t, gts, do_rmi=True)                  # noqa: E731
        head1 = lambda t: O.rmi_loss(t, gts, do_rmi=crit == "rmi_aux")    # noqa: E731
        side = lambda t: O.rmi_loss(t, gts, do_rmi=False)                  # noqa: E731
    with torch.enable_grad():
        L_hi = [leaf(t) for t in hi]
        if two:
            L_lo = [leaf(t) for t in lo]
            L_attn = leaf(lo_attn, 1)
            a = up(torch.sigmoid(L_attn), (hm, wm))
            a_up = up(a, (H, W_))
            joints = [up(a * up(L_lo[k], (hm, wm)), (H, W_)) + (1 - a_up) * up(L_hi[k], (H, W_)) for k in range(heads)]
        else:
            joints = [up(t, (H, W_)) for t in L_hi]
        ref = head0(joints[0])
        if heads > 1:
            ref = ref + 0.4 * head1(joints[1])
        if sup:
            ref = ref + sup * side(up(up(L_lo[0], (hm, wm)), (H, W_))) + sup * side(up(L_hi[0], (H, W_)))
        ref.backward()
    tag = composed_id(row)
    lrel = abs(float(loss[0]) - float(ref)) / abs(float(ref))
    _note("composed loss rel", lrel, tag)
    assert lrel <= COMPOSED_LOSS_REL, (tag, float(loss[0]), float(ref))
    nhwc = lambda t: t.grad.permute(0, 2, 3, 1)                             # noqa: E731
    _check_composed(d_cls[..., :NC], nhwc(L_hi[0]), tag + " d hi cls")
    assert float(d_cls[..., NC:].float().abs().max()) == 0.0, tag
    if heads > 1:
        _check_composed(d_aux[..., :NC], nhwc(L_hi[1]), tag + " d hi aux")
    if two:
        _check_composed(dl_cls[..., :NC], nhwc(L_lo[0]), tag + " d lo cls")
        if heads > 1:
            _check_composed(dl_aux[..., :NC], nhwc(L_lo[1]), tag + " d lo aux")
        _check_composed(dl_attn[..., :1], nhwc(L_attn), tag + " d lo attn", "tensor")
