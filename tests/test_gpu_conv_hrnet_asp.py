"""The dilated 3x3 ASPP branches of basic.HRNet_ASP / mscale.HRNet_ASP at full W48 width, checked against float64: the
720 -> 256 convolution at dilation 12 / 24 / 36 on the stride-4 trunk map of a 1024 x 2048 crop (256 x 512, the 1.0x
pass) and of its 0.5x pass (128 x 256). Forward with batch statistics into a channel slice of the 1280-channel concat,
data gradient into the 720-channel map, weight gradient. Inputs are bf16; the reference is F.conv2d and its transposes
in float64 from exactly those values, and the bounds are tied to fp32 accumulation like tests/test_gpu_conv_classes.py
(A = the same convolution of |inputs|): bf16 outputs within ulp_bf16(r) + ACC_REL * A, fp32 weight gradients within
ACC_REL * A, statistics within 1e-6 of the float64 sums of the stored outputs."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

pytestmark = pytest.mark.gpu

ACC_REL = 2.0 ** -18
CIN, COUT, RED5 = 720, 256, 5 * 256
SIZES = [(256, 512), (128, 256)]
RATES = [12, 24, 36]


def _bf16(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).cuda()


def _ulp_bf16(r):
    e = torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _conv64(x_nhwc, w_oihw, dil):
    return F.conv2d(x_nhwc.permute(0, 3, 1, 2).double(), w_oihw.double(), padding=dil, dilation=dil)


def _weights(seed):
    """[O][9][I] bf16 forward operand and the OIHW float64 view of the same values."""
    w = _bf16((COUT, 9, CIN), seed, CIN ** -0.5 / 3)
    return w, w.double().view(COUT, 3, 3, CIN).permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("hw", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("dil", RATES)
def test_forward_with_statistics_into_the_concat_slice(hw, dil):
    from b200seg import raw
    h, w = hw
    x = _bf16((1, h, w, CIN), 10 + dil)
    wt, w64 = _weights(20 + dil)
    cat = torch.full((1, h, w, RED5), float("nan"), dtype=torch.bfloat16, device="cuda")
    c0 = 2 * COUT + RATES.index(dil) * COUT
    y, (part, grid, cpad) = raw.conv2d_fwd(x, wt, emit_stats=True, dilation=dil, out=cat[..., c0:c0 + COUT])
    torch.cuda.synchronize()
    ref = _conv64(x, w64, dil).permute(0, 2, 3, 1)
    A = _conv64(x.abs(), w64.abs(), dil).permute(0, 2, 3, 1)
    got = cat[..., c0:c0 + COUT].double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    bad = err > _ulp_bf16(ref) + ACC_REL * A
    assert not bad.any(), (int(bad.sum()), float(err.max()))
    others = torch.cat([cat[..., :c0], cat[..., c0 + COUT:]], -1)
    assert torch.isnan(others.float()).all()                    # nothing outside the slice is written
    p = part[: grid * 2 * cpad].view(grid, 2, cpad).double().sum(0)[:, :COUT]
    yf = got.view(-1, COUT)                                     # statistics of the stored (bf16) values
    assert ((p[0] - yf.sum(0)).abs() <= 1e-6 * yf.abs().sum(0) + 1e-6).all()
    assert ((p[1] - (yf * yf).sum(0)).abs() <= 1e-6 * (yf * yf).sum(0) + 1e-6).all()


@pytest.mark.parametrize("hw", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("dil", RATES)
def test_data_gradient_into_the_trunk_map(hw, dil):
    """dx = conv_transpose(dy, w) accumulated onto the gradient the other consumers already left in the map."""
    from b200seg import raw
    h, w = hw
    dy = _bf16((1, h, w, COUT), 30 + dil)
    wt, w64 = _weights(40 + dil)
    w_d = wt.view(COUT, 9, CIN).flip(1).permute(2, 1, 0).contiguous()     # [Cin][taps flipped][Cout]
    addend = _bf16((1, h, w, CIN), 50 + dil)
    ref0 = addend.double()
    dx = raw.conv2d_dgrad(dy, w_d, (1, h, w, CIN), 3, 1, addend=addend.clone(), dilation=dil)
    torch.cuda.synchronize()
    tr = lambda g, ww: F.conv_transpose2d(g.permute(0, 3, 1, 2).double(), ww.double(), padding=dil,
                                          dilation=dil).permute(0, 2, 3, 1)
    ref = tr(dy, w64) + ref0
    A = tr(dy.abs(), w64.abs()) + ref0.abs()
    got = dx.double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    bad = err > _ulp_bf16(ref) + ACC_REL * A
    assert not bad.any(), (int(bad.sum()), float(err.max()))


@pytest.mark.parametrize("hw", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("dil", RATES)
def test_weight_gradient(hw, dil):
    """dw += sum_pixels dy x shifted(x) into a non-zero fp32 accumulator ([Cout][taps][Cin])."""
    from b200seg import raw
    h, w = hw
    x = _bf16((1, h, w, CIN), 60 + dil)
    dy = _bf16((1, h, w, COUT), 70 + dil, 0.1)
    acc0 = torch.randn((COUT, 9, CIN), generator=torch.Generator().manual_seed(80 + dil)).cuda()
    acc = acc0.clone()
    ws = raw.conv2d_wgrad(x, dy, acc, COUT, 3, 1, dilation=dil)
    torch.cuda.synchronize()
    del ws

    def wg(xx, gg):
        out = torch.nn.grad.conv2d_weight(xx.permute(0, 3, 1, 2).double(), (COUT, CIN, 3, 3),
                                          gg.permute(0, 3, 1, 2).double(), padding=dil, dilation=dil)
        return out.permute(0, 2, 3, 1).reshape(COUT, 9, CIN)      # OIHW -> [O][taps][I]
    ref = wg(x, dy) + acc0.double()
    A = wg(x.abs(), dy.abs()) + acc0.double().abs()
    err = (acc.double() - ref).abs()
    assert torch.isfinite(acc).all()
    bad = err > ACC_REL * A
    assert not bad.any(), (int(bad.sum()), float(err.max()), float((err / A).max()))
