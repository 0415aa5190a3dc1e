"""Convolutions whose [8 warps][2][Cout] shared-memory statistics area alone exceeds the 227 KB a CTA may hold:
WideResNet-38's 4096-channel mod7 (2048 -> 4096 1x1 conv3 and projection, with the batch statistics of the stored sum)
and the data gradient into its 4096-channel output. The planner keeps one N tile's statistics per CTA; the outputs and
the per-channel sums must still equal a PyTorch fp32 reference."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("h,w", [(16, 32), (64, 128)])
def test_4096_channel_forward_with_statistics(h, w):
    from b200seg import raw
    g = torch.Generator().manual_seed(1)
    cin, cout = 2048, 4096
    x = torch.randn((1, h, w, cin), generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn((cout, 1, cin), generator=g) * cin ** -0.5).to(torch.bfloat16).cuda()
    add = torch.randn((1, h, w, cout), generator=g).to(torch.bfloat16).cuda()
    y, (part, grid, cpad) = raw.conv2d_fwd(x, wt, emit_stats=True, addend=add)
    torch.cuda.synchronize()
    ref = torch.einsum("nhwc,oc->nhwo", x.float(), wt[:, 0].float()) + add.float()
    assert (y.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
    p = part[: grid * 2 * cpad].view(grid, 2, cpad).double().sum(0)[:, :cout]
    yf = y.double().view(-1, cout)                   # the statistics are those of the stored (bf16) values
    assert torch.allclose(p[0], yf.sum(0), rtol=1e-5, atol=1e-3)
    assert torch.allclose(p[1], (yf * yf).sum(0), rtol=1e-5, atol=1e-3)


def test_4096_channel_data_gradient():
    from b200seg import raw
    g = torch.Generator().manual_seed(2)
    cin, cout, h, w = 4096, 256, 16, 32               # ASPP 1x1 branch: its input gradient has 4096 channels
    dy = torch.randn((1, h, w, cout), generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn((cout, 1, cin), generator=g) * cin ** -0.5).to(torch.bfloat16)
    w_d = wt[:, 0].t().contiguous().view(cin, 1, cout).cuda()      # [Cin][taps][Cout (multiple of 8)]
    dx = raw.conv2d_dgrad(dy, w_d, (1, h, w, cin), 1, 1)
    torch.cuda.synchronize()
    ref = torch.einsum("nhwo,oc->nhwc", dy.float(), wt[:, 0].float().cuda())
    assert (dx.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()
