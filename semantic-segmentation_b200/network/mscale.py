"""Overlay of the reference's network/mscale.py: the arch strings ``mscale.HRNet`` = MscaleBasic (seg head +
scale-attention head straight on the HRNet features, :450-475) and ``mscale.DeepV3W38`` = MscaleV3Plus over the
WideResNet-38 trunk (DeepLabV3+ decoder and scale-attention head on the same 304-channel concat, :232-336) and
``mscale.HRNet_ASP`` = ASPP over the HRNet trunk (seg head and scale-attention head on the bot_aspp output, :479-515),
all with the hierarchical two-scale training forward / n-scale evaluation of MscaleBase (:114-231). The other trunks of
that file (ResNet-50, the fused-ASPP variants ...) are not provided."""
from ._factory import build


def HRNet(num_classes, criterion, s2s4=None):
    """network/mscale.py:473-475."""
    return build("mscale.HRNet", num_classes, criterion)


def DeepV3W38(num_classes, criterion):
    """network/mscale.py:335-336."""
    return build("mscale.DeepV3W38", num_classes, criterion)


def HRNet_ASP(num_classes, criterion, s2s4=None):
    """network/mscale.py:514-515."""
    return build("mscale.HRNet_ASP", num_classes, criterion)
