"""network.basic factories (network/basic.py:104-111) backed by the sm_90a kernels: ``basic.HRNet`` (BASELINE config 1
plumbing model, seg head on the trunk features) and ``basic.HRNet_ASP`` (ASPP, bot_aspp and seg head over the HRNet
trunk, :67-101)."""
from ._factory import build


def HRNet(num_classes, criterion, s2s4=None):
    return build("basic.HRNet", num_classes, criterion)


def HRNet_ASP(num_classes, criterion, s2s4=None):
    """network/basic.py:109-111."""
    return build("basic.HRNet_ASP", num_classes, criterion)
