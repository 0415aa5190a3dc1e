"""network.basic factory (network/basic.py:104) backed by the sm_90a kernels (BASELINE config 1 plumbing model)."""
from ._factory import build


def HRNet(num_classes, criterion, s2s4=None):
    return build("basic.HRNet", num_classes, criterion)
