"""network.ocrnet factories (network/ocrnet.py:337-342) backed by the sm_90a kernels."""
from ._factory import build


def HRNet(num_classes, criterion):
    """OCRNet over HRNetV2-W48, single scale (network/ocrnet.py:94-122)."""
    return build("ocrnet.HRNet", num_classes, criterion)


def HRNet_Mscale(num_classes, criterion):
    """MscaleOCR: hierarchical multi-scale attention (network/ocrnet.py:158-334) — arch of every scripts/*.yml."""
    return build("ocrnet.HRNet_Mscale", num_classes, criterion)
