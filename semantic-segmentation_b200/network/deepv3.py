"""network.deepv3 factory (network/deepv3.py:165-170) backed by the sm_90a kernels (SURVEY.md §8 row f2)."""
from ._factory import build


def DeepV3PlusW38(num_classes, criterion):
    return build("deepv3.DeepV3PlusW38", num_classes, criterion)
