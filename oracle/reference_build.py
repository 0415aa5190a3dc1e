"""Recipe that places the unmodified reference checkout (NVIDIA/semantic-segmentation) under oracle/_ref/ for the
boundary test (tests/test_gpu_train_py.py runs its train.py on the overlay). oracle/_ref/ is git-ignored; the product
never imports it. The checkout is read from $SEG_REFERENCE_DIR (default: /root/reference); without one nothing is made
and the boundary test skips."""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref", "semantic-segmentation")


def build(src=None):
    src = src or os.environ.get("SEG_REFERENCE_DIR", "/root/reference")
    if os.path.isfile(os.path.join(src, "train.py")) and not os.path.isfile(os.path.join(DEST, "train.py")):
        os.makedirs(os.path.dirname(DEST), exist_ok=True)
        shutil.copytree(src, DEST, ignore=shutil.ignore_patterns(".git", "__pycache__", "imgs"), dirs_exist_ok=True)
    return DEST
