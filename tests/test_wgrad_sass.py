"""Compiled-code guard for the weight-gradient convolution (host only: reads the built library with cuobjdump).

Every instantiation of wgrad_igemm_kernel must keep its fp32 accumulators in registers and keep wgmma pipelined: no
stack frame, no local-memory traffic between its first and last HGMMA, and no HGMMA that is immediately waited on
(WARPGROUP.DEPBAR.LE gsb0, 0x0) except the function's last one, which may precede the end-of-unit drain. An MMA whose
width or accumulator offset is decided at run time breaks all three."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "semantic-segmentation_b200", "b200seg", "lib", "libb200seg.so")
KERNEL = "wgrad_igemm_kernel"


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                         "cuobjdump")):
        if cand and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.fixture(scope="module")
def dump():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")

    def run(flag):
        return subprocess.run([tool, flag, LIB], capture_output=True, text=True, check=True).stdout

    sass = {}
    for chunk in re.split(r"\n\s*Function : ", run("-sass"))[1:]:
        name, body = chunk.split("\n", 1)
        if KERNEL in name:
            sass[name.strip()] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    stack = {m.group(1): int(m.group(2))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", run("-res-usage")) if KERNEL in m.group(1)}
    assert sass and set(sass) == set(stack), (sorted(sass), sorted(stack))
    return sass, stack


def test_wgrad_kernels_have_no_stack_frame(dump):
    _, stack = dump
    assert {n: s for n, s in stack.items() if s} == {}


def test_wgrad_mma_loop_has_no_local_memory_traffic(dump):
    bad = {}
    for name, ops in dump[0].items():
        mma = [i for i, op in enumerate(ops) if "HGMMA" in op]
        assert mma, name
        local = [op for op in ops[mma[0]:mma[-1]] if re.match(r"(@!?U?P\w+\s+)?(STL|LDL)\b", op)]
        if local:
            bad[name] = len(local)
    assert bad == {}


def test_wgrad_mma_is_not_waited_on_one_by_one(dump):
    bad = {}
    for name, ops in dump[0].items():
        mma = [i for i, op in enumerate(ops) if "HGMMA" in op]
        serial = 0
        for i in mma[:-1]:
            nxt = next((op for op in ops[i + 1:] if op.strip() != "NOP"), "")
            if re.match(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0$", nxt.strip()):
                serial += 1
        if serial:
            bad[name] = "%d of %d HGMMA waited on immediately" % (serial, len(mma))
    assert bad == {}
