"""Compiled-code guard for the forward / data-gradient convolutions (host only: reads the built library with cuobjdump).

Every instantiation of conv3x3_halo_kernel and conv_igemm_kernel must keep its fp32 accumulators in registers and keep
wgmma pipelined:
  * no stack frame;
  * no local-memory traffic between its first and last HGMMA;
  * no HGMMA that is immediately waited on (WARPGROUP.DEPBAR.LE gsb0, 0x0), except the function's last one, which may
    precede the end-of-tile drain;
  * no two HGMMA in a row that each end a group (gsb0) with a WARPGROUP.ARRIVE but neither a wgmma wait
    (WARPGROUP.DEPBAR) nor an unconditional branch between them: every group of these kernels is followed by a wait
    (reached directly or through a branch to the join of the K-step variants), so such a pair is one group split into
    single-MMA groups by an injected arrive, which ptxas does (warning C7519) when it cannot keep the accumulators of an MMA in
    flight in the registers the MMA names.
An MMA whose width, accumulator offset or K-step count is decided at run time between the fence and the commit of its
group breaks these.

The widest Cout tiles still keep a few bytes of spill next to their 128 (OCC 1) or 64 (OCC 2) accumulator registers,
all of it outside the MMA region except in halo <2, 8> (ptxas -v, stack / spill stores / spill loads in bytes):
halo <1, 16> 8 / 12 / 16, halo <2, 7> 16 / 16 / 68, halo <2, 8> 48 / 88 / 176, igemm <1, 16> 16 / 20 / 20,
igemm <2, 7> 8 / 16 / 16, igemm <2, 8> 64 / 288 / 412. halo <2, 8> is never launched: at BN 128 only three weight-ring
slots fit in half an SM, and halo_smem_layout asks for four before it picks two CTAs per SM. SPILLING lists these
six, and the test fails when one of them stops spilling so that the list stays exact."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "semantic-segmentation_b200", "b200seg", "lib", "libb200seg.so")
KERNELS = ("conv3x3_halo_kernel", "conv_igemm_kernel")
# (OCC, NB16) instantiations each kernel must have: NB16 = BN / 16, the co-resident build only up to 128 columns
EXPECTED = {(1, nb) for nb in range(1, 17)} | {(2, nb) for nb in range(1, 9)}
# (kernel, OCC, NB16) with a stack frame (and, for halo <2, 8>, which the planner never selects, local-memory traffic
# inside the MMA region)
SPILLING = {("conv3x3_halo_kernel", 1, 16), ("conv3x3_halo_kernel", 2, 8), ("conv3x3_halo_kernel", 2, 7),
            ("conv_igemm_kernel", 1, 16), ("conv_igemm_kernel", 2, 8), ("conv_igemm_kernel", 2, 7)}


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                         "cuobjdump")):
        if cand and os.access(cand, os.X_OK):
            return cand
    return None


def _kernel(name):
    return next((k for k in KERNELS if k in name), None)


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
        if _kernel(name):
            sass[name.strip()] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)
    stack = {m.group(1): int(m.group(2))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", run("-res-usage")) if _kernel(m.group(1))}
    assert sass and set(sass) == set(stack), (sorted(sass), sorted(stack))
    return sass, stack


def _hgmma(ops):
    return [i for i, op in enumerate(ops) if "HGMMA" in op]


def _config(name):
    m = re.search(r"(conv3x3_halo_kernel|conv_igemm_kernel)ILi(\d+)ELi(\d+)E", name)
    return (m.group(1), int(m.group(2)), int(m.group(3))) if m else (_kernel(name), 0, 0)


def test_every_configuration_is_instantiated(dump):
    for kernel in KERNELS:
        # mangled: <kernel>ILi<OCC>ELi<NB16>E
        got = {tuple(int(v) for v in m.groups()) for n in dump[1]
               for m in [re.search(kernel + r"ILi(\d+)ELi(\d+)E", n)] if m}
        assert got == EXPECTED, (kernel, sorted(got))


def test_conv_kernels_have_no_stack_frame(dump):
    _, stack = dump
    framed = {_config(n) for n, s in stack.items() if s}
    assert framed == SPILLING, (sorted(framed - SPILLING), sorted(SPILLING - framed))


def test_conv_mma_loop_has_no_local_memory_traffic(dump):
    bad = {}
    for name, ops in dump[0].items():
        mma = _hgmma(ops)
        assert mma, name
        local = [op for op in ops[mma[0]:mma[-1]] if re.match(r"(@!?U?P\w+\s+)?(STL|LDL)\b", op)]
        if local and _config(name) != ("conv3x3_halo_kernel", 2, 8):
            bad[name] = len(local)
    assert bad == {}


def test_conv_mma_is_not_waited_on_one_by_one(dump):
    bad = {}
    for name, ops in dump[0].items():
        mma = _hgmma(ops)
        serial = 0
        for i in mma[:-1]:
            nxt = next((op for op in ops[i + 1:] if op.strip() != "NOP"), "")
            if re.match(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0$", nxt.strip()):
                serial += 1
        if serial:
            bad[name] = "%d of %d HGMMA waited on immediately" % (serial, len(mma))
    assert bad == {}


def test_conv_mma_group_has_no_injected_arrive(dump):
    # Narrower than "no arrive inside a group", because SASS does not mark where a source group starts: the K-step
    # variants are laid out one after another, so the last HGMMA of one variant (gsb0, then a branch to the wait at the
    # join) is followed by the first of the next. An injected arrive makes every MMA its own gsb0 group with no wait
    # before the next one, which is what this looks for; it flags 12 of 49 and 14 of 57 HGMMA pairs in the
    # run-time-width igemm builds these kernels replaced.
    bad = {}
    for name, ops in dump[0].items():
        mma = _hgmma(ops)
        injected = sum(1 for i, j in zip(mma, mma[1:])
                       if re.search(r"\bgsb0\b", ops[i]) and re.search(r"\bgsb0\b", ops[j])
                       and any("WARPGROUP.ARRIVE" in op for op in ops[i + 1:j])
                       and not any("WARPGROUP.DEPBAR" in op or op.startswith("BRA ") for op in ops[i + 1:j]))
        if injected:
            bad[name] = "%d of %d HGMMA followed by an arrive inside their group" % (injected, len(mma))
    assert bad == {}
