"""The kernels that list where the matches of a batch end (pire_gpu_match_ends_batch_from) are in the shipped library,
and a host-only handle is refused.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds MatchEndsBatchKernel
for both walks (counting the entries, writing them), each with the LDS.U8 table walk and within the register and stack
budget DESIGN.md records for them (64 registers, the generic kernels' launch bound, 8 bytes of stack)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

# MatchEndsBatchKernel<kWrite> (Itanium mangling)
WALKS = {"count": r"20MatchEndsBatchKernelILb0EEEvNS_8ScanArgsE", "write": r"20MatchEndsBatchKernelILb1EEEvNS_8ScanArgsE"}
MAX_REGISTERS = 64
MAX_STACK = 8


def _cuobjdump(*args):
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built library")
    return subprocess.run(["cuobjdump", *args, LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def bodies():
    body, name = {}, None
    for line in _cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            body[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            body[name].append(line)
    return {k: "\n".join(v) for k, v in body.items()}


@pytest.fixture(scope="module")
def usage():
    out, name = {}, None
    for line in _cuobjdump("-res-usage").splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"\bREG:(\d+).*\bSTACK:(\d+)", line)
        if name and m:
            out[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    return out


def find(names, pattern):
    hits = [k for k in names if re.search(pattern, k)]
    assert len(hits) == 1, (pattern, hits)
    return hits[0]


@pytest.mark.parametrize("walk", sorted(WALKS))
def test_kernel_walks_the_table(walk, bodies):
    assert re.search(r"\bLDS\.U8", bodies[find(bodies, WALKS[walk])])


@pytest.mark.parametrize("walk", sorted(WALKS))
def test_register_and_stack_budget(walk, usage):
    regs, stack = usage[find(usage, WALKS[walk])]
    assert regs <= MAX_REGISTERS and stack <= MAX_STACK, (walk, regs, stack)


def test_host_only_handle_is_refused():
    from test_string_images import STRING_IMAGES, host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    found = np.zeros(1, np.uint64)
    ends = np.zeros(4, np.uint64)
    rc = N.lib.pire_gpu_match_ends_batch_from(sc._h, None, None, 0, 1, 0, None, None, None, ends.ctypes.data, None, 4,
                                              found.ctypes.data, None, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    assert not found.any() and not ends.any()
    import pire_b200 as P
    with pytest.raises((N.PireGpuError, RuntimeError, ValueError)):
        P.BatchMatchEnds(sc, 1, 4).Begin().End()
