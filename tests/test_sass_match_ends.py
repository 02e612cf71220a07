"""The kernel that lists where the matches of one string end (pire_gpu_match_ends_string) is in the shipped library, and
the C ABI refuses a host-only handle.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds MatchEndsStringKernel
with the LDS.U8 table walk and one grid barrier more than CountStringKernel (the scan of the lanes' entry counts),
within the register and stack budget DESIGN.md records for it (64 registers, the two-CTA-per-SM launch bound, and 8
bytes of stack)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

KERNEL = r"21MatchEndsStringKernelENS_8ScanArgsE"
COUNT_STRING = r"17CountStringKernelILi0ELb0EE"
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


def test_kernel_walks_the_table_and_syncs_the_grid_once_more(bodies):
    text = bodies[find(bodies, KERNEL)]
    assert re.search(r"\bLDS\.U8", text)                                    # the table walk
    grid_syncs = len(re.findall(r"\bMEMBAR\.ALL\.GPU\b", text))             # one per grid.sync() site
    assert grid_syncs == len(re.findall(r"\bMEMBAR\.ALL\.GPU\b", bodies[find(bodies, COUNT_STRING)])) + 1


def test_register_and_stack_budget(usage):
    regs, stack = usage[find(usage, KERNEL)]
    assert regs <= MAX_REGISTERS and stack <= MAX_STACK, (regs, stack)


def test_host_only_handle_is_refused():
    import numpy as np
    from test_string_images import STRING_IMAGES, host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    found = np.zeros(1, np.uint64)
    ends = np.zeros(4, np.uint64)
    rc = N.lib.pire_gpu_match_ends_string(sc._h, None, 0, 0, None, 0, ends.ctypes.data, None, 4, found.ctypes.data, None, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    assert not found.any() and not ends.any()
    import pire_b200 as P
    with pytest.raises(N.PireGpuError):
        P.StringMatchEnds(sc, 4).Begin().End()
