"""The kernel that finds where the matches start (pire_gpu_match_starts_string / _batch) is in the shipped library, and
the C ABI refuses a host-only handle.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds MatchStartsKernel
with the LDS.U8 table walk and the cp.async staging of the suffix scan, within the register and stack budget DESIGN.md
records for it (64 registers, the two-CTA-per-SM launch bound, and no stack)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

KERNEL = r"17MatchStartsKernelENS_8ScanArgsE"
MAX_REGISTERS = 64
MAX_STACK = 0


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


def test_kernel_walks_the_table_from_a_staging_ring(bodies):
    text = bodies[find(bodies, KERNEL)]
    assert re.search(r"\bLDS\.U8", text)                  # the table walk
    assert re.search(r"\bLDGSTS\b", text)                 # per-lane cp.async staging of the 16-byte chunks
    assert re.search(r"\bATOMG\.E\.ADD\.64\b", text)      # groups of 32 entries handed out by a counter


def test_register_and_stack_budget(usage):
    regs, stack = usage[find(usage, KERNEL)]
    assert regs <= MAX_REGISTERS and stack <= MAX_STACK, (regs, stack)


def test_host_only_handle_is_refused():
    import numpy as np
    from start_images import START_IMAGES
    from test_string_images import host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(START_IMAGES["edges"]["reversed"])
    found = np.ones(1, np.uint64)
    ends = np.zeros(4, np.uint64)
    starts = np.full(4, 7, np.uint64)
    rc = N.lib.pire_gpu_match_starts_string(sc._h, None, 0, 0, 0, 0, ends.ctypes.data, None, None, found.ctypes.data, 4,
                                            starts.ctypes.data, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    assert (starts == 7).all()
    rc = N.lib.pire_gpu_match_starts_batch(sc._h, None, None, 0, 1, None, 0, 0, None, ends.ctypes.data, None, None,
                                           found.ctypes.data, 4, starts.ctypes.data, None, None)
    assert rc == -4
    assert (starts == 7).all()
