"""The kernel that counts one string over the whole grid (pire_gpu_count_string) is in the shipped library, and the C ABI
refuses a host-only handle.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds one instantiation per counter
form the launch chooses between (accept lists; packed one or two words, behind the look-ahead pass or on every chunk),
each with the LDS.U8 table walk, the grid barrier and the 64-bit atomics into the caller's counters.  None but the
two-word form without the look-ahead pass uses local memory; that one spills a few words in its counting loop, as the
batch kernel of the same form does (CountKernel<2, false>)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

# CountStringKernel<kWords, kAlways> (Itanium mangling)
COUNT_STRING_KERNELS = {
    "lists": r"17CountStringKernelILi0ELb0EE",
    "packed1": r"17CountStringKernelILi1ELb0EE",
    "packed1, every chunk": r"17CountStringKernelILi1ELb1EE",
    "packed2": r"17CountStringKernelILi2ELb0EE",
    "packed2, every chunk": r"17CountStringKernelILi2ELb1EE",
}
SPILLS = {"packed2"}


@pytest.fixture(scope="module")
def bodies():
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    body, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            body[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            body[name].append(line)
    return {k: "\n".join(v) for k, v in body.items()}


def find(bodies, pattern):
    hits = [k for k in bodies if re.search(pattern, k)]
    assert len(hits) == 1, (pattern, hits)
    return hits[0]


def test_one_kernel_per_counter_form(bodies):
    assert len([k for k in bodies if "CountStringKernel" in k]) == len(COUNT_STRING_KERNELS)
    for what, pattern in COUNT_STRING_KERNELS.items():
        text = bodies[find(bodies, pattern)]
        assert re.search(r"\bLDS\.U8", text), what                       # the table walk
        assert re.search(r"\bREDG\.E\.ADD\.64", text), what           # the u64 counters
        if what not in SPILLS:
            assert not re.search(r"\b(STL|LDL)\b", text), what


def test_host_only_handle_is_refused():
    import numpy as np
    from test_string_images import STRING_IMAGES, host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    counts = np.zeros(4, np.uint64)
    rc = N.lib.pire_gpu_count_string(sc._h, None, 0, 0, None, counts.ctypes.data, None, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    assert not counts.any()
