"""The kernels that count a batch from given states (pire_gpu_count_batch_from) are in the shipped library, and the C ABI
refuses a host-only handle.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds CountKernel<kWords, kAlways,
true> for every counter form the launch chooses between (accept lists; packed one or two words, behind the look-ahead
pass or on every chunk), each with the LDS.U8 table walk, and none using more stack than CountKernel<kWords, kAlways>,
the batch kernel of the same form that pire_gpu_count_batch runs."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

# CountKernel<kWords, kAlways, kFrom> (Itanium mangling)
FORMS = {
    "lists": "ILi0ELb0E",
    "packed1": "ILi1ELb0E",
    "packed1, every chunk": "ILi1ELb1E",
    "packed2": "ILi2ELb0E",
    "packed2, every chunk": "ILi2ELb1E",
}


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
def stack():
    out, name = {}, None
    for line in _cuobjdump("-res-usage").splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"\bSTACK:(\d+)", line)
        if name and m:
            out[name] = int(m.group(1))
            name = None
    return out


def find(names, pattern):
    hits = [k for k in names if re.search(pattern, k)]
    assert len(hits) == 1, (pattern, hits)
    return hits[0]


def test_one_kernel_per_counter_form(bodies, stack):
    assert len([k for k in bodies if re.search(r"11CountKernelI.*Lb1EEEv", k)]) == len(FORMS)
    for what, form in FORMS.items():
        new = find(bodies, r"11CountKernel%sLb1EEEv" % form)
        old = find(bodies, r"11CountKernel%sLb0EEEv" % form)
        assert re.search(r"\bLDS\.U8", bodies[new]), what                 # the table walk
        assert stack[new] <= stack[old], (what, stack[new], stack[old])


def test_host_only_handle_is_refused():
    import numpy as np
    from test_string_images import STRING_IMAGES, host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    counts = np.zeros(4, np.uint64)
    rc = N.lib.pire_gpu_count_batch_from(sc._h, None, None, 0, 1, 0, None, counts.ctypes.data, None, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    assert not counts.any()
