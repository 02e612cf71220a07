"""The kernels that start every string from its own state (pire_gpu_run_batch_from) are in the shipped library
(cuobjdump on pire_b200/libpire_b200.so; no GPU needed): one instantiation per kernel the batch entry points launch, none
using local memory, and the one-string ring kernel within the 64 registers of its one CTA of 1024 threads."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB),
                                reason="needs cuobjdump and the built library")

# the kStarts instantiations (Itanium mangling: Lb1E = true as the last template argument), and the ring kernel's own name
STARTS_KERNELS = {
    "ScanUniformKernel<plain>": r"17ScanUniformKernelILb0ELb1EE",
    "ScanUniformKernel<pred>": r"17ScanUniformKernelILb1ELb1EE",
    "ScanUniformLookKernel<look1>": r"21ScanUniformLookKernelILb0ELi48ELb1ELb1EE",
    "ScanUniformLookKernel<look64>": r"21ScanUniformLookKernelILb1ELi48ELb0ELb1EE",
    "ScanUniformLookRingFromKernel": r"29ScanUniformLookRingFromKernel",
    "ScanUniformLookRing1Kernel": r"26ScanUniformLookRing1KernelILi3ELb1EE",
    "ScanGenericKernel<0>": r"17ScanGenericKernelILi0ELb1EE",
    "ScanGenericKernel<1>": r"17ScanGenericKernelILi1ELb1EE",
    "ScanGenericKernel<2>": r"17ScanGenericKernelILi2ELb1EE",
    "ScanSplitKernel<plain>": r"15ScanSplitKernelILb0ELb1EE",
    "ScanSplitKernel<pred>": r"15ScanSplitKernelILb1ELb1EE",
}


@pytest.fixture(scope="module")
def bodies():
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


def test_every_starts_kernel_exists(bodies):
    for what, pattern in STARTS_KERNELS.items():
        name = find(bodies, pattern)
        assert re.search(r"\bLDS\.U8", bodies[name]), what              # the table walk is there
        assert re.search(r"\bLDG\.E", bodies[name]), what               # and the start read


def test_no_local_memory_in_the_ring_kernels(bodies):
    for what in ("ScanUniformLookRingFromKernel", "ScanUniformLookRing1Kernel"):
        text = bodies[find(bodies, STARTS_KERNELS[what])]
        assert not re.search(r"\b(STL|LDL)\b", text), what


def test_ring1_starts_kernel_fits_64_registers():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    regs = None
    for k, line in enumerate(lines):
        if re.search(STARTS_KERNELS["ScanUniformLookRing1Kernel"], line):
            for follow in lines[k:k + 3]:
                m = re.search(r"REG:(\d+)", follow)
                if m:
                    regs = int(m.group(1))
                    break
            m = re.search(r"STACK:(\d+)", " ".join(lines[k:k + 3]))
            assert m and int(m.group(1)) == 0
            break
    assert regs is not None and regs <= 64, regs
