"""The SlowScanner kernels (pire_gpu_slow_run_batch) are in the shipped library for every set width, with no stack, no
local memory and registers within their launch bounds (256 threads, three lane-path or four warp-path CTAs per SM).
No GPU needed: cuobjdump on pire_b200/libpire_b200.so."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

KERNELS = {  # mangled name -> register budget (65536 / (256 x CTAs per SM), rounded down to a multiple of 8)
    "SlowLaneKernelILi1EEEvNS_8SlowArgsE": 80,
    "SlowLaneKernelILi2EEEvNS_8SlowArgsE": 80,
    "SlowLaneKernelILi4EEEvNS_8SlowArgsE": 80,
    "SlowLaneKernelILi8EEEvNS_8SlowArgsE": 80,
    "SlowWarpKernelILi1EEEvNS_8SlowArgsE": 64,
    "SlowWarpKernelILi2EEEvNS_8SlowArgsE": 64,
    "SlowWarpKernelILi4EEEvNS_8SlowArgsE": 64,
}


def _cuobjdump(*args):
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built library")
    return subprocess.run(["cuobjdump", *args, LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def bodies():
    out, name = {}, None
    for line in _cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            out[name].append(line)
    return out


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_no_local_memory(bodies, kernel):
    hits = [k for k in bodies if k.endswith(kernel)]
    assert len(hits) == 1, hits
    body = "\n".join(bodies[hits[0]])
    assert not re.search(r"\b(STL|LDL)\b", body)
    assert re.search(r"\bFLO\b|\bPOPC\b|\bBREV\b", body)          # the set bits are walked with __ffs


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_register_and_stack_budget(kernel):
    for line in _cuobjdump("-res-usage").split("Function ")[1:]:
        if re.match(r"\S*" + kernel, line):
            m = re.search(r"\bREG:(\d+).*\bSTACK:(\d+)", line)
            regs, stack = int(m.group(1)), int(m.group(2))
            assert regs <= KERNELS[kernel] and stack == 0, (regs, stack)
            return
    raise AssertionError(kernel + " not in the resource usage")
