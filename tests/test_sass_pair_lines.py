"""The kernel that walks the lines of a text for two scanners at once (pire_gpu_run_pair_lines) is in the shipped library,
with no stack, no local memory and registers within its launch bound (one CTA of 512 threads per SM: 128 registers).  No
GPU needed: cuobjdump on pire_b200/libpire_b200.so."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

KERNEL = r"18ScanTextPairKernelENS0_8PairArgsE"
MAX_REGISTERS = 128         # 65536 registers / 512 threads
MAX_STACK = 0


def _cuobjdump(*args):
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built library")
    return subprocess.run(["cuobjdump", *args, LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def body():
    bodies, name = {}, None
    for line in _cuobjdump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            bodies[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            bodies[name].append(line)
    hits = [k for k in bodies if re.search(KERNEL, k)]
    assert len(hits) == 1, hits
    return "\n".join(bodies[hits[0]])


def count(text, pattern):
    return len(re.findall(pattern, text))


def test_two_chains_per_byte_one_load_per_block(body):
    assert count(body, r"\bUBLKCP") >= 2                                       # both scanners' tables by TMA
    assert count(body, r"@!?P\d\s+LDS\.U8") >= 64                              # 32 bytes x 2 chains, exit-filtered
    assert count(body, r"\bLDG\.E\.[A-Z0-9.]*128") == 4                        # first and next block: two LDG.128 each, shared


def test_register_and_stack_budget():
    for line in _cuobjdump("-res-usage").split("Function ")[1:]:
        if re.match(r"\S*" + KERNEL, line):
            m = re.search(r"\bREG:(\d+).*\bSTACK:(\d+)", line)
            regs, stack = int(m.group(1)), int(m.group(2))
            assert regs <= MAX_REGISTERS and stack <= MAX_STACK, (regs, stack)
            return
    raise AssertionError("ScanTextPairKernel not in the resource usage")


def test_no_local_memory(body):
    assert count(body, r"\b(STL|LDL)\b") == 0
