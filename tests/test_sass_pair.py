"""The kernel that scans a uniform batch for two scanners at once (pire_gpu_run_pair_batch) is in the shipped library, and
the C ABI refuses a host-only handle.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds ScanPairKernel with
the tables staged by TMA, the input copied into a per-lane ring with LDGSTS and read back with LDS.128 once per block
for both scanners, two look-ahead LDS.U8 chains per byte, no stack, and registers within its launch bound (one CTA of
768 threads per SM: 80 registers)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

KERNEL = r"14ScanPairKernelENS0_8PairArgsE"
MAX_REGISTERS = 80          # 65536 registers / 768 threads, rounded down to the allocation unit of 8
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


def test_tables_by_tma_input_by_ldgsts_ring(body):
    assert count(body, r"\bUBLKCP") >= 2 and count(body, r"\bSYNCS") >= 2      # both scanners' tables: cp.async.bulk + mbarrier
    assert count(body, r"\bLDGSTS") >= 4                                       # two 16-byte copies per 32-byte block
    assert count(body, r"\bLDS\.128") == 4                                     # 2 halves x 2 blocks, shared by both chains
    assert count(body, r"\bLDG\.E\.[A-Z0-9.]*128") == 0                        # no register-fed input loads


def test_two_look_ahead_chains_per_byte(body):
    steps = count(body, r"@!?P\d\s+LDS\.U8")
    assert steps == 128                                                        # 32 bytes x 2 blocks x 2 scanners
    assert count(body, r"\bIDP\.4A") >= steps
    assert steps // 2 <= count(body, r"\bSHF\.L\.W") <= steps // 2 + 16
    assert count(body, r"\bVOTE\.ALL\b") == 1                                   # the NoExit exit of the warp


def test_register_and_stack_budget():
    for line in _cuobjdump("-res-usage").split("Function ")[1:]:
        if re.match(r"\S*" + KERNEL, line):
            m = re.search(r"\bREG:(\d+).*\bSTACK:(\d+)", line)
            regs, stack = int(m.group(1)), int(m.group(2))
            assert regs <= MAX_REGISTERS and stack <= MAX_STACK, (regs, stack)
            return
    raise AssertionError("ScanPairKernel not in the resource usage")


def test_no_local_memory(body):
    assert count(body, r"\b(STL|LDL)\b") == 0


def test_host_only_handle_is_refused():
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    host = P.Scanner(W.load_image("headline"), -1)
    assert N.lib.pire_gpu_run_pair_batch(host._h, host._h, None, None, 0, 0, 3, None, None, None, None, None, None, None, None,
                                         None) == -4                         # PIRE_GPU_ENODEVICE, before anything else
    assert N.lib.pire_gpu_run_pair_batch(host._h, None, None, None, 0, 0, 3, None, None, None, None, None, None, None, None, None) == -4
    assert N.lib.pire_gpu_run_pair_batch(None, host._h, None, None, 0, 0, 3, None, None, None, None, None, None, None, None, None) == -1
