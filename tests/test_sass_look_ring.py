"""ScanUniformLookRingKernel is what DESIGN.md says it is (cuobjdump -sass on pire_b200/libpire_b200.so; no GPU needed):
tables staged by TMA, input blocks copied into shared memory with LDGSTS and read back with LDS.128, the look-ahead walk
of two strings over two blocks per iteration, and no local memory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB),
                                reason="needs cuobjdump and the built library")


@pytest.fixture(scope="module")
def ring():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    bodies, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            bodies[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            bodies[name].append(line)
    hits = [("\n".join(v)) for k, v in bodies.items() if "ScanUniformLookRingKernel" in k]
    assert len(hits) == 1
    return hits[0]


def count(text, pattern):
    return len(re.findall(pattern, text))


def test_tables_by_tma_input_by_ldgsts_ring(ring):
    assert count(ring, r"\bUBLKCP") >= 1 and count(ring, r"\bSYNCS") >= 1        # cp.async.bulk + mbarrier
    assert count(ring, r"\bLDGSTS") >= 4                                          # two 16-byte copies per 32-byte block
    assert count(ring, r"\bLDS\.128") >= 8                                        # 2 strings x 2 halves x 2 blocks
    assert count(ring, r"\bLDG\.E\.[A-Z0-9.]*128") == 0                           # no register-fed input loads


def test_walk_is_the_look_ahead_step(ring):
    steps = count(ring, r"@!?P\d\s+LDS\.U8")
    assert steps == 128                                                           # 2 strings x 32 bytes x 2 blocks
    assert count(ring, r"\bIDP\.4A") >= steps
    assert steps // 2 <= count(ring, r"\bSHF\.L\.W") <= steps // 2 + 8
    assert steps // 2 <= count(ring, r"\bSHF\.R\.W") <= steps // 2 + 16
    assert count(ring, r"\bLOP3") < steps + 40


def test_no_local_memory(ring):
    assert count(ring, r"\b(STL|LDL)\b") == 0
