"""ScanUniformLookRing1Kernel is what DESIGN.md says it is (cuobjdump -sass on pire_b200/libpire_b200.so; no GPU needed):
tables staged by TMA, input blocks copied into shared memory with LDGSTS and read back with LDS.128, the look-ahead walk
of one string over two blocks per iteration, and no local memory."""
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
def ring1():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    bodies, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            bodies[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            bodies[name].append(line)
    hits = {k: "\n".join(v) for k, v in bodies.items() if "ScanUniformLookRing1Kernel" in k}
    assert hits and not any("ScanUniformLookRingKernel" in k for k in hits)
    return hits


def count(text, pattern):
    return len(re.findall(pattern, text))


def test_tables_by_tma_input_by_ldgsts_ring(ring1):
    for name, body in ring1.items():
        assert count(body, r"\bUBLKCP") >= 1 and count(body, r"\bSYNCS") >= 1, name       # cp.async.bulk + mbarrier
        assert count(body, r"\bLDGSTS") >= 4, name                                        # two 16-byte copies per 32-byte block
        assert count(body, r"\bLDS\.128") >= 4, name                                      # 2 halves x 2 blocks
        assert count(body, r"\bLDG\.E\.[A-Z0-9.]*128") == 0, name                         # no register-fed input loads


def test_walk_is_the_look_ahead_step(ring1):
    for name, body in ring1.items():
        steps = count(body, r"@!?P\d\s+LDS\.U8")
        assert steps == 64, name                                                          # 32 bytes x 2 blocks
        assert count(body, r"\bIDP\.4A") >= steps, name
        assert steps // 2 <= count(body, r"\bSHF\.L\.W") <= steps // 2 + 8, name
        assert steps // 2 <= count(body, r"\bSHF\.R\.W") <= steps // 2 + 16, name
        assert count(body, r"\bLOP3") < steps + 40, name


def test_no_local_memory(ring1):
    for name, body in ring1.items():
        assert count(body, r"\b(STL|LDL)\b") == 0, name
