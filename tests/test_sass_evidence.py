"""The shipped library is what DESIGN.md says it is: sm_90a cubins only, and the instructions the design argues from
are in the kernels that are supposed to have them (cuobjdump -sass on pire_b200/libpire_b200.so; no GPU needed).
Counts move with every compiler version, so the assertions are about presence and proportion, not exact numbers."""
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
def kernels():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    arch = set(re.findall(r"arch = (sm_\w+)", out))
    body, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            body[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            body[name].append(line)
    return arch, {k: "\n".join(v) for k, v in body.items() if "cub" not in k}


def pick(kernels, *needles):
    hits = [text for name, text in kernels[1].items() if all(n in name for n in needles)]
    assert hits, needles
    return hits


def count(text, pattern):
    return len(re.findall(pattern, text))


def test_only_hopper_code(kernels):
    assert kernels[0] == {"sm_90a"}
    for text in kernels[1].values():
        assert not re.search(r"\b(HMMA|IMMA|WGMMA|UTC\w*MMA)", text)          # no contraction on this path: no tensor cores


def test_tables_are_staged_by_tma_and_walked_from_shared_memory(kernels):
    for needle in ("ScanUniformKernel", "ScanGenericKernel", "ScanSplitKernel", "ScanTextKernel",
                   "PrefixKernel", "PrefixUniformKernel", "11CountKernel"):
        for text in pick(kernels, needle):
            assert count(text, r"\bUBLKCP") >= 1 and count(text, r"\bSYNCS") >= 1, needle       # cp.async.bulk + mbarrier
            assert count(text, r"\bLDS\.U8") >= 16, needle                                       # one table read per byte


def test_uniform_kernels_stream_with_128_bit_load_pairs_and_the_csr_kernels_with_ldgsts(kernels):
    for needle in ("ScanUniformKernel", "ScanUniformLookKernel", "PrefixUniformKernel", "ScanSplitKernel"):
        for text in pick(kernels, needle):
            assert count(text, r"\bLDG\.E\.[A-Z0-9.]*128") >= 4, needle                    # two per 32-byte sector
            assert count(text, r"\bLDGSTS") == 0, needle
    for text in pick(kernels, "ScanGenericKernel"):
        assert count(text, r"\bLDGSTS") >= 4

