"""The kernel that lists where the matches end in the lines of a text (pire_gpu_match_ends_lines) is in the shipped
library, and a host-only handle is refused.  No GPU needed: cuobjdump on pire_b200/libpire_b200.so finds
MatchEndsTextKernel for both walks (counting the entries, writing them), each with the LDS.U8 table walk, within the
register budget of its launch bound (two CTAs of 512 threads per SM: 64 registers), with no stack and no spills, and
MatchStartsLinesKernel, the line-window walk of MatchStartsKernel, beside it."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")

# MatchEndsTextKernel<kWrite> (Itanium mangling)
WALKS = {"count": r"19MatchEndsTextKernelILb0EEEvNS_8ScanArgsE", "write": r"19MatchEndsTextKernelILb1EEEvNS_8ScanArgsE"}
STARTS = {"batch": r"17MatchStartsKernelENS_8ScanArgsE", "lines": r"22MatchStartsLinesKernelENS_8ScanArgsE"}
MAX_REGISTERS = 64


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


@pytest.mark.parametrize("walk", sorted(WALKS))
def test_kernel_walks_the_table(walk, bodies):
    body = bodies[find(bodies, WALKS[walk])]
    assert re.search(r"\bLDS\.U8", body)
    assert not re.search(r"\b(LDL|STL)\b", body), "local memory in %s" % walk


@pytest.mark.parametrize("walk", sorted(WALKS))
def test_register_and_stack_budget(walk, usage):
    regs, stack = usage[find(usage, WALKS[walk])]
    assert regs <= MAX_REGISTERS and stack == 0, (walk, regs, stack)


@pytest.mark.parametrize("form", sorted(STARTS))
def test_match_starts_instantiations(form, usage):
    regs, stack = usage[find(usage, STARTS[form])]
    assert regs <= MAX_REGISTERS and stack == 0, (form, regs, stack)


def test_no_spills_in_ptxas_log():
    """The build's ptxas log, when it is there: the new kernels spill nothing."""
    log = os.path.join(ROOT, "build", "ptxas_libpire_b200.so.log")
    if not os.path.exists(log):
        pytest.skip("needs the build's ptxas log")
    text = open(log).read()
    for pattern in list(WALKS.values()) + [STARTS["lines"]]:
        m = re.search(r"Function properties for \S*%s\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                      % pattern, text)
        assert m, pattern
        assert m.groups() == ("0", "0", "0"), (pattern, m.groups())


def test_host_only_handle_is_refused():
    from test_string_images import STRING_IMAGES, host_scanner
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    found = np.zeros(1, np.uint64)
    ends = np.zeros(4, np.uint64)
    offs = np.array([0, 2], np.uint64)
    text = np.frombuffer(b"a\n", np.uint8)
    rc = N.lib.pire_gpu_match_ends_lines(sc._h, text.ctypes.data, offs.ctypes.data, 1, 0, None, ends.ctypes.data, None, 4,
                                         found.ctypes.data, None, None, None)
    assert rc == -4                     # PIRE_GPU_ENODEVICE
    lines = np.zeros(4, np.uint32)
    starts = np.zeros(4, np.uint64)
    rc = N.lib.pire_gpu_match_starts_lines(sc._h, text.ctypes.data, offs.ctypes.data, 1, 0, 0, lines.ctypes.data, ends.ctypes.data,
                                           None, None, found.ctypes.data, 4, starts.ctypes.data, None, None)
    assert rc == -4
    assert not found.any() and not ends.any() and not starts.any()
    import pire_b200 as P
    with pytest.raises((N.PireGpuError, RuntimeError, ValueError)):
        P.LineMatchEnds(sc, 4)
