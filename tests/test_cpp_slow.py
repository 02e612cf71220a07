"""include/pire_gpu.hpp's SlowScanner compiled against the reference headers: the reference's own Pire::Step and
Pire::Runner instantiated on Pire::Gpu::SlowScanner and on Pire::SlowScanner built from the same patterns must reach the
same state sets (tests/cpp/slow_check.cpp).  Needs the reference headers and oracle/_ref (library), so it runs where the
reference is built only; no GPU."""
import os
import subprocess

import pytest

from conftest import ROOT

REF = os.environ.get("PIRE_REF", "/root/reference")


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "pire")), reason="reference headers not present")
def test_slow_mirror_equals_reference(tmp_path):
    ref_so = os.path.join(ROOT, "oracle", "_ref", "libpire_ref.so")
    if not os.path.exists(ref_so):
        pytest.skip("oracle/_ref not built")
    exe = str(tmp_path / "slow_check")
    cmd = ["g++", "-std=c++11", "-O1", "-w", "-DPIRE_NO_CONFIG", "-include", "limits", "-I", REF, "-I", os.path.join(REF, "pire"),
           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "slow_check.cpp"),
           ref_so, os.path.join(ROOT, "pire_b200", "libpire_b200.so"), "-o", exe,
           "-Wl,-rpath," + os.path.dirname(ref_so), "-Wl,-rpath," + os.path.join(ROOT, "pire_b200")]
    subprocess.run(cmd, check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert " 0 mismatches" in out.stdout
