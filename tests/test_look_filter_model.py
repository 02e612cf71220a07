"""The look-ahead exit filters on the CPU: the host model (tools/model_look.cpp) walks the glued benchmark scanner over
synthetic text with every slot function the kernels use -- byte & 31 (LOOK), byte & 63 (LOOK64) -- and with the ones that
were tried and dropped (a multiplicative hash whose multiplier is searched per automaton, the LOOKH experiment, also
with only the even positions hashed), and compares the end state of every string with the plain walk.  A filter that
drops a byte it must not drop shows up as a mismatch here, before any GPU sees it.  The model also counts shared-memory
wavefronts per step: the numbers the choice of filter argues from (the hashed filter is sharper, and its kernel was
slower all the same)."""
import lzma
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANTS = ["$ABCDEFGHIJKLMNOPQRSTUVWXYZ", "$XABCDEFGHIJKLMNOPQRSTUVWXYZ", "$ABCDEFGHIJKLMNOPQRSTUVWXYZ", "$(555) 123-4567",
          "$hello \t world", "error", "fatal", "https://", "^GET ", "$timeout"]

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("model_look")
    exe = str(tmp / "model_look")
    src = [os.path.join(ROOT, "tools", "model_look.cpp"), os.path.join(ROOT, "pire_b200", "csrc", "pire_image.cpp"),
           os.path.join(ROOT, "pire_b200", "csrc", "dfa_tables.cpp")]
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe] + src, check=True)
    image = str(tmp / "glue10.pire")
    with open(os.path.join(ROOT, "pire_b200", "data", "glue10.pire.xz"), "rb") as f, open(image, "wb") as g:
        g.write(lzma.decompress(f.read()))
    return exe, image


def run_model(model, n, length, base=None):
    exe, image = model
    env = dict(os.environ)
    if base is not None:
        env["MODEL_BASE"] = str(base)
    out = subprocess.run([exe, image, str(n), str(length)] + PLANTS, capture_output=True, text=True, check=True, env=env).stdout
    rows = {}
    for line in out.splitlines():
        m = re.match(r"(\S.*?)\s+now: ([\d.]+) wf .*\| look: ([\d.]+) wf ([\d.]+) act .* end-state mismatches (\d+)", line)
        if m:
            rows[m.group(1)] = (float(m.group(2)), float(m.group(3)), float(m.group(4)), int(m.group(5)))
    return out, rows


@pytest.mark.parametrize("base", [1024, 2048, 33792])
def test_every_filter_is_exact_and_the_hashed_one_is_sharper(model, base):
    out, rows = run_model(model, 2048, 256, base)
    assert "lookahead ok" in out
    assert len(rows) >= 6, out
    for name, (_, _, _, mismatches) in rows.items():
        assert mismatches == 0, (name, out)
    hashed = [k for k in rows if k.startswith("mulhi32F") and "even" not in k]
    half = [k for k in rows if k.startswith("mulhi32F") and "even" in k]
    assert len(hashed) == 1 and len(half) == 1, out
    folded, exact = rows["b&31"], rows["exact256"]
    # wavefronts per step with look-ahead: exact <= hashed < even-bytes-only < folded, whatever the table's address
    assert exact[1] <= rows[hashed[0]][1] < rows[half[0]][1] < folded[1], out
    assert rows[hashed[0]][1] < 0.9 * folded[1], out
    # how many of the 95 printable bytes pass the hashed filter (the folded one passes 51 for this automaton)
    m = re.search(r"passes (\d+) of 95, folded filter", out)
    assert m and int(m.group(1)) <= 36, out
