"""tools/pigrep.py with Pire::SlowScanner images: the printed lines are those the reference's SlowScanner accepts (its
recorded answers in tests/golden/slow_images.json.xz, Runner(sc).Begin().Run(line).End() per line, which is
samples/pigrep/pigrep.cpp's loop), from a file read in many small blocks and from standard input; -o and a second
--scanner are refused with a message."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from slow_fixtures import SLOW

PIGREP = os.path.join(ROOT, "tools", "pigrep.py")
NAMES = ["heavy/ab20cd20", "heavy/d3_50_d3", "heavy/foo64bar", "heavy/error200", "approx1"]


def entry(name):
    return next(e for e in SLOW if e.name == name)


def pigrep(args, stdin=None):
    return subprocess.run([sys.executable, PIGREP] + args, input=stdin, capture_output=True, timeout=600)


def test_refusals(tmp_path):
    slow = tmp_path / "slow.pire"
    slow.write_bytes(entry("heavy/a30").image)
    text = tmp_path / "t.txt"
    text.write_bytes(b"abc\n")
    for args in (["--scanner", str(slow), "--scanner", str(slow), str(text)], ["--scanner", str(slow), "-o", str(text)]):
        out = pigrep(args)
        assert out.returncode == 2 and b"DFA" in out.stderr, out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_lines_equal_reference(tmp_path, cuda_device, name):
    e = entry(name)
    assert not any(b"\n" in s for s in e.strings)
    final, _ = e.runs[(True, True, False)]
    image = tmp_path / "slow.pire"
    image.write_bytes(e.image)
    rng = np.random.default_rng(9)
    order = rng.integers(0, len(e.strings), 4000)           # ~1 MiB of lines
    lines = [e.strings[k] for k in order]
    text = b"\n".join(lines) + b"\n"
    path = tmp_path / "text.txt"
    path.write_bytes(text)
    want = [(i, l) for i, (k, l) in enumerate(zip(order, lines)) if final[k]]
    expect = b"".join(b"%d:%s\n" % (i + 1, l) for i, l in want)
    got = pigrep(["--scanner", str(image), "-n", "--block-mb", "0.01", str(path)])
    assert got.returncode == 0, got.stderr
    assert got.stdout == expect
    got = pigrep(["--scanner", str(image), "-c"], stdin=text)
    assert got.returncode == 0 and got.stdout == b"%d\n" % len(want), got.stderr
    pos = np.concatenate([[0], np.cumsum([len(l) + 1 for l in lines])])
    got = pigrep(["--scanner", str(image), "-b", "-"], stdin=text)
    assert got.stdout == b"".join(b"%d:%s\n" % (pos[i], l) for i, l in want)
