"""pire_gpu_line_stream: a text fed from host memory in pieces, delivered as device frames of whole lines.

The framing answer is pire_gpu_split_lines over the whole text (and its host restatement, std::getline's lines): every
frame's offsets shifted by first_byte, its lines by first_line, give split_lines' offsets word for word, and each
frame's bytes are the text's.  The results answer is the same calls on the whole resident text: run_lines,
count_batch with LINES, match_ends_lines and match_starts_lines, shifted by the frame bases, over more than 1 GiB.
pigrep is checked against the reference compiled in oracle/_ref, run line by line."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from refpire import Ref, csr, have_ref
from start_images import START_IMAGES

pytestmark = pytest.mark.gpu

EINVAL, ENODEVICE = -1, -4
MIB = 1 << 20


def split_host(text):
    """std::getline's lines of `text` as pire_gpu_split_lines' offsets (a last line without '\\n' ends one past the text)."""
    t = np.frombuffer(bytes(text), np.uint8)
    offs = [0] + (np.nonzero(t == 10)[0] + 1).tolist()
    if len(t) and t[-1] != 10:
        offs.append(len(t) + 1)
    return offs


def split_device(text):
    import torch
    import pire_b200 as P
    if not text:
        return [0]
    dev = torch.frombuffer(bytearray(text), dtype=torch.uint8).to("cuda:0")
    return P.Batch.from_text(dev).offsets.cpu().tolist()


def as_input(piece, kind):
    import torch
    if kind == "bytes":
        return bytes(piece)
    if kind == "numpy":
        return np.frombuffer(bytes(piece), np.uint8).copy()
    pinned = torch.empty(len(piece), dtype=torch.uint8, pin_memory=True)
    if len(piece):
        pinned.copy_(torch.frombuffer(bytearray(piece), dtype=torch.uint8))
    return pinned


def stream_frames(pieces, slot_bytes, kind="bytes"):
    """Feeds the pieces (the last with last=True); returns every frame as (first_line, first_byte, offsets, bytes)."""
    import pire_b200 as P
    ls = P.LineStream(0, slot_bytes)
    out = []
    for k, piece in enumerate(pieces):
        for f in ls.feed(as_input(piece, kind), last=k == len(pieces) - 1):
            out.append((f.first_line, f.first_byte, f.offsets.cpu().tolist(), f.corpus.cpu().numpy().tobytes()))
            assert f.n == len(out[-1][2]) - 1 and f.n_bytes == len(out[-1][3])
    return out


def check_frames(text, frames):
    """The invariant: the frames, shifted, are split_lines of the whole text."""
    want = split_host(text)
    got, line = [0], 0
    for first_line, first_byte, offs, data in frames:
        assert first_line == line, "frames out of line order"
        assert offs[0] == 0 and first_byte == got[-1], "a frame does not start where the last one ended"
        assert data == bytes(text[first_byte:first_byte + len(data)]), "frame bytes differ from the text"
        assert offs[-1] - (0 if data.endswith(b"\n") or not data else 1) == len(data)
        got += [first_byte + o for o in offs[1:]]
        line += len(offs) - 1
    assert got == want


def cuts(rng, n, k):
    return sorted(rng.integers(0, n + 1, size=k).tolist())


def pieces_at(text, points):
    bounds = [0] + list(points) + [len(text)]
    return [text[a:b] for a, b in zip(bounds[:-1], bounds[1:])]


SHAPES = {
    "empty": b"",
    "one_newline": b"\n",
    "only_newlines": b"\n\n\n\n\n",
    "no_final_newline": b"abc\ndef\nghi",
    "final_newline": b"abc\ndef\nghi\n",
    "empty_lines": b"\n\nabc\n\n\ndef\n\n",
    "crlf": b"GET /a HTTP/1.1\r\nHost: x\r\n\r\nbody",
    "one_line": b"x" * 77,
}


def test_split_host_is_split_lines(cuda_device):
    rng = np.random.default_rng(5)
    for text in list(SHAPES.values()) + [bytes(rng.choice([10, 97, 98, 13], size=n).astype(np.uint8)) for n in (1, 31, 300)]:
        assert split_host(text) == split_device(text)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shapes_every_two_piece_split(cuda_device, name):
    text = SHAPES[name]
    for slot in (4, 16, 0):
        for at in range(len(text) + 1):
            check_frames(text, stream_frames(pieces_at(text, [at]), slot))


def test_every_two_piece_split_of_texts(cuda_device):
    rng = np.random.default_rng(7)
    for n in (37, 128, 300):
        text = bytes(rng.choice(np.frombuffer(b"ab c\n\r", np.uint8), size=n, p=[.3, .3, .15, .05, .15, .05]))
        for at in range(n + 1):
            check_frames(text, stream_frames(pieces_at(text, [at]), 64))


def test_random_many_piece_splits(cuda_device):
    """Zero-byte pieces, a zero-byte last piece, slots from 1 byte up."""
    rng = np.random.default_rng(11)
    for trial in range(60):
        n = int(rng.integers(0, 3000))
        text = bytes(rng.choice(np.frombuffer(b"abcdefgh \n", np.uint8), size=n))
        points = cuts(rng, n, int(rng.integers(0, 12)))
        if trial % 3 == 0:
            points += [points[-1] if points else 0] * 2           # zero-byte feeds
        if trial % 4 == 0:
            points.append(n)                                     # the last feed is empty
        slot = int(rng.choice([1, 7, 64, 256, 4096]))
        check_frames(text, stream_frames(pieces_at(text, sorted(points)), slot, ("bytes", "numpy", "pinned")[trial % 3]))


@pytest.mark.parametrize("kind", ["bytes", "numpy", "pinned"])
def test_inputs_and_long_lines(cuda_device, kind):
    """A line exactly one slot long (with and without its newline), lines of 100 KiB through 4 KiB slots (the slot
    grows), fed in pieces of several sizes from each kind of host memory."""
    rng = np.random.default_rng(13)
    slot = 4096
    exact = b"y" * (slot - 1) + b"\n" + b"z" * slot + b"\n" + b"w" * slot
    lines = [bytes(rng.integers(32, 127, size=int(rng.integers(0, 200))).astype(np.uint8)) for _ in range(200)]
    lines[50] = b"L" * (100 * 1024)
    lines[120] = b"M" * (100 * 1024 + 3)
    big = b"\n".join(lines)
    for text in (exact, big, big + b"\n"):
        for piece in (1000, 4096, 5000, 70000, len(text) or 1):
            points = list(range(piece, len(text), piece))
            check_frames(text, stream_frames(pieces_at(text, points), slot, kind))


def test_frame_is_a_line_batch(cuda_device):
    """A frame goes wherever Batch.from_text goes: Runner, LineMatchEnds, MatchStarts, HalfFinalCount."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    text = b"hello  world\nGET /x\n\nerror timeout\nhello\tworld"
    sc = P.Scanner(W.load_image("headline"), 0)
    e = START_IMAGES["glue10"]
    hf, rev = P.Scanner(e["forward"], 0), P.Scanner(e["reversed"], 0)
    whole = P.Batch.from_text(torch.frombuffer(bytearray(text), dtype=torch.uint8).to("cuda:0"))
    want = P.Runner(sc).Begin().Run(whole).End().Matches()
    counts = P.HalfFinalCount(hf, whole).counts
    got, got_counts = [], []
    for f in P.LineStream(0, 16).feed(text, last=True):
        assert isinstance(f, P.LineFrame) and f.trim == 1
        got += P.Runner(sc).Begin().Run(f).End().Matches().tolist()
        got_counts.append(P.HalfFinalCount(hf, f).counts)
        ends = P.LineMatchEnds(hf, 64).Begin().Run(f).End()
        P.MatchStarts(rev, ends, f).Starts()
    assert got == want.tolist()
    assert np.array_equal(np.concatenate(got_counts), counts)


def test_refusals(cuda_device):
    import ctypes as C
    import pire_b200 as P
    from pire_b200 import _native as N
    ls = P.LineStream(0)
    fr, got = N.LineFrame(), C.c_uint64(0)
    buf = b"abc\n"
    assert N.lib.pire_gpu_line_stream_feed(None, buf, 4, 0, None, C.byref(got), C.byref(fr)) == EINVAL
    assert N.lib.pire_gpu_line_stream_feed(ls._h, None, 4, 0, None, C.byref(got), C.byref(fr)) == EINVAL
    assert N.lib.pire_gpu_line_stream_feed(ls._h, buf, 4, 0, None, None, C.byref(fr)) == EINVAL
    assert N.lib.pire_gpu_line_stream_feed(ls._h, buf, 4, 0, None, C.byref(got), None) == EINVAL
    assert N.lib.pire_gpu_line_stream_feed(ls._h, buf, 4, 1, None, C.byref(got), C.byref(fr)) == 0
    assert got.value == 4 and fr.n_lines == 1
    assert N.lib.pire_gpu_line_stream_feed(ls._h, buf, 4, 0, None, C.byref(got), C.byref(fr)) == EINVAL
    assert b"after the last" in N.lib.pire_gpu_last_error()
    h = C.c_void_p()
    assert N.lib.pire_gpu_line_stream_create(-1, 0, C.byref(h)) == ENODEVICE and not h.value
    assert N.lib.pire_gpu_line_stream_create(1 << 20, 0, C.byref(h)) == ENODEVICE
    assert N.lib.pire_gpu_line_stream_create(0, 0, None) == EINVAL


# ---- results over a text larger than a GiB, streamed through 64 MiB slots, against the resident text -----------------

FLAG_SETS = [(False, False), (True, False), (False, True), (True, True)]


def planted_text(gib):
    """tools/string_bench.py's planted corpus, cut into lines of 80 to 120 bytes."""
    import torch
    from pire_b200 import workloads as W
    total = int(gib * 2 ** 30) // 1024 * 1024
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(total // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    rng = np.random.default_rng(2024)
    ends = np.cumsum(rng.integers(80, 121, size=total // 80 + 1))
    ends = ends[ends < total]
    dev[torch.from_numpy(ends).to("cuda:0")] = 10
    return dev


def unpack(words, n):
    import torch
    w = words.to(torch.int64) & 0xFFFFFFFF
    return ((w.unsqueeze(1) >> torch.arange(32, device=w.device)) & 1).flatten()[:n].to(torch.uint8)


def test_gib_text_equals_resident(cuda_device):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    dev = planted_text(1.0625)
    whole = P.Batch.from_text(dev)
    n = whole.n
    scanners = {name: P.Scanner(W.load_image(name), 0) for name in ("glue10", "headline")}
    e = START_IMAGES["glue10"]
    hf, rev = P.Scanner(W.load_image("hf_glue10"), 0), P.Scanner(e["reversed"], 0)
    assert W.load_image("hf_glue10") == e["forward"]

    def run(sc, batch, begin, end):
        flags = (N.RUN_BEGIN if begin else 0) | (N.RUN_END if end else 0)
        bits = torch.zeros((batch.n + 31) // 32, dtype=torch.int32, device="cuda:0")
        masks = torch.empty(batch.n, dtype=torch.int32, device="cuda:0")
        states = torch.empty(batch.n, dtype=torch.int32, device="cuda:0")
        sc.run_batch(batch, flags, bits, masks, states)
        return unpack(bits, batch.n), masks, states

    def spans(batch, begin, end):
        probe = P.LineMatchEnds(hf, 0)
        probe = (probe.Begin() if begin else probe).Run(batch)
        found = (probe.End() if end else probe).Found()
        m = P.LineMatchEnds(hf, found)
        m = (m.Begin() if begin else m).Run(batch)
        m = m.End() if end else m
        st = P.MatchStarts(rev, m, batch, begin=begin, end=end).StartsTensor()
        return (m.LinesTensor()[:found].to(torch.int64) & 0xFFFFFFFF, m.EndsTensor()[:found], m.IdsTensor()[:found],
                st[:found], m.StateTensor())

    want = {}
    for name, sc in scanners.items():
        for fl in FLAG_SETS:
            want[("run", name) + fl] = run(sc, whole, *fl)
    for fl in FLAG_SETS:
        want[("count",) + fl] = torch.from_numpy(P.HalfFinalCount(hf, whole, *fl).counts.astype(np.int64)).to("cuda:0")
        want[("ends",) + fl] = spans(whole, *fl)
    host = torch.empty(dev.numel(), dtype=torch.uint8, pin_memory=True)
    host.copy_(dev)
    del whole, dev
    torch.cuda.empty_cache()

    ls = P.LineStream(0, 64 * MIB)
    cursor = {fl: 0 for fl in FLAG_SETS}
    lines = frames = 0
    total = host.numel()
    points = [0, total // 3 + 17, 2 * total // 3 - 5, total]
    for k in range(3):
        for f in ls.feed(host[points[k]:points[k + 1]], last=k == 2):
            frames += 1
            lo, hi = f.first_line, f.first_line + f.n
            assert lo == lines
            for name, sc in scanners.items():
                for fl in FLAG_SETS:
                    bits, masks, states = run(sc, f, *fl)
                    wb, wm, ws = want[("run", name) + fl]
                    assert torch.equal(bits, wb[lo:hi]) and torch.equal(masks, wm[lo:hi]) and torch.equal(states, ws[lo:hi]), \
                        (name, fl, lo)
            for fl in FLAG_SETS:
                counts = torch.from_numpy(P.HalfFinalCount(hf, f, *fl).counts.astype(np.int64)).to("cuda:0")
                assert torch.equal(counts, want[("count",) + fl][lo:hi]), ("count", fl, lo)
                ln, en, ids, st, states = spans(f, *fl)
                wl, we, wi, ws, wst = want[("ends",) + fl]
                c, k2 = cursor[fl], ln.numel()
                assert torch.equal(ln + lo, wl[c:c + k2]) and torch.equal(en + f.first_byte, we[c:c + k2]), ("ends", fl, lo)
                assert torch.equal(ids, wi[c:c + k2]) and torch.equal(states, wst[lo:hi]), ("ids", fl, lo)
                none = st == -1
                assert torch.equal(none, ws[c:c + k2] == -1)
                assert torch.equal(st[~none] + f.first_byte, ws[c:c + k2][~none]), ("starts", fl, lo)
                cursor[fl] = c + k2
            lines = hi
    assert lines == n and frames >= 16
    for fl in FLAG_SETS:
        assert cursor[fl] == want[("ends",) + fl][0].numel()


# ---- pigrep ------------------------------------------------------------------------------------------------------------

PATTERN = rb"err(or)?|GET /[a-z]+|time ?out"


def pigrep(args, stdin=None):
    """tools/pigrep.py's main() in this process, with `stdin` (bytes) as its standard input; returns what it printed.
    (One case below runs the tool as its own process, reading a pipe.)"""
    import io
    if os.path.join(ROOT, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
    import pigrep as tool
    out = io.BytesIO()
    saved = sys.argv, sys.stdin, sys.stdout
    sys.argv = ["pigrep.py"] + list(args)
    stdout = io.TextIOWrapper(out, write_through=True)
    sys.stdin, sys.stdout = io.TextIOWrapper(io.BytesIO(stdin or b"")), stdout
    try:
        tool.main()
    finally:
        sys.argv, sys.stdin, sys.stdout = saved
        stdout.flush()
        stdout.detach()                  # the wrapper must not close `out` when it is collected
    return out.getvalue()


def pigrep_process(args, stdin):
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pigrep.py")] + args, input=stdin,
                         capture_output=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr.decode()
    return out.stdout


def grep_text(rng):
    words = [b"error", b"err", b"GET /index", b"timeout", b"time out", b"ok", b"hello", b"\r", b"", b"zz" * 300]
    lines = []
    for _ in range(400):
        k = int(rng.integers(0, 6))
        lines.append(b" ".join(words[int(i)] for i in rng.integers(0, len(words), size=k)))
    return b"\n".join(lines)


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref not built")
def test_pigrep_streams_files_and_stdin(tmp_path):
    """-c, -n, -b and their combinations on a file, on the same bytes through stdin and with blocks smaller than the
    longest line: byte for byte what the reference gives line by line."""
    rng = np.random.default_rng(3)
    data = grep_text(rng)
    path = tmp_path / "in.txt"
    path.write_bytes(data)
    lines = data.split(b"\n")
    offs = split_host(data)
    sc = Ref().compile(PATTERN)
    corpus, co = csr([data[offs[i]:offs[i + 1] - 1] for i in range(len(offs) - 1)])
    final, _, _ = sc.run(corpus, co)
    hits = np.nonzero(final)[0].tolist()
    assert 0 < len(hits) < len(lines)
    for opts in ([], ["-n"], ["-b"], ["-n", "-b"], ["-c"]):
        if opts == ["-c"]:
            want = b"%d\n" % len(hits)
        else:
            want = b"".join((b"%d:" % (i + 1) if "-n" in opts else b"") + (b"%d:" % offs[i] if "-b" in opts else b"")
                            + data[offs[i]:offs[i + 1] - 1] + b"\n" for i in hits)
        base = ["-e", PATTERN.decode()] + opts
        assert pigrep(base + [str(path)]) == want, opts
        assert pigrep(base, stdin=data) == want, opts
        assert pigrep(base + ["--block-mb", str(100 / MIB), "-"], stdin=data) == want, opts
        assert pigrep(base + ["--block-mb", str(37 / MIB), str(path)]) == want, opts
    # several inputs, one of them a pipe into the tool's own process: the reference's prefixes, "(stdin)" for "-"
    two = pigrep_process(["-e", PATTERN.decode(), "-c", str(path), "-"], stdin=data)
    assert two == b"%s: %d\n(stdin): %d\n" % (str(path).encode(), len(hits), len(hits))


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref not built")
def test_pigrep_only_matching_streamed(tmp_path):
    """-o (with -n, -b, -c) at any block size and through stdin prints the spans the resident text gives: the tool's
    documented selection over pire_gpu_match_ends_lines / pire_gpu_match_starts_lines of the whole text."""
    import torch
    import pire_b200 as P
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from pigrep import line_spans
    rng = np.random.default_rng(9)
    data = grep_text(rng)
    path = tmp_path / "in.txt"
    path.write_bytes(data)
    ref = Ref()
    hf = P.Scanner(ref.compile_half_final(PATTERN).save(), 0)
    rev = P.Scanner(ref.compile(PATTERN, "nr").save(), 0)
    batch = P.Batch.from_text(torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0"))
    spans = line_spans(P, hf, rev, batch)
    assert spans
    for opts in (["-o"], ["-o", "-n", "-b"], ["-o", "-c"]):
        if "-c" in opts:
            want = b"%d\n" % len(spans)
        else:
            want = b"".join((b"%d:%d:" % (l + 1, s) if "-n" in opts else b"") + data[s:e] + b"\n"
                            for l in sorted(spans) for s, e in spans[l])
        base = ["-e", PATTERN.decode()] + opts
        assert pigrep(base + [str(path)]) == want, opts
        assert pigrep(base + ["--block-mb", str(50 / MIB)], stdin=data) == want, opts


def test_cpp_line_stream(tmp_path):
    """tests/cpp/line_stream_check.cpp through include/pire_gpu.hpp: LineStream frames against split_lines of the whole
    text, and Runner / LineMatchEnds on the frames against the resident text."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "line_stream_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "line_stream_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    img = tmp_path / "hf.pire"
    img.write_bytes(START_IMAGES["glue10"]["forward"])
    for n, slot, piece, seed in ((5000, 4096, 1000, 1), (3000, 64, 7, 2), (0, 0, 1, 3), (20000, 1 << 20, 65536, 4)):
        out = subprocess.run([exe, str(img), str(n), str(slot), str(piece), str(seed)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ": 0 mismatches" in out.stdout
