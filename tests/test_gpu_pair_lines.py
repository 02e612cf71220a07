"""Two scanners over the lines of a text (pire_gpu_run_pair_lines, Runner(ScannerPair).RunLines): each scanner's three
outputs must equal, bit for bit, what pire_gpu_run_lines gives that scanner alone on the same text -- whole bitmap words,
masks and states -- with 64 sentinel words past the end of every output.  A line sample is also checked against the
in-repo C oracle, each line walked alone with its marks.  Covers glued, headline, hot-set-heavy and many-regexp images in
pairs, one handle twice, tuned and auto-selected handles, the edge images (whose cold start states take the two-launch
route), text shapes from the empty text to a 5 MiB line and a 256 MiB planted text, every text alignment, all mark
combinations, every subset of NULL outputs, LineStream frames, refusals, pigrep with two scanners and the C++ mirror."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from refpire import Oracle, Ref, csr, have_ref
from test_edge_images import EDGE
from test_gpu_edges import EXTRA, MARKS, _filled, _host, _stream, expect_equal, expect_untouched
from test_gpu_pair import image_of, scanner

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
EINVAL, ENODEVICE = -1, -4
WORDS = [b"GET /index", b"error", b"timeout", b"(555) 123-4567", b"https://x", b"hello  world", b"fatal", b"foo", b"\r",
         b"Hello World", b"w017", b"w299", b"zz"]


def _flags(begin, end):
    return (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)


def _ptr(t):
    return None if t is None else t.data_ptr()


def random_text(rng, count, max_words=8, final_newline=True):
    lines = []
    for _ in range(count):
        k = int(rng.integers(0, max_words))
        lines.append(b" ".join(WORDS[int(i)] for i in rng.integers(0, len(WORDS), size=k)))
    return b"\n".join(lines) + (b"\n" if final_newline and lines else b"")


class Text:
    """A text on the device, `shift` bytes into a tensor of exactly shift + len bytes (no padding behind the text), split
    into lines."""

    def __init__(self, data, shift=0):
        import torch
        import pire_b200 as P
        self.data = bytes(data)
        self.buf = torch.empty(len(self.data) + shift, dtype=torch.uint8, device="cuda:0")
        if self.data:
            self.buf[shift:] = torch.frombuffer(bytearray(self.data), dtype=torch.uint8).to("cuda:0")
        self.dev = self.buf[shift:]
        self.batch = P.Batch.from_text(self.dev)
        self.n = self.batch.n
        self.ptr = self.dev.data_ptr() if self.data else None
        self.offs_ptr = self.batch.offsets.data_ptr()


def _outputs(n, want=(True, True, True)):
    return [_filled((n + 31) // 32 + 1) if want[0] else None, _filled(n + EXTRA) if want[1] else None,
            _filled(n + EXTRA) if want[2] else None]


def _read(label, outs, n):
    """Host copies of (bitmap words, masks, states); every word past each one's end must still hold the sentinel."""
    res = []
    for k, (t, valid) in enumerate(zip(outs, ((n + 31) // 32, n, n))):
        if t is None:
            res.append(None)
            continue
        h = _host(t)
        expect_untouched(label, ("match bitmap", "accept masks", "state indices")[k], h, valid)
        res.append(h[:valid].copy())
    return res


def single(sc, t, flags, want=(True, True, True)):
    from pire_b200 import _native as N
    outs = _outputs(t.n, want)
    N.check(N.lib.pire_gpu_run_lines(sc._h, t.ptr, t.offs_ptr, None, t.n, flags, *map(_ptr, outs), _stream()), "pire_gpu_run_lines")
    return _read("single", outs, t.n)


def pair(sc1, sc2, t, flags, want=(True,) * 6):
    from pire_b200 import _native as N
    outs = _outputs(t.n, want[:3]) + _outputs(t.n, want[3:])
    N.check(N.lib.pire_gpu_run_pair_lines(sc1._h, sc2._h, t.ptr, t.offs_ptr, t.n, flags, *map(_ptr, outs), _stream()),
            "pire_gpu_run_pair_lines")
    return _read("pair", outs[:3], t.n) + _read("pair", outs[3:], t.n)


def check(sc1, sc2, t, flags, label, want=(True,) * 6):
    got = pair(sc1, sc2, t, flags, want)
    ref = single(sc1, t, flags, want[:3]) + single(sc2, t, flags, want[3:])
    for k in range(6):
        if want[k]:
            expect_equal(label, ("bits", "masks", "states")[k % 3] + str(k // 3 + 1), got[k], ref[k])
        else:
            assert got[k] is None
    return got


PAIRS = [("glue10", "headline"), ("headline", "glue10"), ("glue10", "hf_glue10"), ("headline", "headline_iu")]


def shapes(rng):
    long_line = bytes(rng.choice(np.frombuffer(b"abcdefgh error ", np.uint8), size=9000)) + b" timeout"
    return [
        ("empty", b""),
        ("one line, no newline", b"error at GET /index"),
        ("no final newline", random_text(rng, 300, final_newline=False)),
        ("only newlines", b"\n" * 77),
        ("empty lines", b"\n\nerror\n\n\nfoo\n\n"),
        ("crlf", b"\r\n".join(random_text(rng, 50).split(b"\n"))),
        ("long line", random_text(rng, 20) + long_line + b"\n" + random_text(rng, 20, final_newline=False)),
    ]


@pytest.mark.parametrize("names", PAIRS, ids=["%s+%s" % p for p in PAIRS])
def test_pairs_shapes_and_marks(cuda_device, names):
    rng = np.random.default_rng(1)
    sc1, sc2 = scanner(names[0]), scanner(names[1])
    for label, data in shapes(rng) + [("random", random_text(rng, 2000))]:
        t = Text(data)
        for begin, end in MARKS:
            check(sc1, sc2, t, _flags(begin, end), "%s+%s %s begin=%d end=%d" % (names + (label, begin, end)))


def test_one_handle_twice_and_lines_flag(cuda_device):
    rng = np.random.default_rng(2)
    g = scanner("glue10")
    t = Text(random_text(rng, 3000))
    for begin, end in MARKS:
        check(g, g, t, _flags(begin, end), "glue10 twice begin=%d end=%d" % (begin, end))
    check(g, g, t, RUN_LINES | RUN_BEGIN | RUN_END, "LINES accepted")


def test_five_mib_line_and_alignments(cuda_device):
    rng = np.random.default_rng(3)
    g, h = scanner("glue10"), scanner("headline")
    big = bytes(rng.choice(np.frombuffer(b"abc error GET /x", np.uint8), size=5 << 20))
    check(g, h, Text(b"first\n" + big + b"\nlast error"), 3, "5 MiB line")
    data = random_text(rng, 400, final_newline=False)
    for shift in range(32):
        check(g, h, Text(data, shift), 3, "shift %d" % shift)


def test_planted_256_mib(cuda_device):
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from match_ends_lines_bench import make_text
    from pire_b200 import workloads as W
    import pire_b200 as P
    text = make_text(torch, W, 0.25)
    b = P.Batch.from_text(text)

    class T:
        pass
    t = T()
    t.n, t.ptr, t.offs_ptr = b.n, text.data_ptr(), b.offsets.data_ptr()
    for a, c in (("glue10", "headline"), ("glue10", "hf_glue10")):
        got = check(scanner(a), scanner(c), t, 3, "256 MiB %s+%s" % (a, c))
        assert 0 < int(np.unpackbits(got[0].view(np.uint8)).sum()) < t.n
    del text, b
    torch.cuda.empty_cache()


def test_null_output_subsets(cuda_device):
    rng = np.random.default_rng(4)
    g, h = scanner("glue10"), scanner("headline")
    t = Text(random_text(rng, 100, final_newline=False))
    for mask in range(64):
        want = tuple(bool(mask >> k & 1) for k in range(6))
        check(g, h, t, 3, "outputs %s" % (want,), want)


def test_tuned_untuned_and_autoselected(cuda_device):
    import pire_b200 as P
    rng = np.random.default_rng(5)
    t = Text(random_text(rng, 3000))
    tuned, plain = scanner("glue10"), scanner("headline")
    tuned.Tune(t.batch)
    check(tuned, plain, t, 3, "tuned+untuned")
    check(plain, tuned, t, 3, "untuned+tuned")
    auto = scanner("headline_iu")
    auto.AutoSelect(t.batch)
    check(auto, tuned, t, 3, "autoselected+tuned")
    assert P.Runner(P.ScannerPair(auto, tuned)).Begin().RunLines(t.batch).End().Matches().any()


EDGE_PAIRS = [(e, "glue10") for e in sorted(EDGE)] + [("glue10", e) for e in sorted(EDGE)] + \
             [("none_hot", "all_final"), ("wide", "absorbing")]


@pytest.mark.parametrize("names", EDGE_PAIRS, ids=["%s+%s" % p for p in EDGE_PAIRS])
def test_edge_images(cuda_device, names):
    """Edge images pair with each other and with glue10; a cold start takes the two-launch route, and where the other
    handle is hot its half must also be what the fused route gives it beside a hot partner."""
    rng = np.random.default_rng(6)
    sc1, sc2 = scanner(names[0]), scanner(names[1])
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789 \n", np.uint8)
    data = random_text(rng, 500) + rng.choice(alpha, size=20000).tobytes()
    t = Text(data)
    for begin, end in MARKS:
        got = check(sc1, sc2, t, _flags(begin, end), "%s+%s begin=%d end=%d" % (names + (begin, end)))
        if "glue10" in names:
            k = names.index("glue10")
            fused = pair(scanner("glue10"), scanner("headline"), t, _flags(begin, end))
            for j in range(3):
                expect_equal("fused vs route of %s+%s" % names, "glue10 output %d" % j, got[3 * k + j], fused[j])


@pytest.mark.parametrize("max_hot", [1, 2])
def test_small_hot_sets(cuda_device, max_hot):
    rng = np.random.default_rng(7)
    t = Text(random_text(rng, 1500))
    small, g = scanner("glue10", max_hot), scanner("headline")
    for begin, end in MARKS:
        check(small, g, t, _flags(begin, end), "max_hot %d begin=%d end=%d" % (max_hot, begin, end))
        check(g, small, t, _flags(begin, end), "max_hot %d second begin=%d end=%d" % (max_hot, begin, end))


def test_past_32_regexps(cuda_device):
    from pire_b200 import _native as N
    rng = np.random.default_rng(8)
    many, g = scanner("w300"), scanner("glue10")
    ids = rng.integers(0, 300, size=400)
    ids[:8] = [0, 31, 32, 33, 63, 64, 255, 299]
    data = b"\n".join(bytes(rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvxyz", np.uint8), size=int(rng.integers(0, 60))))
                      + b"w%03d" % k for k in ids) + b"\n"
    t = Text(data)
    for begin, end in MARKS:
        check(many, g, t, _flags(begin, end), "w300+glue10 begin=%d end=%d" % (begin, end))
    got = check(g, many, t, 0, "glue10+w300 no marks")
    words = N.lib.pire_gpu_accept_words(many._h)
    import torch
    states = torch.from_numpy(got[5].view(np.int32).copy()).to("cuda:0")
    sets = _filled(t.n * words + EXTRA)
    N.check(N.lib.pire_gpu_accept_sets(many._h, states.data_ptr(), t.n, sets.data_ptr(), _stream()), "accept_sets")
    rows = _host(sets)[: t.n * words].reshape(t.n, words)
    high = 0
    for i in range(t.n):
        acc = [r for r in range(words * 32) if (int(rows[i, r // 32]) >> (r % 32)) & 1]
        assert acc == many.AcceptedRegexps(int(got[5][i])), i
        high += any(r >= 32 for r in acc)
    assert high > 0


def test_oracle_sample(cuda_device):
    rng = np.random.default_rng(9)
    names = ("glue10", "headline_iu")
    data = random_text(rng, 600, final_newline=False)
    t = Text(data)
    lines = data.split(b"\n")
    corpus, offs = csr(lines)
    for begin, end in MARKS:
        got = pair(scanner(names[0]), scanner(names[1]), t, _flags(begin, end))
        for k, name in enumerate(names):
            final, mask, state = Oracle(image_of(name)).run(corpus, offs, begin=begin, end=end)
            bits = np.unpackbits(got[3 * k].view(np.uint8), bitorder="little")[: t.n].astype(bool)
            assert (bits == final.astype(bool)).all() and (got[3 * k + 1] == mask).all() and (got[3 * k + 2] == state).all(), \
                "%s begin=%d end=%d" % (name, begin, end)


def test_line_stream_frames(cuda_device):
    """A text fed in random pieces through slots smaller than its longest line: each frame's pair run, shifted by its
    first line, is the resident call's."""
    import pire_b200 as P
    rng = np.random.default_rng(10)
    data = random_text(rng, 4000) + b"x" * 6000 + b" error\n" + random_text(rng, 500, final_newline=False)
    t = Text(data)
    sc1, sc2 = scanner("glue10"), scanner("headline")
    want = [r.tolist() for r in pair(sc1, sc2, t, 3)]
    bits1 = np.unpackbits(np.array(want[0], np.uint32).view(np.uint8), bitorder="little")[: t.n].astype(bool)
    bits2 = np.unpackbits(np.array(want[3], np.uint32).view(np.uint8), bitorder="little")[: t.n].astype(bool)
    ls = P.LineStream(0, 4096)
    cuts = sorted(set(rng.integers(0, len(data), size=12).tolist())) + [len(data)]
    at, seen = 0, 0
    r1, r2, m1, s2, m = [], [], [], [], []
    for k, cut in enumerate(cuts):
        for f in ls.feed(data[at:cut], last=k == len(cuts) - 1):
            assert f.first_line == seen
            r = P.Runner(P.ScannerPair(sc1, sc2)).Begin().RunLines(f).End()
            r1 += r.First().Matches().tolist()
            r2 += r.Second().Matches().tolist()
            m1 += r.First().AcceptMasks().tolist()
            s2 += r.Second().States().tolist()
            m += r.Matches().tolist()
            seen += f.n
        at = cut
    assert seen == t.n
    assert r1 == bits1.tolist() and r2 == bits2.tolist() and m1 == want[1] and s2 == want[5]
    assert m == (bits1 | bits2).tolist()


def test_python_face(cuda_device):
    import torch
    import pire_b200 as P
    rng = np.random.default_rng(11)
    t = Text(random_text(rng, 500))
    sc1, sc2 = scanner("glue10"), scanner("headline")
    r = P.Runner(P.ScannerPair(sc1, sc2)).Begin().RunLines(t.batch).End()
    a, b = P.Runner(sc1).Begin().Run(t.batch).End(), P.Runner(sc2).Begin().Run(t.batch).End()
    assert (r.First().States() == a.States()).all() and (r.Second().AcceptMasks() == b.AcceptMasks()).all()
    assert (r.Matches() == (a.Matches() | b.Matches())).all()
    pair_ = P.ScannerPair(sc1, sc2)
    with pytest.raises(ValueError):
        P.Runner(pair_).Run(t.batch).Matches()                        # Run() keeps refusing a line batch
    with pytest.raises(ValueError):
        P.Runner(pair_).RunLines(P.Batch(t.dev, fixed_len=1, n=8))     # not lines
    st = torch.zeros(t.n, dtype=torch.int32, device="cuda:0")
    with pytest.raises(ValueError):
        P.Runner(pair_, (st, None)).RunLines(t.batch)


def test_refusals(cuda_device):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    g, h = scanner("glue10"), scanner("headline")
    t = Text(b"error\nfoo\n")
    out = _filled(64)
    o = out.data_ptr()

    def call(h1, h2, text, offs, n, flags):
        return N.lib.pire_gpu_run_pair_lines(h1, h2, text, offs, n, flags, o, o, o, o, o, o, _stream())

    assert call(g._h, h._h, t.ptr, t.offs_ptr, t.n, 3) == 0
    for flags in (8, 16, 1 << 31):
        assert call(g._h, h._h, t.ptr, t.offs_ptr, t.n, flags) == EINVAL
    assert call(g._h, h._h, None, t.offs_ptr, t.n, 3) == EINVAL
    assert call(g._h, h._h, t.ptr, None, t.n, 3) == EINVAL
    assert call(g._h, h._h, t.ptr, t.offs_ptr, 1 << 31, 3) == EINVAL
    assert call(None, h._h, t.ptr, t.offs_ptr, t.n, 3) == EINVAL
    host = P.Scanner(image_of("glue10"), -1)
    assert call(host._h, h._h, t.ptr, t.offs_ptr, t.n, 3) == ENODEVICE
    assert call(g._h, host._h, t.ptr, t.offs_ptr, t.n, 3) == ENODEVICE
    torch.cuda.synchronize()
    before = _host(out).copy()
    assert call(g._h, h._h, None, None, 0, 3) == 0                    # no lines: a no-op
    torch.cuda.synchronize()
    assert (_host(out) == before).all()
    if torch.cuda.device_count() >= 2:
        other = P.Scanner(image_of("headline"), 1)
        assert call(g._h, other._h, t.ptr, t.offs_ptr, t.n, 3) == EINVAL


# ---- pigrep ------------------------------------------------------------------------------------------------------------

def pigrep(args, stdin=None):
    from test_gpu_line_stream import pigrep as run
    return run(args, stdin)


def test_pigrep_two_scanners(tmp_path):
    """--scanner a --scanner b prints the union of the two single-scanner runs, with -c, -n and -b, from a file and
    through stdin in small blocks; where oracle/_ref is built, the reference run line by line agrees."""
    rng = np.random.default_rng(12)
    data = random_text(rng, 800, final_newline=False)
    path = tmp_path / "in.txt"
    path.write_bytes(data)
    for name in ("glue10", "headline_iu"):
        (tmp_path / (name + ".pire")).write_bytes(image_of(name))
    a, b = str(tmp_path / "glue10.pire"), str(tmp_path / "headline_iu.pire")
    lines = data.split(b"\n")
    offs = [0]
    for ln in lines:
        offs.append(offs[-1] + len(ln) + 1)
    corpus, co = csr(lines)
    finals = [Oracle(image_of(n)).run(corpus, co)[0].astype(bool) for n in ("glue10", "headline_iu")]
    hits = np.nonzero(finals[0] | finals[1])[0].tolist()
    assert 0 < len(hits) < len(lines) and finals[0].any() and finals[1].any()
    if have_ref():
        ref = [Ref().load(image_of(n)).run(corpus, co)[0].astype(bool) for n in ("glue10", "headline_iu")]
        assert np.nonzero(ref[0] | ref[1])[0].tolist() == hits
    for opts in ([], ["-n"], ["-b"], ["-n", "-b"], ["-c"]):
        if opts == ["-c"]:
            want = b"%d\n" % len(hits)
        else:
            want = b"".join((b"%d:" % (i + 1) if "-n" in opts else b"") + (b"%d:" % offs[i] if "-b" in opts else b"")
                            + lines[i] + b"\n" for i in hits)
        one = [pigrep(["--scanner", s] + opts + [str(path)]) for s in (a, b)]
        base = ["--scanner", a, "--scanner", b] + opts
        got = pigrep(base + [str(path)])
        assert got == want, opts
        if opts != ["-c"]:
            assert set(got.splitlines()) == set(one[0].splitlines()) | set(one[1].splitlines()), opts
        assert pigrep(base + ["--block-mb", str(300 / (1 << 20)), "-"], stdin=data) == want, opts


# ---- C++ ----------------------------------------------------------------------------------------------------------------

def test_cpp_pair_lines(tmp_path):
    """tests/cpp/pair_lines_check.cpp through include/pire_gpu.hpp: Runner(pair).Run(frame) over a resident text and over
    LineStream frames against Runner(sc).Run(frame) for each scanner, and From() starts refused with a LineFrame."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "pair_lines_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pair_lines_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    for name in ("glue10", "headline"):
        (tmp_path / (name + ".pire")).write_bytes(image_of(name))
    for n, seed in ((5000, 1), (1, 2), (0, 3)):
        out = subprocess.run([exe, str(tmp_path / "glue10.pire"), str(tmp_path / "headline.pire"), str(n), str(seed)],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ": 0 mismatches" in out.stdout
