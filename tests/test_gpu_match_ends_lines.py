"""pire_gpu_match_ends_lines / pire_gpu_match_starts_lines: where the matches end and start in every line of a text,
each line its own HalfFinalScanner run with its own marks, positions in the text.

The independent answers are pire_gpu_match_ends_string / pire_gpu_match_starts_string called once per line (the line
alone, base offsets[l]) and appended through one *d_found, the in-repo oracle's positions walk (ends_from) per line on a
sample, pire_gpu_count_batch with PIRE_GPU_RUN_LINES for the per-line histograms and pire_gpu_run_lines for the match
bits and states.  Every output buffer is longer than the call may write and pre-filled with a sentinel that must
survive: entries below the incoming *d_found and past the capacity, state and bitmap words past the lines."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from refpire import Oracle
from start_images import START_IMAGES
from test_count_images import COUNT_IMAGES, w_strings
from test_edge_images import ALPHABETS, EDGE
from test_gpu_batch_count_resume import FLAGS, LITERALS, RUN_BEGIN, RUN_END, RUN_LINES, load
from test_gpu_count_edges import LITERALS as EDGE_LITERALS
from test_gpu_edges import EXTRA, GLUE10_ALPHABET, SENTINEL, _filled, _host, _stream, expect_equal, expect_untouched, unpack_bits
from test_gpu_match_ends import GUARD, SENTINEL64, ends_from
from test_string_images import host_scanner

pytestmark = pytest.mark.gpu

BELOW = 3                       # sentinel entries before the incoming *d_found
NO_START = 0xFFFFFFFFFFFFFFFF
EINVAL, ENODEVICE = -1, -4


def _lib():
    from pire_b200 import _native as N
    return N


def scanner(name, max_hot=None):
    import pire_b200 as P
    image = EDGE[name]["image"] if name in EDGE else load(name)
    sc = P.Scanner(image, 0)
    if max_hot is not None:
        sc.set_max_hot(max_hot)
    return sc


def alphabet_of(name):
    if name in EDGE:
        return ALPHABETS[name], EDGE_LITERALS.get(name, [])
    if name in COUNT_IMAGES:
        return b"abcdefghijklmnopqrstuvwxyz ", []
    return GLUE10_ALPHABET, LITERALS


def random_lines(rng, name, count, max_len=160):
    """Lines drawn from the image's alphabet (never '\\n'), with its literals planted and some empty lines."""
    if name in COUNT_IMAGES:
        k = COUNT_IMAGES[name]["regexps"]
        return [s.replace(b"\n", b" ") for s in w_strings(rng, k, count, max_len)]
    alphabet, literals = alphabet_of(name)
    alpha = np.frombuffer(alphabet.replace(b"\n", b""), np.uint8)
    out = []
    for _ in range(count):
        n = 0 if rng.random() < 0.1 else int(rng.integers(0, max_len))
        line = bytearray(rng.choice(alpha, size=n).tobytes())
        if literals and n > 20 and rng.random() < 0.5:
            lit = literals[int(rng.integers(len(literals)))]
            at = int(rng.integers(0, n - len(lit))) if n > len(lit) else 0
            line[at:at + len(lit)] = lit
        out.append(bytes(line[:n]))
    return out


def text_of(lines, final_newline=True):
    return b"\n".join(lines) + (b"\n" if final_newline and lines else b"")


class Text:
    """A text on the device, `shift` bytes into its allocation (zeros around it), split into lines."""

    def __init__(self, data, shift=0):
        import torch
        import pire_b200 as P
        self.data = bytes(data)
        self.buf = torch.zeros(len(self.data) + shift + 64, dtype=torch.uint8, device="cuda:0")
        if self.data:
            self.buf[shift:shift + len(self.data)] = torch.frombuffer(bytearray(self.data), dtype=torch.uint8).to("cuda:0")
        self.dev = self.buf[shift:shift + len(self.data)]
        self.batch = P.Batch.from_text(self.dev)
        self.n = self.batch.n
        self.offs = self.batch.offsets.cpu().numpy().astype(np.uint64)
        self.ptr = self.dev.data_ptr()

    def line(self, l):
        return self.data[int(self.offs[l]):int(self.offs[l + 1]) - 1]


class LinesCall:
    """One pire_gpu_match_ends_lines call's buffers: BELOW + capacity + GUARD entries, *d_found = BELOW on entry, state and
    bitmap words past the lines, all sentinel-filled."""

    def __init__(self, n, capacity, below=BELOW):
        import torch
        self.n, self.below, self.capacity = n, below, below + capacity
        size = self.capacity + GUARD
        self.lines = _filled(size)
        self.ends = torch.full((size,), SENTINEL64, dtype=torch.int64, device="cuda:0")
        self.ids = _filled(size)
        self.found = torch.tensor([below], dtype=torch.int64, device="cuda:0")
        self.state = _filled(n + EXTRA)
        self.bits = _filled((n + 31) // 32 + 1)

    def run(self, sc, t, flags, arrays=(True, True, True), outs=(True, True)):
        N = _lib()
        l, e, i = (x.data_ptr() if on else None for x, on in zip((self.lines, self.ends, self.ids), arrays))
        rc = N.lib.pire_gpu_match_ends_lines(sc._h, t.ptr, t.batch.offsets.data_ptr(), t.n, flags, l, e, i, self.capacity,
                                             self.found.data_ptr(), self.bits.data_ptr() if outs[0] else None,
                                             self.state.data_ptr() if outs[1] else None, _stream())
        assert rc == 0, N.lib.pire_gpu_last_error()
        return self

    def results(self, label):
        """(lines, ends, ids, found, bits, states) on the host, every sentinel checked."""
        found = int(self.found.item()) - self.below
        top = min(self.below + found, self.capacity)
        ln, ids = _host(self.lines), _host(self.ids)
        ends = self.ends.cpu().numpy().view(np.uint64)
        for what, arr, sent in (("lines", ln, SENTINEL), ("ends", ends, SENTINEL64), ("ids", ids, SENTINEL)):
            assert (arr[:self.below] == sent).all(), "%s: %s written below the incoming *d_found" % (label, what)
            assert (arr[top:] == sent).all(), "%s: %s written past the entries or the capacity" % (label, what)
        states = _host(self.state)
        expect_untouched(label, "state indices", states, self.n)
        bits = unpack_bits(label, _host(self.bits), self.n)
        return ln[self.below:top], ends[self.below:top], ids[self.below:top], found, bits, states[: self.n]


def regs(sc):
    return max(1, sc.RegexpsCount())


def count_lines(sc, t, flags):
    """pire_gpu_count_batch with PIRE_GPU_RUN_LINES: (lines, regs) u32."""
    import torch
    N = _lib()
    if t.n == 0:
        return np.zeros((0, regs(sc)), np.uint32)
    counts = torch.empty(t.n * regs(sc), dtype=torch.int32, device="cuda:0")
    rc = N.lib.pire_gpu_count_batch(sc._h, t.ptr, t.batch.offsets.data_ptr(), 0, t.n, flags | RUN_LINES, counts.data_ptr(), None,
                                    _stream())
    assert rc == 0, N.lib.pire_gpu_last_error()
    return _host(counts).reshape(t.n, regs(sc))


def run_lines(sc, t, flags):
    """pire_gpu_run_lines: (bits, states)."""
    import torch
    N = _lib()
    bits = torch.zeros((t.n + 31) // 32 + 1, dtype=torch.int32, device="cuda:0")
    states = torch.empty(t.n + 1, dtype=torch.int32, device="cuda:0")
    rc = N.lib.pire_gpu_run_lines(sc._h, t.ptr, t.batch.offsets.data_ptr(), None, t.n, flags, bits.data_ptr(), None, states.data_ptr(),
                                  _stream())
    assert rc == 0, N.lib.pire_gpu_last_error()
    words = _host(bits)
    return np.unpackbits(words.view(np.uint8), bitorder="little")[: t.n].astype(bool), _host(states)[: t.n]


def per_line(sc, t, flags, per_line_counts):
    """pire_gpu_match_ends_string once per line (the line alone, base offsets[l]), all appended through one *d_found:
    (lines, ends, ids, found)."""
    import torch
    N = _lib()
    total = int(per_line_counts.sum())
    cap = total + 16
    ends = torch.empty(cap, dtype=torch.int64, device="cuda:0")
    ids = torch.empty(cap, dtype=torch.int32, device="cuda:0")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    for l in range(t.n):
        b, e = int(t.offs[l]), int(t.offs[l + 1]) - 1
        rc = N.lib.pire_gpu_match_ends_string(sc._h, t.ptr + b, e - b, flags & (RUN_BEGIN | RUN_END), None, b, ends.data_ptr(),
                                              ids.data_ptr(), cap, found.data_ptr(), None, None, _stream())
        assert rc == 0, N.lib.pire_gpu_last_error()
    f = int(found.item())
    assert f == total, "per-line match_ends_string found %d entries, count_batch counted %d" % (f, total)
    lines = np.repeat(np.arange(t.n, dtype=np.uint32), per_line_counts.astype(np.int64))
    return lines, ends[:f].cpu().numpy().view(np.uint64), _host(ids[:f]), f


def check_lines(label, sc, t, flags, capacity=None, oracle_sample=0, name=None):
    """One call against every independent answer (with `name`, the oracle of that image on a sample of lines); returns
    its results."""
    counts = count_lines(sc, t, flags)
    per = counts.sum(axis=1) if t.n else np.zeros(0, np.uint64)
    total = int(per.sum())
    call = LinesCall(t.n, total if capacity is None else capacity).run(sc, t, flags)
    lines, ends, ids, found, bits, states = call.results(label)
    assert found == total, "%s: %d entries, count_batch counts %d" % (label, found, total)
    want_l, want_e, want_i, _ = per_line(sc, t, flags, per)
    k = len(lines)
    expect_equal(label, "lines", lines, want_l[:k])
    expect_equal(label, "ends", ends, want_e[:k])
    expect_equal(label, "ids", ids, want_i[:k])
    if k == total and t.n:
        hist = np.zeros((t.n, regs(sc)), np.uint32)
        np.add.at(hist, (lines.astype(np.int64), ids.astype(np.int64)), 1)
        expect_equal(label, "per-line histograms (count_batch LINES)", hist, counts)
    want_bits, want_states = run_lines(sc, t, flags)
    expect_equal(label, "match bits (run_lines)", bits, want_bits)
    expect_equal(label, "states (run_lines)", states, want_states)
    if oracle_sample and t.n:
        orc = Oracle(EDGE[name]["image"] if name in EDGE else load(name))
        rng = np.random.default_rng(t.n)
        begin, end = bool(flags & RUN_BEGIN), bool(flags & RUN_END)
        for l in sorted(set(int(x) for x in rng.integers(0, t.n, size=oracle_sample))):
            we, wi, _ = ends_from(orc, np.frombuffer(t.line(l), np.uint8), None, begin, end, int(t.offs[l]))
            sel = lines == l
            expect_equal("%s line %d" % (label, l), "ends (oracle)", ends[sel], we)
            expect_equal("%s line %d" % (label, l), "ids (oracle)", ids[sel], wi)
    return lines, ends, ids, found, bits, states


MANY = next(n for n in sorted(COUNT_IMAGES) if COUNT_IMAGES[n]["regexps"] > 32)
IMAGES = ["hf_glue10", "count_words5", MANY] + sorted(EDGE)


@pytest.mark.parametrize("name", IMAGES)
@pytest.mark.parametrize("flags", FLAGS + [RUN_LINES | RUN_BEGIN | RUN_END])
def test_images_and_marks(name, flags):
    """Every image, every mark combination (LINES accepted), against per-line calls, count_batch and run_lines."""
    rng = np.random.default_rng(len(name) * 7 + flags)
    lines = random_lines(rng, name, 700)
    t = Text(text_of(lines, final_newline=bool(flags & 1)), shift=int(rng.integers(0, 32)))
    check_lines("%s flags %d" % (name, flags), scanner(name), t, flags, oracle_sample=12 if name != MANY else 3, name=name)


SHAPES = {
    "empty": b"",
    "one line, no newline": b"GET error hello world the cat",
    "only newlines": b"\n" * 70,
    "runs of empty lines": b"error\n\n\n\nGET \n\n" * 40 + b"\n\nhello world",
    "crlf": b"GET /x HTTP/1.1\r\nerror: timeout\r\n\r\nhello world\r\n" * 30,
    "one newline": b"\n",
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("name", ["hf_glue10", "anchored", "all_final"])
def test_text_shapes(shape, name):
    """Empty text, one line without newline, empty lines, \\r\\n (the \\r belongs to the line); on a glued image, a ^...$
    image and one whose patterns match the empty string (Initialize / BeginMark report on every line)."""
    t = Text(SHAPES[shape])
    for flags in FLAGS:
        check_lines("%s / %s flags %d" % (shape, name, flags), scanner(name), t, flags)


def test_long_line_and_alignments():
    """A line of several MiB spanning many segments, among short lines; lines starting at every alignment 0..31; the
    text at every pointer offset 1..31 into its allocation."""
    rng = np.random.default_rng(5)
    sc = scanner("hf_glue10")
    big = b"".join(random_lines(rng, "hf_glue10", 40000, 200)).replace(b"\n", b" ")[: 5 << 20]
    t = Text(b"GET error\n" + big + b"\nhello world\n" + text_of(random_lines(rng, "hf_glue10", 50)))
    for flags in FLAGS:
        check_lines("long line flags %d" % flags, sc, t, flags)
    aligned = text_of([b"x" * k + b"error" for k in range(64)])
    for shift in range(32):
        t = Text(aligned, shift)
        check_lines("alignment shift %d" % shift, sc, t, RUN_BEGIN | RUN_END)


@pytest.mark.parametrize("name,max_hot", [("hf_glue10", 1), ("hf_glue10", 2), ("none_hot", None), ("wide", 1)])
def test_one_line_per_lane_route(name, max_hot):
    """Handles whose start state is not a hot row walk one line per lane; the answers equal the in-stream kernel's."""
    rng = np.random.default_rng(11)
    t = Text(text_of(random_lines(rng, name, 900)))
    full = scanner(name)
    cut = scanner(name, max_hot) if max_hot is not None else full
    for flags in FLAGS:
        a = check_lines("%s max_hot %s flags %d" % (name, max_hot, flags), cut, t, flags)
        b = check_lines("%s flags %d" % (name, flags), full, t, flags)
        for x, y in zip(a, b):
            expect_equal(name, "one-line-per-lane vs in-stream", np.asarray(x), np.asarray(y))


def test_tuned_and_autoselected():
    rng = np.random.default_rng(13)
    t = Text(text_of(random_lines(rng, "hf_glue10", 2000)))
    for how in ("tune", "auto"):
        sc = scanner("hf_glue10")
        if how == "tune":
            sc.Tune(t.batch, t.n)
        else:
            sc.AutoSelect(t.batch)
        check_lines(how, sc, t, RUN_BEGIN | RUN_END)


def test_capacity_append_null_arrays_and_repeat():
    """Capacity 0, 1, short and exact; an incoming *d_found > 0; every subset of NULL arrays; two calls identical."""
    rng = np.random.default_rng(17)
    sc = scanner("count_words5")
    t = Text(text_of(random_lines(rng, "count_words5", 400)))
    flags = RUN_BEGIN | RUN_END
    total = int(count_lines(sc, t, flags).sum())
    full = LinesCall(t.n, total).run(sc, t, flags).results("full")
    for cap in (0, 1, 7, total // 3, total - 1, total):
        for below in (0, BELOW):
            got = LinesCall(t.n, cap, below).run(sc, t, flags).results("capacity %d" % cap)
            assert got[3] == total
            for g, w, what in zip(got[:3], full[:3], ("lines", "ends", "ids")):
                expect_equal("capacity %d" % cap, what, g, w[:cap])
    for mask in range(8):
        arrays = tuple(bool(mask >> k & 1) for k in range(3))
        c = LinesCall(t.n, total).run(sc, t, flags, arrays, outs=(mask & 1 == 0, mask & 2 == 0))
        ln, e, i = (_host(c.lines), c.ends.cpu().numpy().view(np.uint64), _host(c.ids))
        assert int(c.found.item()) - BELOW == total
        for on, arr, want, sent in zip(arrays, (ln, e, i), full[:3], (SENTINEL, SENTINEL64, SENTINEL)):
            if on:
                expect_equal("arrays %d" % mask, "entries", arr[BELOW:BELOW + total], want)
            else:
                assert (arr == sent).all(), "a NULL array's stand-in was written"
    a = LinesCall(t.n, total + 5).run(sc, t, flags)
    b = LinesCall(t.n, total + 5).run(sc, t, flags)
    for x, y in ((a.lines, b.lines), (a.ends, b.ends), (a.ids, b.ids), (a.state, b.state), (a.bits, b.bits)):
        assert bytes(x.cpu().numpy().tobytes()) == bytes(y.cpu().numpy().tobytes()), "two calls differ"


def test_refusals():
    import torch
    N = _lib()
    sc = scanner("hf_glue10")
    t = Text(b"error\nGET \n")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    offs = t.batch.offsets.data_ptr()

    def call(flags=0, text=t.ptr, offsets=offs, n=t.n, fnd=found.data_ptr(), h=sc._h):
        return N.lib.pire_gpu_match_ends_lines(h, text, offsets, n, flags, None, None, None, 0, fnd, None, None, _stream())

    assert call() == 0
    assert call(flags=8) == EINVAL
    assert call(flags=RUN_BEGIN | 16) == EINVAL
    assert call(fnd=None) == EINVAL
    assert call(offsets=None) == EINVAL
    assert call(text=None) == EINVAL
    assert call(n=1 << 32) == EINVAL
    assert call(text=None, n=0) == 0
    assert int(found.item()) == int(count_lines(sc, t, 0).sum())
    host = host_scanner(load("hf_glue10"))
    assert call(h=host._h) == ENODEVICE
    ends = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    starts = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    lines = torch.zeros(4, dtype=torch.int32, device="cuda:0")

    def starts_call(offsets=offs, ln=lines.data_ptr(), flags=0, h=sc._h):
        return N.lib.pire_gpu_match_starts_lines(h, t.ptr, offsets, t.n, flags, 0, ln, ends.data_ptr(), None, None,
                                                 found.data_ptr(), 4, starts.data_ptr(), None, _stream())

    assert starts_call(ln=None) == EINVAL
    assert starts_call(offsets=None) == EINVAL
    assert starts_call(flags=8) == EINVAL
    assert starts_call(h=host._h) == ENODEVICE


# ---------------------------------------------------------------- starts

def starts_per_line(case, t, flags, max_back, lines, ends, ids, use_ids):
    """pire_gpu_match_starts_string once per line with entries, the line as its window and base offsets[l]."""
    import torch
    N = _lib()
    k = len(lines)
    e_dev = torch.from_numpy(ends.view(np.int64).copy()).to("cuda:0")
    i_dev = torch.from_numpy(ids.view(np.int32).copy()).to("cuda:0")
    out = torch.full((k + 1,), -1, dtype=torch.int64, device="cuda:0")
    opened = torch.zeros(k + 1, dtype=torch.uint8, device="cuda:0")
    bounds = np.searchsorted(lines, np.arange(t.n + 1)) if k else np.zeros(t.n + 1, np.int64)
    cnt = torch.from_numpy(np.diff(bounds).astype(np.int64)).to("cuda:0")
    for l in range(t.n):
        a, b = int(bounds[l]), int(bounds[l + 1])
        if a == b:
            continue
        lo, hi = int(t.offs[l]), int(t.offs[l + 1]) - 1
        rc = N.lib.pire_gpu_match_starts_string(case.rev._h, t.ptr + lo, hi - lo, lo, flags, max_back, e_dev.data_ptr() + 8 * a,
                                                i_dev.data_ptr() + 4 * a if use_ids else None, None, cnt.data_ptr() + 8 * l,
                                                b - a, out.data_ptr() + 8 * a, opened.data_ptr() + a, _stream())
        assert rc == 0, N.lib.pire_gpu_last_error()
    return out[:k].cpu().numpy().view(np.uint64), opened[:k].cpu().numpy()


def starts_lines(case, t, flags, max_back, c, use_ids=True, first=None):
    import torch
    N = _lib()
    cap = c.capacity
    out = torch.full((cap + GUARD,), -1, dtype=torch.int64, device="cuda:0")
    opened = torch.full((cap + GUARD,), 0x5A, dtype=torch.uint8, device="cuda:0")
    fst = None if first is None else torch.tensor([first], dtype=torch.int64, device="cuda:0")
    rc = N.lib.pire_gpu_match_starts_lines(case.rev._h, t.ptr, t.batch.offsets.data_ptr(), t.n, flags, max_back, c.lines.data_ptr(),
                                           c.ends.data_ptr(), c.ids.data_ptr() if use_ids else None,
                                           None if fst is None else fst.data_ptr(), c.found.data_ptr(), cap, out.data_ptr(),
                                           opened.data_ptr(), _stream())
    assert rc == 0, N.lib.pire_gpu_last_error()
    return out.cpu().numpy().view(np.uint64), opened.cpu().numpy()


class StartCase:
    _cache = {}

    def __new__(cls, name):
        if name not in cls._cache:
            import pire_b200 as P
            c = object.__new__(cls)
            c.fwd = P.Scanner(START_IMAGES[name]["forward"], 0)
            c.rev = P.Scanner(START_IMAGES[name]["reversed"], 0)
            cls._cache[name] = c
        return cls._cache[name]


def start_text(rng, count):
    lines = random_lines(rng, "hf_glue10", count, 120)
    return text_of(lines)


@pytest.mark.parametrize("name", sorted(START_IMAGES))
@pytest.mark.parametrize("flags", FLAGS)
def test_starts_lines(name, flags):
    """Every start-image set and mark combination, with and without ids, max_back 0 and 7: against per-line
    match_starts_string calls."""
    rng = np.random.default_rng(len(name) + 3 * flags)
    case = StartCase(name)
    alpha = sorted(set(b"".join(p for p, _ in START_IMAGES[name]["patterns"])) | set(b" abcxyz0123"))
    alpha = bytes(b for b in alpha if b != 10)
    lines = [bytes(rng.choice(np.frombuffer(alpha, np.uint8), size=int(rng.integers(0, 90))).tobytes()) for _ in range(300)]
    t = Text(text_of(lines, final_newline=bool(flags & 1)), shift=int(rng.integers(0, 32)))
    total = int(count_lines(case.fwd, t, flags).sum())
    c = LinesCall(t.n, total).run(case.fwd, t, flags)
    ln, ends, ids, found, _, _ = c.results("ends")
    for use_ids in (True, False):
        for max_back in (0, 7):
            got, opened = starts_lines(case, t, flags, max_back, c, use_ids)
            want, want_open = starts_per_line(case, t, flags, max_back, ln, ends, ids, use_ids)
            label = "%s flags %d ids %s max_back %d" % (name, flags, use_ids, max_back)
            assert (got[:BELOW] == NO_START).all() and (got[BELOW + found:] == NO_START).all(), label + ": written outside"
            expect_equal(label, "starts", got[BELOW:BELOW + found], want)
            expect_equal(label, "open", opened[BELOW:BELOW + found], want_open)
            ok = want != NO_START
            assert (want[ok] >= t.offs[ln[ok]]).all() and (want[ok] <= ends[ok]).all()


def test_starts_windows_and_foreign_entries():
    """d_first windows, entries whose end lies outside their line and entries of lines >= n_lines are not written."""
    import torch
    rng = np.random.default_rng(23)
    name = sorted(START_IMAGES)[0]
    case = StartCase(name)
    t = Text(start_text(rng, 200))
    flags = RUN_BEGIN | RUN_END
    total = int(count_lines(case.fwd, t, flags).sum())
    c = LinesCall(t.n, total).run(case.fwd, t, flags)
    ln, ends, ids, found, _, _ = c.results("ends")
    full, _ = starts_lines(case, t, flags, 0, c)
    if found > 4:
        got, opened = starts_lines(case, t, flags, 0, c, first=BELOW + found // 2)
        assert (got[:BELOW + found // 2] == NO_START).all()
        expect_equal("d_first", "starts", got[BELOW + found // 2:BELOW + found], full[BELOW + found // 2:BELOW + found])
    # move some entries to another line or past the lines: not written
    if found:
        bad = c.lines.clone()
        host_l = _host(bad).copy()
        host_l[BELOW] = t.n + 5
        if found > 1:
            host_l[BELOW + 1] = (int(host_l[BELOW + 1]) + 1) % max(1, t.n)
        c.lines.copy_(torch.from_numpy(host_l.view(np.int32)).to("cuda:0"))
        got, _ = starts_lines(case, t, flags, 0, c)
        assert got[BELOW] == NO_START
        if found > 1:
            l1 = int(host_l[BELOW + 1])
            inside = t.offs[l1] <= ends[1] <= t.offs[l1 + 1] - 1
            if not inside:
                assert got[BELOW + 1] == NO_START


# ---------------------------------------------------------------- Python and pigrep

def test_python_face():
    import pire_b200 as P
    rng = np.random.default_rng(29)
    t = Text(text_of(random_lines(rng, "hf_glue10", 500)))
    sc = scanner("hf_glue10")
    flags = RUN_BEGIN | RUN_END
    total = int(count_lines(sc, t, flags).sum())
    r = P.LineMatchEnds(sc, total + 3).Begin().Run(t.batch).End()
    assert r.FoundTensor().is_cuda and r.EndsTensor().numel() == total + 3
    want = LinesCall(t.n, total).run(sc, t, flags).results("C")
    assert r.Found() == total
    expect_equal("python", "lines", r.Lines(), want[0])
    expect_equal("python", "ends", r.Ends(), want[1])
    expect_equal("python", "ids", r.Ids(), want[2])
    expect_equal("python", "matches", r.Matches(), want[4])
    expect_equal("python", "states", r.States(), want[5])
    with pytest.raises(ValueError):
        P.LineMatchEnds(sc, 4).Run(P.Batch.from_strings([b"a", b"b"]))
    ordered = P.Batch.from_text(t.dev)
    ordered.order = ordered.offsets
    with pytest.raises(ValueError):
        P.LineMatchEnds(sc, 4).Run(ordered)
    with pytest.raises(ValueError):
        P.BatchMatchEnds(sc, t.n, 4).Run(t.batch)
    name = sorted(START_IMAGES)[0]
    case = StartCase(name)
    total = int(count_lines(case.fwd, t, flags).sum())
    r = P.LineMatchEnds(case.fwd, total).Begin().Run(t.batch).End()
    s = P.MatchStarts(case.rev, r, t.batch, begin=True, end=True)
    c = LinesCall(t.n, total, 0).run(case.fwd, t, flags)
    want, _ = starts_per_line(case, t, flags, 0, *c.results("C")[:3], True)
    expect_equal("python starts", "starts", s.Starts(), want)
    ends_b = P.BatchMatchEnds(case.fwd, t.n, 4)
    with pytest.raises(ValueError):
        P.MatchStarts(case.rev, ends_b, t.batch)


def select_spans(spans):
    """Leftmost-longest non-overlapping spans of one line: by start ascending, then end descending; a span is taken when it
    starts at or after the previous one's end."""
    out, last = [], -1
    for s, e in sorted(set(spans), key=lambda x: (x[0], -x[1])):
        if s >= last:
            out.append((s, e))
            last = e
    return out


def test_pigrep_only_matching(tmp_path):
    """tools/pigrep.py -o -n -b (and -c) against a host-side selection over the per-line calls' spans."""
    name = "glue10" if "glue10" in START_IMAGES else sorted(START_IMAGES)[0]
    e = START_IMAGES[name]
    rng = np.random.default_rng(31)
    lines = random_lines(rng, "hf_glue10", 300, 100) + [b"", b"error error", b"GET GET "]
    data = text_of(lines)
    (tmp_path / "in.txt").write_bytes(data)
    (tmp_path / "hf.pire").write_bytes(e["forward"])
    (tmp_path / "rev.pire").write_bytes(e["reversed"])
    t = Text(data)
    case = StartCase(name)
    flags = RUN_BEGIN | RUN_END
    total = int(count_lines(case.fwd, t, flags).sum())
    c = LinesCall(t.n, total, 0).run(case.fwd, t, flags)
    ln, ends, ids, _, _, _ = c.results("C")
    st, _ = starts_per_line(case, t, flags, 0, ln, ends, ids, True)
    want = []
    for l in range(t.n):
        sel = (ln == l) & (st != NO_START)
        spans = [(int(s), int(x)) for s, x in zip(st[sel], ends[sel]) if x > s]
        for s, x in select_spans(spans):
            want.append(b"%d:%d:%s" % (l + 1, s, data[s:x]))
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pigrep.py"), "--half-final", str(tmp_path / "hf.pire"),
                          "--reverse", str(tmp_path / "rev.pire"), "-o", "-n", "-b", str(tmp_path / "in.txt")],
                         capture_output=True, env=env)
    assert out.returncode in (0, 1), out.stderr.decode()
    assert out.stdout.splitlines() == want
    cnt = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pigrep.py"), "--half-final", str(tmp_path / "hf.pire"),
                          "--reverse", str(tmp_path / "rev.pire"), "-o", "-c", str(tmp_path / "in.txt")],
                         capture_output=True, env=env)
    lines_hit = len({w.split(b":", 1)[0] for w in want})
    assert cnt.stdout.strip() == str(lines_hit).encode(), cnt.stderr.decode()



def test_cpp_match_ends_lines(tmp_path):
    """tests/cpp/match_ends_lines_check.cpp through include/pire_gpu.hpp: LineMatchEnds and the line form of MatchStarts
    against StringMatchEnds and MatchStarts run on each line alone."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "match_ends_lines_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "match_ends_lines_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    for name in ("glue10", "words"):
        fwd, rev = tmp_path / (name + "_forward.pire"), tmp_path / (name + "_reversed.pire")
        fwd.write_bytes(START_IMAGES[name]["forward"])
        rev.write_bytes(START_IMAGES[name]["reversed"])
        for n, seed in ((3000, 1), (1, 2), (0, 3)):
            out = subprocess.run([exe, str(fwd), str(rev), str(n), str(seed)], capture_output=True, text=True, timeout=300)
            assert out.returncode == 0, out.stdout + out.stderr
            assert ": 0 mismatches" in out.stdout
