"""pire_gpu_count_batch_from: HalfFinalScanner counts of many streams at once, each from Initialize() or resumed from its
own state, with the counts added to u64 rows and the states carried in place from round to round.

The independent answers are pire_gpu_count_batch on whole strings and the in-repo oracle's count walk from any state
(tests/count_oracle.py); match bits and states are compared with pire_gpu_run_batch_from.  Every output buffer is larger
than the call may write and pre-filled with a sentinel that must survive: EXTRA rows of counters, EXTRA state words and
one bitmap word past n."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, GOLDEN_COUNTS, ROOT
from count_oracle import count_from
from refpire import Oracle, oracle_count
from test_count_images import COUNT_IMAGES, w_strings
from test_edge_images import ALPHABETS, EDGE
from test_gpu_batch_resume import _i32, csr_at, random_starts, run_from_batch, strings_of
from test_gpu_count_edges import LITERALS as EDGE_LITERALS
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, SENTINEL, _filled, _host, _stream, csr_batch, expect_equal, expect_untouched,
                            fixed_batch, is_uniform, random_rows, random_strings, unpack_bits)

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
FLAGS = [0, RUN_BEGIN, RUN_END, RUN_BEGIN | RUN_END]
LITERALS = [b"GET ", b"error", b"timeout", b"(555) 123-4567", b"https://", b"hello world", b"the cat"]


def regs_of(sc):
    return max(1, sc.RegexpsCount())


def flag_marks(flags):
    return bool(flags & RUN_BEGIN), bool(flags & RUN_END)


class Streams:
    """n streams on the device: one state array, one array of u64 counter rows and one bitmap, each longer than n and
    pre-filled with the sentinel past n.  ``starts`` (StateIndex values) fills the state array; without it the first
    round passes d_start == NULL (Initialize(), counted)."""

    def __init__(self, sc, n, starts=None, prefill=None):
        import torch
        self.sc, self.n, self.regs = sc, n, regs_of(sc)
        self.counts = torch.full((n + EXTRA, self.regs), SENTINEL, dtype=torch.int64, device="cuda:0")
        self.counts[:n] = 0 if prefill is None else torch.from_numpy(np.asarray(prefill, np.int64)).to("cuda:0")
        self.state = _filled(n + EXTRA)
        if starts is not None:
            self.state[:n] = _i32(starts)
        self.bits = _filled((n + 31) // 32 + 1)
        self.resumed = starts is not None

    def round(self, hb, flags, bits=True):
        """One call with d_start == d_state_idx (or NULL before the first round of fresh streams)."""
        from pire_b200 import _native as N
        N.check(N.lib.pire_gpu_count_batch_from(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, self.n, flags,
                                                self.state.data_ptr() if self.resumed else None, self.counts.data_ptr(),
                                                self.bits.data_ptr() if bits else None, self.state.data_ptr(), _stream()),
                "pire_gpu_count_batch_from")
        self.resumed = True
        return self

    def results(self, label):
        """(counts[n, regs] as int64, match bits, states) on the host, the sentinels past n checked."""
        c = self.counts.cpu().numpy()
        if not (c[self.n:] == SENTINEL).all():
            raise AssertionError("%s: counters written past row n - 1" % label)
        s = _host(self.state)
        expect_untouched(label, "state indices", s, self.n)
        return c[: self.n], unpack_bits(label, _host(self.bits), self.n), s[: self.n]


def count_batch(sc, hb, flags):
    """pire_gpu_count_batch: (counts widened to int64, match bits)."""
    import torch
    from pire_b200 import _native as N
    counts = torch.zeros((hb.n, regs_of(sc)), dtype=torch.int32, device="cuda:0")
    bits = _filled((hb.n + 31) // 32 + 1, 0)
    N.check(N.lib.pire_gpu_count_batch(sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, hb.n, flags, counts.data_ptr(),
                                       bits.data_ptr(), _stream()), "pire_gpu_count_batch")
    return counts.cpu().numpy().view(np.uint32).astype(np.int64), unpack_bits("count_batch", _host(bits)[: (hb.n + 31) // 32], hb.n)


def oracle_from(orc, strings, starts, flags):
    """count_from per string: counts[n, regs] and (final, state) per string; starts None = Initialize() (counted)."""
    begin, end = flag_marks(flags)
    counts, final, state = [], [], []
    for k, s in enumerate(strings):
        c, res = count_from(orc, np.frombuffer(s, np.uint8), None if starts is None else int(starts[k]), begin, end)
        counts.append(c)
        final.append(res[0])
        state.append(res[2])
    regs = max(1, orc.regexps)
    return (np.array(counts, np.int64).reshape(len(strings), regs), np.array(final, np.uint8), np.array(state, np.uint32))


def check_against_run_from(label, sc, hb, starts, flags, bits, states):
    begin, end = flag_marks(flags)
    want_bits, _, want_states = run_from_batch(sc, hb, starts, begin, end)
    expect_equal(label, "StateIndex (run_batch_from)", states, want_states)
    expect_equal(label, "match bits (run_batch_from)", bits, want_bits)


def load(name):
    from pire_b200 import workloads as W
    if name in COUNT_IMAGES:
        return COUNT_IMAGES[name]["image"]
    return W.load_image(name)


def batches_for(name, rng, regexps):
    """A uniform batch (32-byte aligned, length % 32 == 0) and ragged CSR batches at unaligned starts."""
    if name in COUNT_IMAGES:
        alphabet = b"abcdefghijklmnopqrstuvwxyz"
        rows = np.frombuffer(b"".join(s.ljust(64, b"q")[:64] for s in w_strings(rng, regexps, 32 * 3 + 5, 60)), np.uint8).reshape(-1, 64)
        strings = w_strings(rng, regexps, 150, 300)
    else:
        alphabet = GLUE10_ALPHABET
        rows = random_rows(rng, 32 * 3 + 5, 256, alphabet, LITERALS)
        strings = random_strings(rng, alphabet, [0, 1, 15, 16, 17, 33] + [int(x) for x in rng.integers(0, 700, size=120)], LITERALS)
    out = [("uniform", fixed_batch(rows))]
    for base in (1, 17):
        out.append(("CSR base=%d" % base, csr_at(strings, base)))
    return out


# ------------------------------------------------------------------------------------------------ (1) NULL starts

@pytest.mark.parametrize("name", ["hf_glue10", "count_words5"] + sorted(COUNT_IMAGES))
def test_null_starts_equal_count_batch(name, cuda_device):
    """d_start == NULL: count_batch's counts widened to u64 and its match bits, in every count mode; states equal
    run_batch_from's from Initialize()."""
    import pire_b200 as P
    sc = P.Scanner(load(name), 0)
    rng = np.random.default_rng(sum(name.encode()))
    batches = batches_for(name, rng, sc.RegexpsCount())
    hb0 = batches[0][1]
    assert is_uniform(hb0.corpus_ptr(), hb0.offsets_ptr(), hb0.fixed_len)
    assert not is_uniform(batches[1][1].corpus_ptr(), batches[1][1].offsets_ptr(), batches[1][1].fixed_len)
    counted = 0
    for what, hb in batches:
        for flags in FLAGS:
            want = {}
            for mode in (1, 2, 3, 0):
                sc.set_count_mode(mode)
                label = "%s %s flags=%d mode=%d" % (name, what, flags, mode)
                counts, bits, states = Streams(sc, hb.n).round(hb, flags).results(label)
                wc, wb = count_batch(sc, hb, flags)
                expect_equal(label, "counts", counts, wc)
                expect_equal(label, "match bits", bits, wb)
                want.setdefault("states", states)
                expect_equal(label, "StateIndex across modes", states, want["states"])
                counted += int(counts.sum())
            check_against_run_from("%s %s flags=%d" % (name, what, flags), sc, hb, [sc.Initialize()] * hb.n, flags, bits, states)
    assert counted > 0


# ------------------------------------------------------------------------------------------- (2) rounds chained in place

def cut_strings(rng, strings, rounds):
    """Every string cut at its own random boundaries into `rounds` pieces: empty, 1-byte and short pieces included."""
    parts = []
    for k, s in enumerate(strings):
        if k % 4 == 0:
            cuts = sorted(int(c) for c in rng.integers(0, len(s) + 1, size=rounds - 1))
        else:
            step = [0, 1, int(rng.integers(2, 16))][k % 3]
            cuts = sorted(min(len(s), int(rng.integers(0, len(s) + 1)) + j * step) for j in range(rounds - 1))
        b = [0] + cuts + [len(s)]
        parts.append([s[b[r]:b[r + 1]] for r in range(rounds)])
    return parts


@pytest.mark.parametrize("name", ["hf_glue10", "count_words5", "w257"])
def test_rounds_chained_in_place(name, cuda_device):
    """Rounds through one state array (d_state_idx is d_start) and one counts array, with BEGIN on the first round and
    END on the last in every combination: the counts equal count_batch over the whole strings and the oracle per string;
    states and bits equal run_batch_from's."""
    import pire_b200 as P
    sc = P.Scanner(load(name), 0)
    orc = Oracle(load(name))
    rng = np.random.default_rng(40 + len(name))
    rounds = 4
    if name in COUNT_IMAGES:
        strings = w_strings(rng, sc.RegexpsCount(), 130, 200)
    else:
        strings = random_strings(rng, GLUE10_ALPHABET, [0, 1, 2, 15, 31] + [int(x) for x in rng.integers(0, 600, size=125)], LITERALS)
    parts = cut_strings(rng, strings, rounds)
    lens = np.array([[len(p[r]) for r in range(rounds)] for p in parts])
    assert (lens == 0).any() and (lens == 1).any() and ((lens > 1) & (lens < 16)).any()
    pieces = [csr_at([p[r] for p in parts], 5 * r + 1) for r in range(rounds)]
    whole = csr_batch(strings)
    # and a uniform chain: 1 KiB rows in four 256-byte rounds
    rows = random_rows(rng, 32 * 2 + 7, 1024, GLUE10_ALPHABET, LITERALS)
    if name in COUNT_IMAGES:
        rows = np.frombuffer(b"".join(s.ljust(1024, b"z")[:1024] for s in w_strings(rng, sc.RegexpsCount(), 71, 900)), np.uint8).reshape(-1, 1024)
    uni_whole = fixed_batch(rows)
    uni_pieces = [fixed_batch(np.ascontiguousarray(rows[:, 256 * r:256 * (r + 1)])) for r in range(rounds)]
    assert is_uniform(uni_pieces[1].corpus_ptr(), None, 256)
    for mode in (0, 1, 2, 3):
        sc.set_count_mode(mode)
        for flags in FLAGS:
            begin, end = flag_marks(flags)
            for what, wb, pcs in (("CSR", whole, pieces), ("uniform", uni_whole, uni_pieces)):
                label = "%s %s mode=%d flags=%d" % (name, what, mode, flags)
                s = Streams(sc, wb.n)
                for r, hb in enumerate(pcs):
                    s.round(hb, (RUN_BEGIN if begin and r == 0 else 0) | (RUN_END if end and r == rounds - 1 else 0))
                counts, bits, states = s.results(label)
                wc, wbits = count_batch(sc, wb, flags)
                expect_equal(label, "counts (count_batch on whole strings)", counts, wc)
                expect_equal(label, "match bits (count_batch)", bits, wbits)
                if mode == 0:
                    corpus, offs, fl = wb.oracle_args()
                    oc, ofin = oracle_count(orc, corpus, offs, fl, wb.n, begin, end)
                    expect_equal(label, "counts (oracle)", counts, oc.astype(np.int64))
                    expect_equal(label, "match bits (oracle)", bits, ofin)
                    check_against_run_from(label, sc, wb, [sc.Initialize()] * wb.n, flags, bits, states)


# ------------------------------------------------------------------------------------------------ (3) arbitrary starts

def test_every_state_as_a_start(cuda_device):
    """Every state of a small HalfFinalScanner, plus Size() and 0xFFFFFFFF, against count_from(start=...); two rounds
    chained in place, and starts outside the scanner add nothing in either round."""
    import pire_b200 as P
    case = GOLDEN_COUNTS[0]
    sc, orc = P.Scanner(case.image, 0), Oracle(case.image)
    size = sc.Size()
    rng = np.random.default_rng(9)
    texts = list(case.strings) + [b"", b"a", b"ab" * 9, bytes(rng.integers(0x20, 0x7F, size=45).astype(np.uint8))]
    states = list(range(size)) + [size, 0xFFFFFFFF]
    pairs = [(t, st) for st in states for t in texts]
    starts = np.array([p[1] for p in pairs], dtype=np.uint64)
    first = [p[0][: len(p[0]) // 2] for p in pairs]
    second = [p[0][len(p[0]) // 2:] for p in pairs]
    invalid = starts >= size
    whole = csr_at([p[0] for p in pairs], 0)
    for flags in FLAGS:
        begin, end = flag_marks(flags)
        want1 = oracle_from(orc, first, starts, RUN_BEGIN if begin else 0)
        want2 = oracle_from(orc, [a + b for a, b in zip(first, second)], starts, flags)
        for mode in (1, 2, 3):
            sc.set_count_mode(mode)
            label = "every state flags=%d mode=%d" % (flags, mode)
            s = Streams(sc, len(pairs), starts)
            s.round(csr_at(first, 3), RUN_BEGIN if begin else 0)
            counts, bits, st = s.results(label + " round 1")
            expect_equal(label, "counts after round 1", counts, want1[0])
            expect_equal(label, "states after round 1", st, want1[2])
            expect_equal(label, "bits after round 1", bits, want1[1])
            assert not counts[invalid].any() and (st[invalid] == 0xFFFFFFFF).all()
            s.round(csr_at(second, 1), RUN_END if end else 0)
            counts, bits, st = s.results(label + " round 2")
            expect_equal(label, "counts after round 2", counts, want2[0])
            expect_equal(label, "states after round 2", st, want2[2])
            expect_equal(label, "bits after round 2", bits, want2[1])
            assert not counts[invalid].any() and (st[invalid] == 0xFFFFFFFF).all()
            check_against_run_from(label, sc, whole, starts, flags, bits, st)


# ------------------------------------------------------------------------------------------------- (4) scanner shapes

SHAPES = [("hf_glue10", 255), ("hf_glue10", 2)] + [(name, h) for name in sorted(EDGE) for h in ((255, 2) if name == "wide" else (255, 2, 1))]


@pytest.mark.parametrize("name,max_hot", SHAPES)
def test_scanner_shapes(name, max_hot, cuda_device):
    """Hot sets of 255, 2 (and 1) rows: cold starts and walks that leave the hot rows, on hf_glue10 and the edge images
    (32-bit tables, NoExit starts, all-final); random starts with some outside the scanner, against the oracle's count
    walk and run_batch_from."""
    import pire_b200 as P
    image = load(name) if name not in EDGE else EDGE[name]["image"]
    sc, orc = P.Scanner(image, 0), Oracle(image)
    sc.set_max_hot(max_hot)
    assert sc.info().hot_rows <= max_hot
    alphabet, literals = (GLUE10_ALPHABET, LITERALS) if name not in EDGE else (ALPHABETS[name], EDGE_LITERALS[name])
    rng = np.random.default_rng(len(name) * 31 + max_hot)
    size = sc.Size()
    rows = random_rows(rng, 32 + 9, 128, alphabet, literals)
    ragged = csr_at(random_strings(rng, alphabet, [0, 1, 7, 16, 40] + [int(x) for x in rng.integers(0, 300, size=50)], literals), 3)
    noexit = [s for s in range(min(size, 300)) if all(sc.Next(s, b) == s for b in range(256))]   # no byte leaves them
    for what, hb in (("uniform", fixed_batch(rows)), ("CSR", ragged)):
        starts = random_starts(rng, size, hb.n)
        starts[0] = sc.Initialize()
        if noexit:
            starts[3::7] = noexit[0]
        strings = strings_of(hb)
        for flags in FLAGS:
            want = oracle_from(orc, strings, starts, flags)
            for mode in (1, 2, 3):
                sc.set_count_mode(mode)
                label = "%s max_hot=%d %s flags=%d mode=%d" % (name, max_hot, what, flags, mode)
                counts, bits, states = Streams(sc, hb.n, starts).round(hb, flags).results(label)
                expect_equal(label, "counts (oracle)", counts, want[0])
                expect_equal(label, "match bits (oracle)", bits, want[1])
                expect_equal(label, "StateIndex (oracle)", states, want[2])
            check_against_run_from(label, sc, hb, starts, flags, bits, states)


# ------------------------------------------------------------------------------------------------- (5) 64-bit adding

def test_counts_are_added_to_u64_rows(cuda_device):
    """Rows pre-filled near 2^32: the result is the prefill plus count_batch's counts, carried into the high word."""
    import pire_b200 as P
    sc = P.Scanner(load("hf_glue10"), 0)
    rng = np.random.default_rng(55)
    strings = [b"error timeout GET https://" * int(k) for k in rng.integers(1, 12, size=90)]
    strings += random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(0, 400, size=40)], LITERALS)
    hb = csr_at(strings, 7)
    regs = regs_of(sc)
    prefill = 0xFFFFFFF0 + (np.arange(hb.n * regs, dtype=np.int64).reshape(hb.n, regs) % 16)
    for mode in (1, 2, 3):
        sc.set_count_mode(mode)
        for flags in (0, RUN_BEGIN | RUN_END):
            label = "prefill mode=%d flags=%d" % (mode, flags)
            counts, _, _ = Streams(sc, hb.n, prefill=prefill).round(hb, flags).results(label)
            wc, _ = count_batch(sc, hb, flags)
            want = prefill + wc
            assert (want >= 1 << 32).any()
            expect_equal(label, "counts", counts, want)


# ---------------------------------------------------------------------------------------- (6) a stream joining late

@pytest.mark.parametrize("name", ["hf_glue10", "all_final"])
def test_stream_joining_in_a_later_round(name, cuda_device):
    """A stream whose start word is Initialize()'s StateIndex in round 2: its Initialize() TakeAction is not counted
    (as documented), which differs from a fresh start only when the initial state is final."""
    import pire_b200 as P
    image = load(name) if name not in EDGE else EDGE[name]["image"]
    sc, orc = P.Scanner(image, 0), Oracle(image)
    alphabet, literals = (GLUE10_ALPHABET, LITERALS) if name not in EDGE else (ALPHABETS[name], EDGE_LITERALS[name])
    rng = np.random.default_rng(66)
    n = 70
    first = random_strings(rng, alphabet, [int(x) for x in rng.integers(0, 200, size=n)], literals)
    second = random_strings(rng, alphabet, [int(x) for x in rng.integers(0, 200, size=n)], literals)
    joiners = np.arange(n) % 3 == 0
    first = [b"" if j else s for s, j in zip(first, joiners)]
    init = sc.Initialize()
    s = Streams(sc, n)
    s.round(csr_at(first, 0), RUN_BEGIN)
    s.state[:n] = _i32(np.where(joiners, init, _host(s.state)[:n].astype(np.uint64)))
    s.counts[:n][torch_bool(joiners)] = 0
    s.round(csr_at(second, 2), RUN_END)
    counts, bits, states = s.results(name + " joining")
    for i in range(n):
        if joiners[i]:
            want, res = count_from(orc, np.frombuffer(second[i], np.uint8), init, False, True)
            fresh, _ = count_from(orc, np.frombuffer(second[i], np.uint8), None, False, True)
            taken = np.array(fresh) - np.array(want)          # Initialize()'s TakeAction
            assert taken.any() == (sc.Final(init) and bool(sc.AcceptedRegexps(init))), (i, taken)
        else:
            want, res = count_from(orc, np.frombuffer(first[i] + second[i], np.uint8), None, True, True)
        assert counts[i].tolist() == want, (name, i)
        assert (int(bits[i]), int(states[i])) == (res[0], res[2]), (name, i)
    if name == "all_final":
        assert sc.Final(init) and sc.AcceptedRegexps(init)      # the rule changes the counts here


def torch_bool(mask):
    import torch
    return torch.from_numpy(np.asarray(mask, bool)).to("cuda:0")


# ------------------------------------------------------------------------------------------------- (7) bad arguments

def test_bad_arguments_empty_scanner_and_n_zero(cuda_device):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    sc = P.Scanner(load("hf_glue10"), 0)
    hb = fixed_batch(random_rows(np.random.default_rng(1), 40, 64, GLUE10_ALPHABET))
    s = Streams(sc, 40)
    lib = N.lib

    def call(h, corpus, offs, fl, n, flags, counts=s.counts.data_ptr(), start=None):
        return lib.pire_gpu_count_batch_from(h, corpus, offs, fl, n, flags, start, counts, s.bits.data_ptr(), s.state.data_ptr(),
                                             _stream())
    for flags in (RUN_LINES, RUN_LINES | RUN_BEGIN, 8, 1 << 31):
        assert call(sc._h, hb.corpus_ptr(), None, 64, 40, flags) == -1
    assert call(sc._h, hb.corpus_ptr(), None, 64, 40, 3, counts=None) == -1                 # NULL counts
    assert call(sc._h, None, None, 64, 40, 3) == -1                                         # NULL corpus, fixed length
    assert call(sc._h, None, csr_batch([b"ab"]).offsets_ptr(), 0, 1, 3) == -1              # NULL corpus, CSR
    assert call(sc._h, None, None, 0, (1 << 40) + 1, 3) == -1                               # n > 2^40
    assert call(None, hb.corpus_ptr(), None, 64, 40, 3) == -1
    torch.cuda.synchronize()
    assert (s.counts.cpu().numpy()[:40] == 0).all()
    # n == 0 writes nothing, whatever the pointers
    assert call(sc._h, None, None, 0, 0, 3) == 0
    assert call(sc._h, hb.corpus_ptr(), None, 64, 0, 3, start=s.state.data_ptr()) == 0
    torch.cuda.synchronize()
    assert (s.counts.cpu().numpy()[:40] == 0).all()
    assert (_host(s.state) == SENTINEL).all() and (_host(s.bits) == SENTINEL).all()
    # strings of length 0 with a NULL corpus are fine: the marks alone
    e0 = Streams(sc, 33)
    N.check(lib.pire_gpu_count_batch_from(sc._h, None, None, 0, 33, 3, None, e0.counts.data_ptr(), e0.bits.data_ptr(),
                                          e0.state.data_ptr(), _stream()), "empty strings")
    counts, bits, states = e0.results("empty strings")
    want = oracle_from(Oracle(load("hf_glue10")), [b""] * 33, None, 3)
    expect_equal("empty strings", "counts", counts, want[0])
    expect_equal("empty strings", "StateIndex", states, want[2])
    # the empty scanner
    empty = next(x for x in GOLDEN if x.name == "EmptyScanner@784")
    e = P.Scanner(empty.image, 0)
    rng = np.random.default_rng(2)
    hb = csr_at(random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(0, 300, size=50)]), 1)
    for flags in FLAGS:
        counts, bits, states = Streams(e, hb.n).round(hb, flags).results("empty scanner")
        wc, wb = count_batch(e, hb, flags)
        expect_equal("empty scanner", "counts", counts, wc)
        expect_equal("empty scanner", "match bits", bits, wb)
        check_against_run_from("empty scanner", e, hb, [e.Initialize()] * hb.n, flags, bits, states)


# --------------------------------------------------------------------------------------------- (8) Python and C++

def test_python_batch_counter(cuda_device):
    """BatchCounter(sc, n) round after round, and BatchCounter(sc, n, prev.StateTensor()) resumed, equal HalfFinalCount
    over the whole strings; batches it cannot take raise ValueError."""
    import torch
    import pire_b200 as P
    sc = P.Scanner(load("hf_glue10"), 0)
    rng = np.random.default_rng(77)
    n, length, rounds = 32 * 9 + 5, 512, 4
    rows = random_rows(rng, n, length, GLUE10_ALPHABET, LITERALS)
    whole = P.HalfFinalCount(sc, P.Batch(torch.from_numpy(rows.reshape(-1).copy()).to("cuda:0"), fixed_len=length, n=n))
    pieces = []
    for r in range(rounds):
        piece = np.ascontiguousarray(rows[:, r * length // rounds:(r + 1) * length // rounds])
        pieces.append(P.Batch(torch.from_numpy(piece.reshape(-1)).to("cuda:0"), fixed_len=piece.shape[1], n=n))
    c = P.BatchCounter(sc, n).Begin()
    for b in pieces:
        c.Run(b)
    c.End()
    assert c.Counts().shape == (n, regs_of(sc)) and c.Counts().dtype == torch.int64 and c.StateTensor().dtype == torch.int32
    assert (c.Counts().cpu().numpy() == whole.counts.astype(np.int64)).all()
    assert (c.Matches() == np.array([whole.Final(i) for i in range(n)])).all()
    for i in (0, 7, n - 1):
        assert c.AcceptedRegexps(i) == whole.AcceptedRegexps(i)
        assert c.Final(i) == whole.Final(i)
        assert all(c.Result(i, r) == whole.Result(i, r) for r in range(regs_of(sc)))
    # the first two rounds, then a second counter resumed from their states (counted from there on)
    a = P.BatchCounter(sc, n).Begin().Run(pieces[0]).Run(pieces[1])
    b = P.BatchCounter(sc, n, a.StateTensor()).Run(pieces[2]).Run(pieces[3]).End()
    assert ((a.Counts() + b.Counts()).cpu().numpy() == whole.counts.astype(np.int64)).all()
    runner = P.Runner(sc).Begin().Run(P.Batch(torch.from_numpy(rows.reshape(-1).copy()).to("cuda:0"), fixed_len=length, n=n)).End()
    assert (b.States() == runner.States()).all()
    # nothing run: the start states themselves
    fresh = P.BatchCounter(sc, 3)
    assert (fresh.States() == sc.Initialize()).all()
    with pytest.raises(ValueError):
        P.BatchCounter(sc, n + 1).Run(pieces[0])
    with pytest.raises(ValueError):
        P.BatchCounter(sc, 2).Run(P.Batch.from_text(torch.tensor(list(b"a\nb\n"), dtype=torch.uint8, device="cuda:0")))
    with pytest.raises(ValueError):
        P.BatchCounter(sc, 3).Run(P.Batch.from_strings([b"a", b"bb", b"ccc"]).bin_by_length())


def test_cpp_batch_counter(tmp_path, cuda_device):
    """tests/cpp/batch_count_check.cpp through include/pire_gpu.hpp's BatchCounter: rounds chained in place, and a counter
    resumed with BatchCounter::From, equal pire_gpu_count_batch over the whole strings."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "batch_count_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "batch_count_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    image = tmp_path / "hf_glue10.pire"
    image.write_bytes(W.load_image("hf_glue10"))
    for n, length, rounds in ((100_003, 1024, 4), (33, 256, 8), (1, 32, 2)):
        out = subprocess.run([exe, str(image), str(n), str(length), str(rounds), "7"], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ": 0 mismatches" in out.stdout, out.stdout
