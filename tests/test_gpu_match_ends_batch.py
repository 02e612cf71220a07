"""pire_gpu_match_ends_batch_from: where the HalfFinalScanner matches end in many streams at once, each from Initialize()
or resumed from its own state, with the states and the streams' byte offsets carried in place from round to round.

The independent answers are pire_gpu_match_ends_string called once per string (start and base per string, appended
through one *d_found: their concatenation is what the batch call must write), the in-repo oracle's positions walk
(ends_from of test_gpu_match_ends.py), pire_gpu_count_batch_from's rows for the per-string histograms and
pire_gpu_run_batch_from's match bits and states.  Every output buffer is longer than the call may write and pre-filled
with a sentinel that must survive: entries below the incoming *d_found and past the capacity, and state, position and
bitmap words past n."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN_COUNTS, ROOT
from refpire import Oracle
from test_count_images import COUNT_IMAGES, w_strings
from test_edge_images import ALPHABETS, EDGE
from test_gpu_batch_count_resume import FLAGS, LITERALS, RUN_BEGIN, RUN_END, RUN_LINES, Streams, cut_strings, flag_marks, load, regs_of
from test_gpu_batch_resume import _i32, csr_at, random_starts, run_from_batch, strings_of
from test_gpu_count_edges import LITERALS as EDGE_LITERALS
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, SENTINEL, HostBatch, _filled, _host, _stream, csr_batch, expect_equal,
                            expect_untouched, fixed_batch, is_uniform, random_rows, random_strings, unpack_bits)
from test_gpu_match_ends import GUARD, SENTINEL64, ends_from

pytestmark = pytest.mark.gpu

BELOW = 3                       # sentinel entries before the incoming *d_found


def _u64(values, extra=EXTRA):
    import torch
    v = np.concatenate([np.asarray(values, np.uint64), np.full(extra, SENTINEL64, np.uint64)]).view(np.int64)
    return torch.from_numpy(v.copy()).to("cuda:0")


class Calls:
    """One batch call's buffers: entry arrays of BELOW + capacity + GUARD entries, *d_found = BELOW on entry, and
    state, position and bitmap words past n, all sentinel-filled."""

    def __init__(self, sc, n, capacity, starts=None, pos=None):
        import torch
        self.sc, self.n, self.capacity = sc, n, BELOW + capacity
        size = self.capacity + GUARD
        self.strings = _filled(size)
        self.ends = torch.full((size,), SENTINEL64, dtype=torch.int64, device="cuda:0")
        self.ids = _filled(size)
        self.found = torch.tensor([BELOW], dtype=torch.int64, device="cuda:0")
        self.state = _filled(n + EXTRA)
        if starts is not None:
            self.state[:n] = _i32(starts)
        self.pos = None if pos is None else _u64(pos)
        self.bits = _filled((n + 31) // 32 + 1)
        self.resumed = starts is not None

    def round(self, hb, flags, arrays=(True, True, True)):
        """One call with d_start == d_state_idx (or NULL before the first round of fresh streams)."""
        from pire_b200 import _native as N
        s, e, i = (t.data_ptr() if on else None for t, on in zip((self.strings, self.ends, self.ids), arrays))
        N.check(N.lib.pire_gpu_match_ends_batch_from(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, self.n, flags,
                                                     self.state.data_ptr() if self.resumed else None,
                                                     None if self.pos is None else self.pos.data_ptr(), s, e, i, self.capacity,
                                                     self.found.data_ptr(), self.bits.data_ptr(), self.state.data_ptr(), _stream()),
                "pire_gpu_match_ends_batch_from")
        self.resumed = True
        return self

    def results(self, label):
        """(strings, ends, ids, found, bits, states, pos) on the host, every sentinel checked."""
        found = int(self.found.item()) - BELOW
        top = min(BELOW + found, self.capacity)
        s, i = _host(self.strings), _host(self.ids)
        e = self.ends.cpu().numpy().view(np.uint64)
        for what, arr, sent in (("strings", s, SENTINEL), ("ends", e, SENTINEL64), ("ids", i, SENTINEL)):
            assert (arr[:BELOW] == sent).all(), "%s: %s written below the incoming *d_found" % (label, what)
            assert (arr[top:] == sent).all(), "%s: %s written past the entries or the capacity" % (label, what)
        states = _host(self.state)
        expect_untouched(label, "state indices", states, self.n)
        pos = None
        if self.pos is not None:
            pos = self.pos.cpu().numpy().view(np.uint64)
            assert (pos[self.n:] == SENTINEL64).all(), "%s: positions written past n" % label
            pos = pos[: self.n]
        return s[BELOW:top], e[BELOW:top], i[BELOW:top], found, unpack_bits(label, _host(self.bits), self.n), states[: self.n], pos


def batch_ends(sc, hb, flags, starts=None, pos=None, capacity=None):
    """One call with room for every entry (unless `capacity`): the results of Calls.results."""
    if capacity is None:
        capacity = int(count_rows(sc, hb, flags, starts).sum())
    return Calls(sc, hb.n, capacity, starts, pos).round(hb, flags).results("match_ends_batch_from")


def count_rows(sc, hb, flags, starts=None):
    """pire_gpu_count_batch_from's rows (n, regs)."""
    s = Streams(sc, hb.n, starts)
    return s.round(hb, flags).results("count_batch_from")[0]


def per_string(sc, hb, flags, starts=None, pos=None):
    """pire_gpu_match_ends_string once per string of the batch, start starts[i] (or NULL) and base pos[i] (or 0), all
    appended through one *d_found with no synchronise: (ends, ids, found, match, state per string)."""
    import torch
    from pire_b200 import _native as N
    strings = strings_of(hb)
    corpus, offs, fl = hb.oracle_args()
    cap = sum(16 * (len(x) + 2) for x in strings) + 16
    ends = torch.empty(cap, dtype=torch.int64, device="cuda:0")
    ids = torch.empty(cap, dtype=torch.int32, device="cuda:0")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    words = torch.empty((hb.n, 2), dtype=torch.int32, device="cuda:0")
    st = None if starts is None else _i32(starts)
    for k in range(hb.n):
        off = int(offs[k]) if offs is not None else k * fl
        N.check(N.lib.pire_gpu_match_ends_string(sc._h, hb.corpus_ptr() + off if len(strings[k]) else None, len(strings[k]), flags,
                                                 None if st is None else st.data_ptr() + 4 * k, 0 if pos is None else int(pos[k]),
                                                 ends.data_ptr(), ids.data_ptr(), cap, found.data_ptr(), words[k].data_ptr(),
                                                 words[k].data_ptr() + 4, _stream()), "pire_gpu_match_ends_string")
    total = int(found.item())
    assert total <= cap
    w = _host(words).reshape(hb.n, 2)
    return ends.cpu().numpy().view(np.uint64)[:total], _host(ids)[:total], total, w[:, 0] & 1, w[:, 1]


def histogram(strings, ids, n, regs):
    return np.bincount(strings.astype(np.int64) * regs + ids.astype(np.int64), minlength=n * regs).reshape(n, regs)


def check_batch(label, sc, hb, flags, starts=None, pos=None):
    """One batch call against per-string match_ends_string calls, count_batch_from's rows and run_batch_from."""
    rows = count_rows(sc, hb, flags, starts)
    s, e, i, found, bits, states, newpos = batch_ends(sc, hb, flags, starts, pos)
    we, wi, wfound, wmatch, wstate = per_string(sc, hb, flags, starts, pos)
    assert found == wfound == int(rows.sum()), (label, found, wfound, int(rows.sum()))
    expect_equal(label, "ends (match_ends_string per string)", e, we)
    expect_equal(label, "ids (match_ends_string per string)", i, wi)
    assert (np.diff(s.astype(np.int64)) >= 0).all(), "%s: entries out of string order" % label
    expect_equal(label, "per-string histograms (count_batch_from)", histogram(s, i, hb.n, regs_of(sc)), rows)
    expect_equal(label, "StateIndex (match_ends_string)", states, wstate)
    expect_equal(label, "match bits (match_ends_string)", bits, wmatch)
    begin, end = flag_marks(flags)
    wbits, _, wstates = run_from_batch(sc, hb, [sc.Initialize()] * hb.n if starts is None else starts, begin, end)
    expect_equal(label, "StateIndex (run_batch_from)", states, wstates)
    expect_equal(label, "match bits (run_batch_from)", bits, wbits)
    if pos is not None:
        lens = np.array([len(x) for x in strings_of(hb)], np.uint64)
        expect_equal(label, "positions advanced", newpos, np.asarray(pos, np.uint64) + lens)
    return found


def glue10_batches(rng):
    """Ragged CSR batches at unaligned starts (empty strings among them), a uniform fixed-length batch and fixed_len 0."""
    strings = random_strings(rng, GLUE10_ALPHABET, [0, 1, 15, 16, 17, 33, 0] + [int(x) for x in rng.integers(0, 700, size=90)], LITERALS)
    rows = random_rows(rng, 32 * 2 + 5, 256, GLUE10_ALPHABET, LITERALS)
    out = [("CSR base=%d" % b, csr_at(strings, b)) for b in (1, 17)]
    out.append(("uniform", fixed_batch(rows)))
    out.append(("fixed_len 0", HostBatch(np.zeros(64, np.uint8), fixed_len=0, n=45)))
    return out


# ------------------------------------------------------------------------------------------------------ (1) golden

def test_golden_counts(cuda_device):
    """The count_ut.cpp strings as one CSR batch, max_hot 255 and 3: the oracle walk per string, concatenated, and the
    fixture counts per string."""
    import pire_b200 as P
    for k, case in enumerate(GOLDEN_COUNTS):
        orc = Oracle(case.image)
        hb = csr_batch(case.strings)
        for max_hot in (255, 3):
            sc = P.Scanner(case.image, 0)
            sc.set_max_hot(max_hot)
            s, e, i, found, bits, states, _ = batch_ends(sc, hb, RUN_BEGIN | RUN_END)
            want = [ends_from(orc, np.frombuffer(x, np.uint8)) for x in case.strings]
            label = "golden case %d max_hot=%d" % (k, max_hot)
            expect_equal(label, "ends (oracle)", e, np.concatenate([w[0] for w in want]))
            expect_equal(label, "ids (oracle)", i, np.concatenate([w[1] for w in want]))
            expect_equal(label, "strings", s, np.concatenate([np.full(len(w[0]), j, np.uint32) for j, w in enumerate(want)]))
            expect_equal(label, "histograms (fixture)", histogram(s, i, hb.n, regs_of(sc)), np.array(case.counts, np.int64))
            expect_equal(label, "match bits (fixture)", bits, np.array(case.final, np.uint8))
            assert found == sum(map(sum, case.counts))


# ---------------------------------------------------------------------------------------------- (2) differential

@pytest.mark.parametrize("name", ["hf_glue10", "count_words5"])
def test_differential(name, cuda_device):
    """Every batch shape, the four flag combinations, NULL and random starts (>= Size() among them), NULL and non-zero
    positions: per string what match_ends_string writes."""
    import pire_b200 as P
    sc = P.Scanner(load(name), 0)
    rng = np.random.default_rng(sum(name.encode()) + 5)
    batches = glue10_batches(rng)
    hb = batches[2][1]
    assert is_uniform(hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len)
    assert not is_uniform(batches[0][1].corpus_ptr(), batches[0][1].offsets_ptr(), batches[0][1].fixed_len)
    total = 0
    for what, hb in batches:
        for flags in FLAGS:
            for starts in (None, random_starts(rng, sc.Size(), hb.n)):
                for pos in (None, rng.integers(0, 1 << 40, size=hb.n).astype(np.uint64)):
                    label = "%s %s flags=%d starts=%s pos=%s" % (name, what, flags, starts is not None, pos is not None)
                    total += check_batch(label, sc, hb, flags, starts, pos)
    assert total > 100


# ----------------------------------------------------------------------------------------------------- (3) rounds

@pytest.mark.parametrize("name", ["hf_glue10", "count_words5", "w257"])
def test_rounds_chained_in_place(name, cuda_device):
    """Four rounds through one state array (d_start == d_state_idx) and one position array advanced by the calls,
    appended through one *d_found: taken stream by stream, the entries of one call over the whole strings, byte for
    byte; states, bits and positions too.  Some streams are empty in some rounds."""
    import pire_b200 as P
    sc = P.Scanner(load(name), 0)
    rng = np.random.default_rng(90 + len(name))
    rounds = 4
    if name in COUNT_IMAGES:
        strings = w_strings(rng, sc.RegexpsCount(), 130, 200)
    else:
        strings = random_strings(rng, GLUE10_ALPHABET, [0, 1, 2, 15, 31] + [int(x) for x in rng.integers(0, 600, size=125)], LITERALS)
    parts = cut_strings(rng, strings, rounds)
    lens = np.array([[len(p[r]) for r in range(rounds)] for p in parts])
    assert (lens == 0).any() and (lens == 1).any()
    pieces = [csr_at([p[r] for p in parts], 5 * r + 1) for r in range(rounds)]
    whole = csr_batch(strings)
    rows = random_rows(rng, 32 * 2 + 7, 1024, GLUE10_ALPHABET, LITERALS)
    if name in COUNT_IMAGES:
        rows = np.frombuffer(b"".join(s.ljust(1024, b"z")[:1024] for s in w_strings(rng, sc.RegexpsCount(), 71, 900)), np.uint8).reshape(-1, 1024)
    uni_whole = fixed_batch(rows)
    uni_pieces = [fixed_batch(np.ascontiguousarray(rows[:, 256 * r:256 * (r + 1)])) for r in range(rounds)]
    assert is_uniform(uni_pieces[1].corpus_ptr(), None, 256)
    seen = 0
    for flags in FLAGS:
        begin, end = flag_marks(flags)
        for what, wb, pcs in (("CSR", whole, pieces), ("uniform", uni_whole, uni_pieces)):
            label = "%s %s flags=%d" % (name, what, flags)
            want = batch_ends(sc, wb, flags, pos=np.zeros(wb.n, np.uint64))
            c = Calls(sc, wb.n, want[3], pos=np.zeros(wb.n, np.uint64))
            for r, hb in enumerate(pcs):
                c.round(hb, (RUN_BEGIN if begin and r == 0 else 0) | (RUN_END if end and r == rounds - 1 else 0))
            s, e, i, found, bits, states, pos = c.results(label)
            assert found == want[3], label
            seen += found
            order = np.argsort(s, kind="stable")
            expect_equal(label, "strings", s[order], want[0])
            expect_equal(label, "ends", e[order], want[1])
            expect_equal(label, "ids", i[order], want[2])
            expect_equal(label, "match bits", bits, want[4])
            expect_equal(label, "StateIndex", states, want[5])
            expect_equal(label, "positions", pos, want[6])
            expect_equal(label, "positions (lengths)", pos, np.array([len(x) for x in strings_of(wb)], np.uint64))
    assert seen > 0


# --------------------------------------------------------------------------------------------------- (4) capacity

def test_capacity(cuda_device):
    """Capacity 0, 1, inside a string's slice, on a slice boundary and the exact total: the written entries are the
    answer's first `capacity`, *d_found the full total; each of the three arrays may be NULL."""
    import pire_b200 as P
    sc = P.Scanner(load("count_words5"), 0)
    rng = np.random.default_rng(11)
    hb = csr_at(random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(0, 400, size=70)], LITERALS), 3)
    flags = RUN_BEGIN | RUN_END
    full = batch_ends(sc, hb, flags)
    total = full[3]
    per = np.bincount(full[0].astype(np.int64), minlength=hb.n)
    j = int(np.nonzero(per[1:] >= 2)[0][0])             # string j + 1 has two entries or more
    boundary = int(per[: j + 1].sum())                  # where its slice begins
    inside = boundary + 1
    assert total > 50 and 0 < boundary < inside < total
    # -BELOW: an ABI capacity of 0, below the incoming *d_found
    for cap in (-BELOW, 0, 1, boundary, inside, total - 1, total):
        label = "capacity %d" % cap
        s, e, i, found, bits, states, _ = Calls(sc, hb.n, cap).round(hb, flags).results(label)
        k = max(0, min(cap, total))
        assert found == total, (cap, found, total)
        expect_equal(label, "strings", s, full[0][:k])
        expect_equal(label, "ends", e, full[1][:k])
        expect_equal(label, "ids", i, full[2][:k])
        expect_equal(label, "StateIndex", states, full[5])
        expect_equal(label, "match bits", bits, full[4])
    for arrays in ((False, True, True), (True, False, True), (True, True, False), (False, False, False)):
        c = Calls(sc, hb.n, total).round(hb, flags, arrays)
        s, e, i, found, bits, states, _ = c.results("NULL arrays %s" % (arrays,))
        assert found == total
        for on, got, want, sent in zip(arrays, (s, e, i), full[:3], (SENTINEL, SENTINEL64, SENTINEL)):
            assert (got == want).all() if on else (got == sent).all(), arrays


# --------------------------------------------------------------------------------------------------- (5) scanners

SHAPES = [(name, h) for name in sorted(EDGE) for h in ((255, 2) if name == "wide" else (255, 2, 1))] + \
         [(name, 255) for name in sorted(COUNT_IMAGES)]


@pytest.mark.parametrize("name,max_hot", SHAPES)
def test_scanner_shapes(name, max_hot, cuda_device):
    """The edge images at hot sets of 255, 2 and 1, and the count images past 256 regexps: a CSR and a uniform batch,
    NULL and random starts."""
    import pire_b200 as P
    image = EDGE[name]["image"] if name in EDGE else COUNT_IMAGES[name]["image"]
    sc = P.Scanner(image, 0)
    sc.set_max_hot(max_hot)
    rng = np.random.default_rng(len(name) * 7 + max_hot)
    if name in COUNT_IMAGES:
        strings = w_strings(rng, sc.RegexpsCount(), 90, 300)
        rows = np.frombuffer(b"".join(s.ljust(128, b"q")[:128] for s in w_strings(rng, sc.RegexpsCount(), 40, 120)), np.uint8).reshape(-1, 128)
    else:
        alphabet = ALPHABETS[name] + b"".join(EDGE_LITERALS.get(name, []))
        strings = random_strings(rng, alphabet, [0, 1, 17] + [int(x) for x in rng.integers(0, 500, size=60)], EDGE_LITERALS.get(name, ()))
        rows = random_rows(rng, 40, 128, alphabet, EDGE_LITERALS.get(name, ()))
    for what, hb in (("CSR", csr_at(strings, 7)), ("uniform", fixed_batch(rows))):
        for flags in (RUN_BEGIN | RUN_END, 0):
            for starts in (None, random_starts(rng, sc.Size(), hb.n)):
                check_batch("%s max_hot=%d %s flags=%d" % (name, max_hot, what, flags), sc, hb, flags, starts,
                            rng.integers(0, 1 << 33, size=hb.n).astype(np.uint64))


# -------------------------------------------------------------------------------------------------- (6) arguments

def test_bad_arguments_and_n_zero(cuda_device):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    sc = P.Scanner(load("hf_glue10"), 0)
    hb = fixed_batch(random_rows(np.random.default_rng(1), 40, 64, GLUE10_ALPHABET))
    c = Calls(sc, 40, 100, pos=np.zeros(40, np.uint64))

    def call(h, corpus, offs, fl, n, flags, found=c.found.data_ptr(), start=None):
        return N.lib.pire_gpu_match_ends_batch_from(h, corpus, offs, fl, n, flags, start, c.pos.data_ptr(), c.strings.data_ptr(),
                                                    c.ends.data_ptr(), c.ids.data_ptr(), c.capacity, found, c.bits.data_ptr(),
                                                    c.state.data_ptr(), _stream())
    for flags in (RUN_LINES, RUN_LINES | RUN_BEGIN, 8, 1 << 31):
        assert call(sc._h, hb.corpus_ptr(), None, 64, 40, flags) == -1
    assert call(sc._h, hb.corpus_ptr(), None, 64, 40, 3, found=None) == -1                 # NULL d_found
    assert call(sc._h, None, None, 64, 40, 3) == -1                                        # NULL corpus, fixed length
    assert call(sc._h, None, csr_batch([b"ab"]).offsets_ptr(), 0, 1, 3) == -1              # NULL corpus, CSR
    assert call(sc._h, None, None, 0, 1 << 32, 3) == -1                                    # n >= 2^32
    assert call(None, hb.corpus_ptr(), None, 64, 40, 3) == -1
    # n == 0 writes nothing, whatever the pointers
    assert call(sc._h, None, None, 0, 0, 3) == 0
    assert call(sc._h, hb.corpus_ptr(), None, 64, 0, 3, start=c.state.data_ptr()) == 0
    torch.cuda.synchronize()
    assert int(c.found.item()) == BELOW and (c.pos.cpu().numpy().view(np.uint64)[:40] == 0).all()
    assert (_host(c.strings) == SENTINEL).all() and (_host(c.ids) == SENTINEL).all() and (c.ends.cpu().numpy().view(np.uint64) == SENTINEL64).all()
    assert (_host(c.state) == SENTINEL).all() and (_host(c.bits) == SENTINEL).all()
    # strings of length 0 with a NULL corpus are fine: the marks alone
    e0 = Calls(sc, 33, 100)
    N.check(N.lib.pire_gpu_match_ends_batch_from(sc._h, None, None, 0, 33, 3, None, None, e0.strings.data_ptr(), e0.ends.data_ptr(),
                                                 e0.ids.data_ptr(), e0.capacity, e0.found.data_ptr(), e0.bits.data_ptr(),
                                                 e0.state.data_ptr(), _stream()), "empty strings")
    s, e, i, found, bits, states, _ = e0.results("empty strings")
    want = ends_from(Oracle(load("hf_glue10")), np.zeros(0, np.uint8))
    assert found == 33 * len(want[0]) and (e == np.tile(want[0], 33)).all() and (i == np.tile(want[1], 33)).all()


# ---------------------------------------------------------------------------------------------- (7) Python and C++

def test_python_batch_match_ends(cuda_device):
    """BatchMatchEnds(sc, n, capacity) round after round equals BatchCounter's counts and states; resumed from a state
    tensor it reports nothing twice; batches it cannot take raise ValueError."""
    import torch
    import pire_b200 as P
    sc = P.Scanner(load("hf_glue10"), 0)
    rng = np.random.default_rng(78)
    n, length, rounds = 32 * 5 + 3, 512, 4
    rows = random_rows(rng, n, length, GLUE10_ALPHABET, LITERALS)
    pieces = []
    for r in range(rounds):
        piece = np.ascontiguousarray(rows[:, r * length // rounds:(r + 1) * length // rounds])
        pieces.append(P.Batch(torch.from_numpy(piece.reshape(-1)).to("cuda:0"), fixed_len=piece.shape[1], n=n))
    c = P.BatchCounter(sc, n).Begin()
    m = P.BatchMatchEnds(sc, n, 100_000).Begin()
    for b in pieces:
        c.Run(b)
        m.Run(b)
    c.End()
    m.End()
    counts = c.Counts().cpu().numpy()
    assert m.Found() == int(counts.sum()) > 0
    s, e, i = m.Strings(), m.Ends(), m.Ids()
    assert s.dtype == np.uint32 and e.dtype == np.uint64 and i.dtype == np.uint32
    assert (histogram(s, i, n, regs_of(sc)) == counts).all() and (e <= length).all()
    assert (m.States() == c.States()).all() and (m.Matches() == c.Matches()).all()
    assert (m.PosTensor().cpu().numpy() == length).all()
    for t in (m.StringsTensor(), m.EndsTensor(), m.IdsTensor(), m.FoundTensor(), m.StateTensor(), m.PosTensor()):
        assert t.is_cuda
    # the first two rounds, then one resumed from their states: the entries of the last two rounds, ends counted from
    # the start of the resumed object's bytes
    a = P.BatchMatchEnds(sc, n, 100_000).Begin().Run(pieces[0]).Run(pieces[1])
    b = P.BatchMatchEnds(sc, n, 100_000, a.StateTensor()).Run(pieces[2]).Run(pieces[3]).End()
    assert a.Found() + b.Found() == m.Found()
    late = e > length // 2
    assert (np.sort(b.Ends().astype(np.int64) + length // 2) == np.sort(e[late].astype(np.int64))).all()
    assert (b.States() == m.States()).all()
    # short capacity: the first entries, the full total
    short = P.BatchMatchEnds(sc, n, 5).Begin()
    for p in pieces:
        short.Run(p)
    short.End()
    assert short.Found() == m.Found() and len(short.Ends()) == 5
    assert (P.BatchMatchEnds(sc, 3, 4).States() == sc.Initialize()).all()
    with pytest.raises(ValueError):
        P.BatchMatchEnds(sc, n + 1, 4).Run(pieces[0])
    with pytest.raises(ValueError):
        P.BatchMatchEnds(sc, 2, 4).Run(P.Batch.from_text(torch.tensor(list(b"a\nb\n"), dtype=torch.uint8, device="cuda:0")))
    with pytest.raises(ValueError):
        P.BatchMatchEnds(sc, 3, 4).Run(P.Batch.from_strings([b"a", b"bb", b"ccc"]).bin_by_length())
    with pytest.raises(ValueError):
        P.BatchMatchEnds(sc, 3, 4, torch.zeros(3, dtype=torch.int64, device="cuda:0"))


def test_cpp_batch_match_ends(tmp_path, cuda_device):
    """tests/cpp/match_ends_batch_check.cpp through include/pire_gpu.hpp's BatchMatchEnds: chained and resumed rounds
    equal one call over the whole strings, stream by stream, and BatchCounter's counts."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "match_ends_batch_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "match_ends_batch_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    for name in ("hf_glue10", "count_words5"):
        image = tmp_path / (name + ".pire")
        image.write_bytes(W.load_image(name))
        for n, length, rounds in ((20_003, 1024, 4), (33, 256, 8), (1, 32, 2)):
            out = subprocess.run([exe, str(image), str(n), str(length), str(rounds), "7"], capture_output=True, text=True, timeout=300)
            assert out.returncode == 0, out.stdout + out.stderr
            assert ": 0 mismatches" in out.stdout, out.stdout
