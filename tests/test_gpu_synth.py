"""Every scan family on synthesized automata (tests/synth_dfa.py), bit for bit against the plain walker over the
generator's own tables.  The automata are written from fixed seeds in this process: nothing here needs the reference
or recorded answers.  They reach the table shapes compiled regexes rarely make: hot sets of exactly 254-256 rows, PRIV's
tier edges, a first hot row that leaves the hot set (no look-ahead filter), 65 536 and 65 537 states, walks that
converge late or never, marks that lead where no byte does, absorbing finals, and accept lists that name an id 15 or 16
times.  Every output buffer is larger than the answer and pre-filled with a sentinel that must survive past its end."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import refpire  # noqa: E402
import synth_dfa as SD  # noqa: E402

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END = 1, 2
MARKS = ((True, True), (False, False), (True, False), (False, True))
SENTINEL = 0x5A5A5A5A
SENTINEL64 = 0x5A5A5A5A5A5A5A5A
EXTRA = 64
NO_PREFIX = 0xFFFFFFFF

RUN_FAMILIES = sorted(n for n in SD.FAMILIES if not n.startswith("count_"))
COUNT_FAMILIES = sorted(n for n in SD.FAMILIES if n.startswith("count_")) + ["uniform_p1", "marks", "absorb_early", "width_65537",
                                                                          "hot_255"]


def _flags(begin, end):
    return (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)


def _stream():
    import torch
    return torch.cuda.current_stream(0).cuda_stream


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _filled(count, wide=False):
    import torch
    if wide:
        return torch.full((count,), SENTINEL64, dtype=torch.int64, device="cuda:0")
    return torch.full((count,), SENTINEL, dtype=torch.int32, device="cuda:0")


def _host(t, valid, label, what):
    """The first ``valid`` entries of an output, after checking that everything past them still holds the sentinel."""
    h = t.cpu().numpy()
    h = h.view(np.uint64) if h.dtype == np.int64 else h.view(np.uint32)
    tail = h[valid:]
    sentinel = SENTINEL64 if h.dtype == np.uint64 else SENTINEL
    if not (tail == sentinel).all():
        k = int(np.nonzero(tail != sentinel)[0][0])
        raise AssertionError("%s: %s written past its end: [%d] = %#x" % (label, what, valid + k, int(tail[k])))
    return h[:valid]


def _bits(t, n, label):
    words = _host(t, (n + 31) // 32, label, "match bits")
    if n % 32:
        assert int(words[-1]) >> (n % 32) == 0, "%s: match bits past n set" % label
    return ((words[np.arange(n) // 32] >> (np.arange(n) % 32).astype(np.uint32)) & 1).astype(np.uint8)


def expect(label, what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, "%s: %s shape %s, want %s" % (label, what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    if len(bad):
        ix = tuple(bad[0])
        raise AssertionError("%s: %s differs in %d of %d, first at %s: got %s want %s" % (
            label, what, len(bad), got.size, ix, got[ix], want[ix]))


def check(rc, where):
    from pire_b200 import _native as N
    N.check(rc, where)


# --------------------------------------------------------------------------------------------------------- inputs

def strings_for(d, rng, lengths):
    """Random strings for automaton d.  The absorbing families draw mostly from the class that walks their chain, so
    that the absorbing row is reached early in some strings and late in others."""
    out = []
    chain_bytes = np.nonzero(d.cls == 0)[0].astype(np.uint8)
    for k in lengths:
        k = int(k)
        if d.name.startswith("absorb"):
            s = rng.choice(chain_bytes, size=k)
            flip = rng.random(k) < 0.002
            s[flip] = rng.integers(0, 256, int(flip.sum()))
        else:
            s = rng.integers(0, 256, k, dtype=np.uint8)
        out.append(s.astype(np.uint8).tobytes())
    return out


class Batch:
    """A batch on the device: fixed-length (``fixed_len``) at a 32-byte aligned corpus, or CSR at byte ``base`` of its
    buffer (unaligned when base is odd)."""

    def __init__(self, strings, fixed=False, base=0):
        self.strings = strings
        self.n = len(strings)
        if fixed:
            self.fixed_len = len(strings[0]) if strings else 0
            assert all(len(s) == self.fixed_len for s in strings)
            self.offsets = None
            buf = b"".join(strings) + bytes(64)
        else:
            self.fixed_len = 0
            corpus, offs = refpire.csr(strings)
            self.offsets = offs
            buf = bytes(base) + corpus.tobytes()
        self.base = base
        self.buf = _dev(np.frombuffer(buf, np.uint8).copy())
        self.doffs = None if self.offsets is None else _dev(self.offsets.astype(np.int64))

    @property
    def corpus(self):
        return self.buf.data_ptr() + self.base

    @property
    def offs(self):
        return None if self.doffs is None else self.doffs.data_ptr()


def uniform_batches(d, seed):
    rng = np.random.default_rng(seed)
    return [Batch(strings_for(d, rng, [ln] * n), fixed=True) for ln, n in ((32, 200), (64, 97), (1024, 40))]


def ragged_batch(d, seed, long=False):
    rng = np.random.default_rng(seed)
    lens = [0, 0, 1, 0] + list(rng.integers(0, 90, 200)) + [0, 15, 16, 17, 33]
    if long:
        lens += [8192, 9001, 12345]
    return Batch(strings_for(d, rng, lens), base=3)


_HANDLES = {}


def handle(name):
    import pire_b200 as P
    if name not in _HANDLES:
        _HANDLES[name] = P.Scanner(SD.family(name).image(), 0)
    return _HANDLES[name]


# ------------------------------------------------------------------------------------------------------- run family

def run_batch(sc, d, b, begin, end, label, starts=None, ordered=False):
    """pire_gpu_run_batch / _ordered / _from against the walker."""
    import torch
    from pire_b200 import _native as N
    n = b.n
    bits, masks, states = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
    order = None
    if ordered:
        order = torch.empty(n, dtype=torch.int32, device="cuda:0")
        check(N.lib.pire_gpu_length_order(b.offs, n, order.data_ptr(), 0, _stream()), "length_order")
    if starts is not None:
        dstart = _dev(np.asarray(starts, np.uint32).view(np.int32))
        check(N.lib.pire_gpu_run_batch_from(sc._h, b.corpus, b.offs, None if order is None else order.data_ptr(), b.fixed_len, n,
                                            _flags(begin, end), dstart.data_ptr(), bits.data_ptr(), masks.data_ptr(),
                                            states.data_ptr(), _stream()), label)
    elif ordered:
        check(N.lib.pire_gpu_run_batch_ordered(sc._h, b.corpus, b.offs, order.data_ptr(), n, _flags(begin, end), bits.data_ptr(),
                                               masks.data_ptr(), states.data_ptr(), _stream()), label)
    else:
        check(N.lib.pire_gpu_run_batch(sc._h, b.corpus, b.offs, b.fixed_len, n, _flags(begin, end), bits.data_ptr(),
                                       masks.data_ptr(), states.data_ptr(), _stream()), label)
    fin, mask, state = d.run(b.strings, starts, begin, end)
    expect(label, "StateIndex", _host(states, n, label, "states"), state)
    expect(label, "accept masks", _host(masks, n, label, "masks"), mask)
    expect(label, "match bits", _bits(bits, n, label), fin)
    return state


@pytest.mark.parametrize("variant", range(8))
@pytest.mark.parametrize("name", RUN_FAMILIES + ["count_r16_x15", "count_abs16_x15"])
def test_run_batch(name, variant, cuda_device):
    """run_batch with variant 0-7 on uniform batches of 32, 64 and 1024 bytes and on a ragged CSR batch with empty
    strings at an unaligned corpus, under all four mark combinations; the CSR batch also length-ordered."""
    d, sc = SD.family(name), handle(name)
    sc.set_variant(variant)
    try:
        batches = uniform_batches(d, 1) + [ragged_batch(d, 2, long=variant == 0)]
        for begin, end in MARKS:
            for k, b in enumerate(batches):
                label = "%s variant=%d batch=%d begin=%d end=%d" % (name, variant, k, begin, end)
                run_batch(sc, d, b, begin, end, label)
                if b.offsets is not None and variant in (0, 1):
                    run_batch(sc, d, b, begin, end, label + " ordered", ordered=True)
    finally:
        sc.set_variant(0)


HOT_SETTINGS = ("max_hot_1", "max_hot_2", "max_hot_255", "tuned", "autoselect")


@pytest.mark.parametrize("setting", HOT_SETTINGS)
@pytest.mark.parametrize("name", ["uniform_L200", "hot_256", "priv_116", "look_cold", "width_65536", "marks", "shift_33"])
def test_run_batch_hot_sets(name, setting, cuda_device):
    """Handles with one, two and 255 hot rows, and after Tune and AutoSelect, every variant."""
    import pire_b200 as P
    d = SD.family(name)
    sc = P.Scanner(d.image(), 0)
    batches = uniform_batches(d, 3)[:2] + [ragged_batch(d, 4)]
    if setting.startswith("max_hot"):
        sc.set_max_hot(int(setting.split("_")[-1]))
    else:
        b = batches[1]
        pb = P.Batch(b.buf[: b.n * b.fixed_len], fixed_len=b.fixed_len, n=b.n)
        sc.Tune(pb) if setting == "tuned" else sc.AutoSelect(pb)
    for variant in range(8):
        if setting == "autoselect" and variant:
            break                                                # AUTO's recorded choice
        sc.set_variant(variant)
        for begin, end in ((True, True), (False, False)):
            for k, b in enumerate(batches):
                run_batch(sc, d, b, begin, end, "%s %s variant=%d batch=%d begin=%d end=%d" % (name, setting, variant, k, begin, end))


@pytest.mark.parametrize("name", ["uniform_L2", "hot_255", "look_cold", "width_65537", "marks", "perm_5", "absorb_late"])
def test_run_batch_from_chained(name, cuda_device):
    """run_batch_from with random starts, some >= Size(), and three rounds chained through the state array."""
    d, sc = SD.family(name), handle(name)
    rng = np.random.default_rng(5)
    for k, b in enumerate(uniform_batches(d, 6)[:2] + [ragged_batch(d, 7)]):
        starts = rng.integers(0, d.states, b.n).astype(np.uint32)
        starts[::7] = d.states + rng.integers(0, 3, len(starts[::7]))
        starts[1::11] = SD.UNKNOWN
        st = starts
        for rnd, (begin, end) in enumerate(((True, False), (False, False), (False, True))):
            st = run_batch(sc, d, b, begin, end, "%s from batch=%d round=%d" % (name, k, rnd), starts=st)


PAIRS = [("width_65537", "hot_255"), ("look_cold", "priv_116"), ("marks", "marks")]


@pytest.mark.parametrize("pair", PAIRS, ids=["%s+%s" % p for p in PAIRS])
def test_run_pair_batch(pair, cuda_device):
    """Two synthesized scanners with different hot sets over one batch, uniform and CSR, with and without starts."""
    from pire_b200 import _native as N
    (n1, n2) = pair
    d1, d2 = SD.family(n1), SD.family(n2)
    s1, s2 = handle(n1), handle(n2)
    rng = np.random.default_rng(8)
    for k, b in enumerate(uniform_batches(d1, 9) + [ragged_batch(d1, 10)]):
        for begin, end in MARKS:
            starts2 = rng.integers(0, d2.states + 2, b.n).astype(np.uint32)
            ds2 = _dev(starts2.view(np.int32))
            outs = [_filled((b.n + 31) // 32 + 1), _filled(b.n + EXTRA), _filled(b.n + EXTRA)]
            outs2 = [_filled((b.n + 31) // 32 + 1), _filled(b.n + EXTRA), _filled(b.n + EXTRA)]
            label = "pair %s+%s batch=%d begin=%d end=%d" % (n1, n2, k, begin, end)
            check(N.lib.pire_gpu_run_pair_batch(s1._h, s2._h, b.corpus, b.offs, b.fixed_len, b.n, _flags(begin, end), None,
                                                ds2.data_ptr(), *[t.data_ptr() for t in outs], *[t.data_ptr() for t in outs2],
                                                _stream()), label)
            for d, o, st, half in ((d1, outs, None, 1), (d2, outs2, starts2, 2)):
                fin, mask, state = d.run(b.strings, st, begin, end)
                lab = "%s half %d" % (label, half)
                expect(lab, "match bits", _bits(o[0], b.n, lab), fin)
                expect(lab, "masks", _host(o[1], b.n, lab, "masks"), mask)
                expect(lab, "states", _host(o[2], b.n, lab, "states"), state)


# ---------------------------------------------------------------------------------------------- one long string

def _text(d, seed, n):
    return strings_for(d, np.random.default_rng(seed), [n])[0]


def run_string_check(sc, d, text, begin, end, label, start=None, orc=None):
    """pire_gpu_run_string on text (optionally in chunks chained through the state word) against the walker, or
    against the C oracle for strings too long for it."""
    from pire_b200 import _native as N
    dtext = _dev(np.frombuffer(text + bytes(16), np.uint8).copy())
    bits, masks, state = _filled(1 + EXTRA), _filled(1 + EXTRA), _filled(1 + EXTRA)
    dstart = None if start is None else _dev(np.array([start], np.uint32).view(np.int32))
    check(N.lib.pire_gpu_run_string(sc._h, dtext.data_ptr() if text else None, len(text), _flags(begin, end),
                                    None if dstart is None else dstart.data_ptr(), bits.data_ptr(), masks.data_ptr(),
                                    state.data_ptr(), _stream()), label)
    if orc is not None:
        assert start is None
        corpus, offs = refpire.csr([text])
        fin, mask, st = orc.run(corpus, offs, begin=begin, end=end)
    else:
        fin, mask, st = d.run([text], None if start is None else [start], begin, end)
    expect(label, "state", _host(state, 1, label, "state"), st)
    expect(label, "mask", _host(masks, 1, label, "mask"), mask)
    expect(label, "match word", _host(bits, 1, label, "match"), fin.astype(np.uint32))


STRING_FAMILIES = {
    # name: longest text (bytes) walked on the GPU
    "shift_16": 64 << 20, "shift_33": 4 << 20, "shift_64": 16 << 20, "perm_5": 1 << 20, "uniform_L2": 4 << 20,
    "width_65537": 4 << 20, "marks": 1 << 20, "absorb_late": 4 << 20, "look_cold": 1 << 20,
}


@pytest.mark.parametrize("name", sorted(STRING_FAMILIES))
def test_run_string(name, cuda_device):
    """run_string: empty text, a few bytes, about one, two and three pieces of a persistent grid, up to the family's
    longest text; chunks chained through the state word; every start state of small automata."""
    d, sc = SD.family(name), handle(name)
    orc = refpire.Oracle(d.image())
    longest = STRING_FAMILIES[name]
    sizes = [0, 1, 2, 3, 31, 4096, 65537, 300001, longest]
    for n in sizes:
        text = _text(d, n, n)
        for begin, end in MARKS:
            run_string_check(sc, d, text, begin, end, "%s run_string n=%d begin=%d end=%d" % (name, n, begin, end),
                             orc=orc if n > (1 << 20) else None)
    text = _text(d, 99, min(longest, 3 << 20))
    cuts = [0, 1, len(text) // 3, len(text) // 3 + 17, len(text)]
    st = None
    for k in range(len(cuts) - 1):
        chunk = text[cuts[k]:cuts[k + 1]]
        run_string_check(sc, d, chunk, k == 0, k == len(cuts) - 2, "%s chained chunk %d" % (name, k), start=st)
        st = int(d.run([chunk], None if st is None else [st], k == 0, k == len(cuts) - 2)[2][0])
    if d.states <= 64:
        text = _text(d, 5, 200000)
        for s in list(range(d.states)) + [d.states, SD.UNKNOWN]:
            run_string_check(sc, d, text, False, True, "%s start=%d" % (name, s), start=s)


# ---------------------------------------------------------------------------------------------- prefix and suffix

@pytest.mark.parametrize("name", RUN_FAMILIES)
def test_prefix_suffix(name, cuda_device):
    """Longest and Shortest Prefix and Suffix with every flag, on uniform and CSR batches."""
    from pire_b200 import _native as N
    d, sc = SD.family(name), handle(name)
    for k, b in enumerate(uniform_batches(d, 11)[:2] + [ragged_batch(d, 12)]):
        for tb, te in MARKS:
            for shortest in (False, True):
                for suffix in (False, True):
                    out = _filled(b.n + EXTRA)
                    fn = N.lib.pire_gpu_suffix_batch if suffix else N.lib.pire_gpu_prefix_batch
                    label = "%s %s%s batch=%d begin=%d end=%d" % (name, "Shortest" if shortest else "Longest",
                                                                  "Suffix" if suffix else "Prefix", k, tb, te)
                    check(fn(sc._h, b.corpus, b.offs, b.fixed_len, b.n, _flags(tb, te), int(shortest), out.data_ptr(), _stream()),
                          label)
                    got = _host(out, b.n, label, "lengths").astype(np.int64)
                    got[got == NO_PREFIX] = -1
                    want = d.suffix(b.strings, shortest, te, tb) if suffix else d.prefix(b.strings, shortest, tb, te)
                    expect(label, "length", got, want)


# ---------------------------------------------------------------------------------------------------------- counting

def count_batches(d, seed):
    rng = np.random.default_rng(seed)
    return [Batch(strings_for(d, rng, [32] * 70), fixed=True), Batch(strings_for(d, rng, [1024] * 9), fixed=True),
            Batch(strings_for(d, rng, [0, 1, 2, 15, 16, 17, 18, 31, 33] + list(rng.integers(0, 70, 150))), base=5),
            Batch(strings_for(d, rng, list(rng.integers(1, 16, 200))), base=1)]


@pytest.mark.parametrize("mode", range(4))
@pytest.mark.parametrize("name", COUNT_FAMILIES)
def test_count_batch(name, mode, cuda_device):
    """count_batch in modes AUTO, LISTS, PACKED and EVERY_CHUNK, uniform and unaligned CSR batches whose heads and tails
    are 1 to 15 bytes, every mark combination."""
    from pire_b200 import _native as N
    d, sc = SD.family(name), handle(name)
    regs = max(1, d.regexps)
    sc.set_count_mode(mode)
    try:
        for k, b in enumerate(count_batches(d, 13)):
            for begin, end in MARKS:
                label = "%s mode=%d batch=%d begin=%d end=%d" % (name, mode, k, begin, end)
                counts, bits = _filled((b.n + EXTRA) * regs), _filled((b.n + 31) // 32 + 1)
                check(N.lib.pire_gpu_count_batch(sc._h, b.corpus, b.offs, b.fixed_len, b.n, _flags(begin, end), counts.data_ptr(),
                                                 bits.data_ptr(), _stream()), label)
                wc, wf, _ = d.count(b.strings, None, begin, end)
                expect(label, "counts", _host(counts, b.n * regs, label, "counts").reshape(b.n, regs), wc)
                expect(label, "final bits", _bits(bits, b.n, label), wf)
    finally:
        sc.set_count_mode(0)


@pytest.mark.parametrize("mode", (0, 1, 2))
@pytest.mark.parametrize("name", ["count_r8_x15", "count_r16_x15", "count_r16_x16", "count_abs16_x15", "count_r257", "marks"])
def test_count_chained(name, mode, cuda_device):
    """count_batch_from over three rounds chained in place, and count_string (u64) over chained chunks."""
    from pire_b200 import _native as N
    d, sc = SD.family(name), handle(name)
    regs = max(1, d.regexps)
    sc.set_count_mode(mode)
    try:
        rng = np.random.default_rng(14)
        n = 150
        rounds = [strings_for(d, rng, rng.integers(0, 40, n)) for _ in range(3)]
        counts = _filled((n + EXTRA) * regs, wide=True)
        counts[: n * regs] = 0
        states, bits = _filled(n + EXTRA), _filled((n + 31) // 32 + 1)
        want = np.zeros((n, regs), np.int64)
        st = None
        for r, strings in enumerate(rounds):
            b = Batch(strings, base=r)
            begin, end = r == 0, r == 2
            label = "%s mode=%d count_batch_from round=%d" % (name, mode, r)
            check(N.lib.pire_gpu_count_batch_from(sc._h, b.corpus, b.offs, 0, n, _flags(begin, end),
                                                  None if r == 0 else states.data_ptr(), counts.data_ptr(), bits.data_ptr(),
                                                  states.data_ptr(), _stream()), label)
            wc, wf, st = d.count(strings, st, begin, end)
            want += wc
            expect(label, "counts", _host(counts, n * regs, label, "counts").reshape(n, regs).astype(np.int64), want)
            expect(label, "final bits", _bits(bits, n, label), wf)
            expect(label, "states", _host(states, n, label, "states"), st)
        text = _text(d, 15, 1 << 20)
        cuts = [0, 7, 4096 + 3, 500001, len(text)]
        counts = _filled(regs + EXTRA, wide=True)
        counts[:regs] = 0
        state, bits = _filled(1 + EXTRA), _filled(1 + EXTRA)
        want = np.zeros(regs, np.int64)
        st = None
        for k in range(len(cuts) - 1):
            chunk = text[cuts[k]:cuts[k + 1]]
            begin, end = k == 0, k == len(cuts) - 2
            dtext = _dev(np.frombuffer(chunk, np.uint8).copy())
            label = "%s mode=%d count_string chunk=%d" % (name, mode, k)
            check(N.lib.pire_gpu_count_string(sc._h, dtext.data_ptr(), len(chunk), _flags(begin, end),
                                              None if k == 0 else state.data_ptr(), counts.data_ptr(), bits.data_ptr(),
                                              state.data_ptr(), _stream()), label)
            wc, wf, st = d.count([chunk], st, begin, end)
            want += wc[0]
            expect(label, "counts", _host(counts, regs, label, "counts").astype(np.int64), want)
            expect(label, "state", _host(state, 1, label, "state"), st)
            expect(label, "match word", _host(bits, 1, label, "match"), wf.astype(np.uint32))
    finally:
        sc.set_count_mode(0)


# -------------------------------------------------------------------------------------------------------- match ends

ENDS_FAMILIES = ["count_r8_x15", "count_r16_x16", "count_abs16_x15", "count_r33", "marks", "absorb_early", "hot_255",
                 "width_65537", "uniform_p1"]


@pytest.mark.parametrize("name", ENDS_FAMILIES)
def test_match_ends(name, cuda_device):
    """match_ends_string (chained chunks), match_ends_batch_from (chained rounds) and match_ends_lines, each with an
    exact capacity and a short one."""
    from pire_b200 import _native as N
    d, sc = SD.family(name), handle(name)
    rng = np.random.default_rng(16)
    # one string in chunks
    text = _text(d, 17, 200000)
    cuts = [0, 5, 70001, len(text)]
    st, wends, wids = None, [], []
    for k in range(len(cuts) - 1):
        chunk = text[cuts[k]:cuts[k + 1]]
        _, e, i, _, s = d.match_ends([chunk], st, k == 0, k == len(cuts) - 2, bases=[cuts[k]])
        wends.append(e), wids.append(i)
        st = s
    wends, wids = np.concatenate(wends), np.concatenate(wids)
    total = len(wends)
    for cap in (total, max(0, total - 37)):
        ends, ids, found = _filled(cap + EXTRA, wide=True), _filled(cap + EXTRA), _filled(1 + EXTRA, wide=True)
        found[0] = 0
        state = _filled(1 + EXTRA)
        for k in range(len(cuts) - 1):
            chunk = text[cuts[k]:cuts[k + 1]]
            dtext = _dev(np.frombuffer(chunk, np.uint8).copy())
            check(N.lib.pire_gpu_match_ends_string(sc._h, dtext.data_ptr(), len(chunk), _flags(k == 0, k == len(cuts) - 2),
                                                   None if k == 0 else state.data_ptr(), cuts[k], ends.data_ptr(), ids.data_ptr(),
                                                   cap, found.data_ptr(), None, state.data_ptr(), _stream()), "match_ends_string")
        label = "%s match_ends_string cap=%d" % (name, cap)
        expect(label, "found", _host(found, 1, label, "found"), [total])
        expect(label, "ends", _host(ends, cap, label, "ends"), wends[:cap])
        expect(label, "ids", _host(ids, cap, label, "ids"), wids[:cap])
    # a batch of streams over two rounds
    n = 120
    rounds = [strings_for(d, rng, rng.integers(0, 50, n)) for _ in range(2)]
    st, pos = None, np.zeros(n, np.int64)
    wparts = []
    for r, strings in enumerate(rounds):
        s_, e_, i_, f_, st_new = d.match_ends(strings, st, r == 0, r == 1, bases=pos)
        wparts.append((s_, e_, i_))
        st = st_new
        pos = pos + np.array([len(x) for x in strings])
    ws = np.concatenate([p[0] for p in wparts])
    we = np.concatenate([p[1] for p in wparts])
    wi = np.concatenate([p[2] for p in wparts])
    total = len(ws)
    for cap in (total, total // 2):
        strs, ends, ids = _filled(cap + EXTRA), _filled(cap + EXTRA, wide=True), _filled(cap + EXTRA)
        found, dpos = _filled(1 + EXTRA, wide=True), _filled(n + EXTRA, wide=True)
        found[0] = 0
        dpos[:n] = 0
        states = _filled(n + EXTRA)
        for r, strings in enumerate(rounds):
            b = Batch(strings, base=r + 1)
            check(N.lib.pire_gpu_match_ends_batch_from(sc._h, b.corpus, b.offs, 0, n, _flags(r == 0, r == 1),
                                                       None if r == 0 else states.data_ptr(), dpos.data_ptr(), strs.data_ptr(),
                                                       ends.data_ptr(), ids.data_ptr(), cap, found.data_ptr(), None,
                                                       states.data_ptr(), _stream()), "match_ends_batch_from")
        label = "%s match_ends_batch_from cap=%d" % (name, cap)
        expect(label, "found", _host(found, 1, label, "found"), [total])
        expect(label, "strings", _host(strs, cap, label, "strings"), ws[:cap])
        expect(label, "ends", _host(ends, cap, label, "ends"), we[:cap])
        expect(label, "ids", _host(ids, cap, label, "ids"), wi[:cap])
        expect(label, "positions", _host(dpos, n, label, "positions"), pos.astype(np.uint64))
        expect(label, "states", _host(states, n, label, "states"), st)


# ------------------------------------------------------------------------------------------------------------- lines

def split_text(text):
    """(offsets, lines) with std::getline semantics: line i is text[off[i], off[i+1] - 1)."""
    lines = text.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    offs = [0]
    for ln in lines:
        offs.append(offs[-1] + len(ln) + 1)
    return np.array(offs, np.uint64), lines


@pytest.mark.parametrize("name", ["lines", "count_r16_x15"])
def test_lines(name, cuda_device):
    """split_lines, run_lines and match_ends_lines on texts where '\\n' has a class of its own (or shares one)."""
    import torch
    from pire_b200 import _native as N
    d, sc = SD.family(name), handle(name)
    rng = np.random.default_rng(18)
    nl = np.frombuffer(b"\n", np.uint8)
    for k, n_lines in enumerate((0, 1, 300, 3000)):
        parts = []
        for _ in range(n_lines):
            ln = int(rng.choice([0, 0, 1, 5, 15, 16, 17, 31, 33, 64, 100, 700]))
            s = strings_for(d, rng, [ln])[0].replace(b"\n", b" ")
            parts.append(s)
        text = b"\n".join(parts) + (b"\n" if k % 2 else b"")
        offs, lines = split_text(text)
        n = len(lines)
        dtext = _dev(np.frombuffer(text + bytes(32), np.uint8).copy())
        doffs = _dev(np.full(n + 1 + EXTRA, SENTINEL64, np.uint64).view(np.int64))
        cnt = ctypes.c_uint64(0)
        check(N.lib.pire_gpu_split_lines(dtext.data_ptr(), len(text), doffs.data_ptr(), n + 1 + EXTRA - 1,
                                         ctypes.byref(cnt), 0, _stream()), "split_lines")
        label = "%s lines text=%d" % (name, k)
        assert cnt.value == n, (label, cnt.value, n)
        if n == 0:                                               # no lines: nothing to frame
            continue
        expect(label, "offsets", _host(doffs, n + 1, label, "offsets"), offs)
        for begin, end in MARKS:
            lab = "%s begin=%d end=%d" % (label, begin, end)
            bits, masks, states = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
            check(N.lib.pire_gpu_run_lines(sc._h, dtext.data_ptr(), doffs.data_ptr(), None, n, _flags(begin, end), bits.data_ptr(),
                                           masks.data_ptr(), states.data_ptr(), _stream()), lab)
            fin, mask, state = d.run(lines, None, begin, end)
            expect(lab, "states", _host(states, n, lab, "states"), state)
            expect(lab, "masks", _host(masks, n, lab, "masks"), mask)
            expect(lab, "bits", _bits(bits, n, lab), fin)
            ws, we, wi, _, _ = d.match_ends(lines, None, begin, end, bases=offs[:-1].astype(np.int64))
            total = len(ws)
            for cap in (total, total // 3):
                lns, ends, ids = _filled(cap + EXTRA), _filled(cap + EXTRA, wide=True), _filled(cap + EXTRA)
                found = torch.zeros(1 + EXTRA, dtype=torch.int64, device="cuda:0")
                found[1:] = SENTINEL64
                check(N.lib.pire_gpu_match_ends_lines(sc._h, dtext.data_ptr(), doffs.data_ptr(), n, _flags(begin, end),
                                                      lns.data_ptr(), ends.data_ptr(), ids.data_ptr(), cap, found.data_ptr(), None,
                                                      None, _stream()), lab)
                l2 = "%s match_ends_lines cap=%d" % (lab, cap)
                expect(l2, "found", _host(found, 1, l2, "found"), [total])
                expect(l2, "lines", _host(lns, cap, l2, "lines"), ws[:cap])
                expect(l2, "ends", _host(ends, cap, l2, "ends"), we[:cap])
                expect(l2, "ids", _host(ids, cap, l2, "ids"), wi[:cap])


# ------------------------------------------------------------------------------------------------------ match starts

STARTS_PAIRS = [("marks", "marks"), ("count_r8_x15", "count_r9"), ("hot_255", "uniform_L2")]


def _starts_check(label, rd, text, wlo, whi, ends, ids, begin, end, max_back, starts, opened, n_entries):
    ws, wo = rd.match_starts(text, wlo, whi, ends, ids, begin, end, max_back)
    expect(label, "starts", _host(starts, n_entries, label, "starts"), ws)
    got_open = opened.cpu().numpy()
    assert (got_open[n_entries:] == 0xA5).all(), "%s: open flags written past their end" % label
    expect(label, "open", got_open[:n_entries], wo)


def _open_buf(count):
    import torch
    return torch.full((count,), 0xA5, dtype=torch.uint8, device="cuda:0")


@pytest.mark.parametrize("pair", STARTS_PAIRS, ids=["%s-%s" % p for p in STARTS_PAIRS])
def test_match_starts(pair, cuda_device):
    """match_starts_string, _batch and _lines with a second synthesized scanner as the reversed one, fed the entries
    match ends wrote: with and without ids, max_back 0, 3 and 40, every mark combination."""
    import torch
    from pire_b200 import _native as N
    fwd, rev = pair
    d, sc = SD.family(fwd), handle(fwd)
    rd, rsc = SD.family(rev), handle(rev)
    cap = 300
    rng = np.random.default_rng(19)
    text = _text(d, 20, 3000)
    dtext = _dev(np.frombuffer(text + bytes(16), np.uint8).copy())
    strings = strings_for(d, rng, rng.integers(0, 60, 40))
    b = Batch(strings, base=7)
    ltext = b"\n".join(s.replace(b"\n", b" ") for s in strings) + b"\n"
    loffs, lines = split_text(ltext)
    dl = _dev(np.frombuffer(ltext + bytes(16), np.uint8).copy())
    dloffs = _dev(loffs.astype(np.int64))
    for begin, end in MARKS:
        fl = _flags(begin, end)
        # one string
        ends, ids, found = _filled(cap, wide=True), _filled(cap), torch.zeros(1, dtype=torch.int64, device="cuda:0")
        check(N.lib.pire_gpu_match_ends_string(sc._h, dtext.data_ptr(), len(text), fl, None, 0, ends.data_ptr(), ids.data_ptr(), cap,
                                               found.data_ptr(), None, None, _stream()), "match_ends_string")
        m = min(int(found.item()), cap)
        he, hi = ends.cpu().numpy().view(np.uint64)[:m], ids.cpu().numpy().view(np.uint32)[:m]
        for max_back in (0, 3, 40):
            for with_ids in (True, False):
                starts, opened = _filled(m + EXTRA, wide=True), _open_buf(m + EXTRA)
                label = "%s/%s string begin=%d end=%d max_back=%d ids=%d" % (fwd, rev, begin, end, max_back, with_ids)
                check(N.lib.pire_gpu_match_starts_string(rsc._h, dtext.data_ptr(), len(text), 0, fl, max_back, ends.data_ptr(),
                                                         ids.data_ptr() if with_ids else None, None, found.data_ptr(), cap,
                                                         starts.data_ptr(), opened.data_ptr(), _stream()), label)
                _starts_check(label, rd, text, 0, len(text), he, hi if with_ids else None, begin, end, max_back, starts, opened, m)
        # a batch: each entry's window is its own string, ends offsets within it
        strs, ends, ids = _filled(cap), _filled(cap, wide=True), _filled(cap)
        found, pos = torch.zeros(1, dtype=torch.int64, device="cuda:0"), torch.zeros(b.n, dtype=torch.int64, device="cuda:0")
        check(N.lib.pire_gpu_match_ends_batch_from(sc._h, b.corpus, b.offs, 0, b.n, fl, None, pos.data_ptr(), strs.data_ptr(),
                                                   ends.data_ptr(), ids.data_ptr(), cap, found.data_ptr(), None, None, _stream()),
              "match_ends_batch_from")
        m = min(int(found.item()), cap)
        hs = strs.cpu().numpy().view(np.uint32)[:m]
        he, hi = ends.cpu().numpy().view(np.uint64)[:m], ids.cpu().numpy().view(np.uint32)[:m]
        for max_back in (0, 3):
            starts, opened = _filled(m + EXTRA, wide=True), _open_buf(m + EXTRA)
            label = "%s/%s batch begin=%d end=%d max_back=%d" % (fwd, rev, begin, end, max_back)
            check(N.lib.pire_gpu_match_starts_batch(rsc._h, b.corpus, b.offs, 0, b.n, pos.data_ptr(), fl, max_back, strs.data_ptr(),
                                                    ends.data_ptr(), ids.data_ptr(), None, found.data_ptr(), cap, starts.data_ptr(),
                                                    opened.data_ptr(), _stream()), label)
            ws = np.zeros(m, np.uint64)
            wo = np.zeros(m, np.uint8)
            for k in range(m):
                s = strings[hs[k]]
                a, o = rd.match_starts(s, 0, len(s), he[k:k + 1], hi[k:k + 1], begin, end, max_back)
                ws[k], wo[k] = a[0], o[0]
            expect(label, "starts", _host(starts, m, label, "starts"), ws)
            expect(label, "open", opened.cpu().numpy()[:m], wo)
            assert (opened.cpu().numpy()[m:] == 0xA5).all(), label
        # the lines of a text
        lns, ends, ids = _filled(cap), _filled(cap, wide=True), _filled(cap)
        found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
        check(N.lib.pire_gpu_match_ends_lines(sc._h, dl.data_ptr(), dloffs.data_ptr(), len(lines), fl, lns.data_ptr(), ends.data_ptr(),
                                              ids.data_ptr(), cap, found.data_ptr(), None, None, _stream()), "match_ends_lines")
        m = min(int(found.item()), cap)
        hl = lns.cpu().numpy().view(np.uint32)[:m]
        he, hi = ends.cpu().numpy().view(np.uint64)[:m], ids.cpu().numpy().view(np.uint32)[:m]
        starts, opened = _filled(m + EXTRA, wide=True), _open_buf(m + EXTRA)
        label = "%s/%s lines begin=%d end=%d" % (fwd, rev, begin, end)
        check(N.lib.pire_gpu_match_starts_lines(rsc._h, dl.data_ptr(), dloffs.data_ptr(), len(lines), fl, 0, lns.data_ptr(),
                                                ends.data_ptr(), ids.data_ptr(), None, found.data_ptr(), cap, starts.data_ptr(),
                                                opened.data_ptr(), _stream()), label)
        ws = np.zeros(m, np.uint64)
        wo = np.zeros(m, np.uint8)
        for k in range(m):
            lo_, hi_ = int(loffs[hl[k]]), int(loffs[hl[k] + 1]) - 1
            a, o = rd.match_starts(ltext, lo_, hi_, he[k:k + 1], hi[k:k + 1], begin, end, 0)
            ws[k], wo[k] = a[0], o[0]
        expect(label, "starts", _host(starts, m, label, "starts"), ws)
        expect(label, "open", opened.cpu().numpy()[:m], wo)
