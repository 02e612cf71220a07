"""The launch paths off the default shapes, against the in-repo oracle (oracle/pire_oracle.c, the plain byte-by-byte
walk): start states outside the hot rows, hot sets of one to three rows, 32-bit transition tables, fixed-length
batches that are not uniform (length not a multiple of 32, base not 32-byte aligned), writes past the last string,
and strings past the 4 GiB mark.

Every group first asserts the precondition that puts it on its path, so that a change to the hot order or to the
dispatch cannot quietly move it off.  Every output buffer is larger than the batch and pre-filled with a sentinel:
whatever lies past the last valid entry must still hold it afterwards."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from refpire import Oracle, csr, oracle_count, oracle_prefix, oracle_suffix  # noqa: E402
from test_edge_images import ALPHABETS, EDGE  # noqa: E402

pytestmark = pytest.mark.gpu

BeginMark, EndMark = 258, 259
RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
SENTINEL = 0x5A5A5A5A
EXTRA = 64                       # entries past n in every output (and one more bitmap word)
MARKS = ((True, True), (False, False), (True, False), (False, True))
_SERIAL = itertools.count()


def kernels_launched(fn):
    """The names of the kernels that ``fn`` launches, space-separated, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events())


def is_uniform(corpus_ptr, offsets_ptr, fixed_len):
    """capi.cu IsUniform: the batches the uniform kernels take."""
    return offsets_ptr is None and fixed_len != 0 and fixed_len % 32 == 0 and corpus_ptr % 32 == 0


# ----------------------------------------------------------------------------------------------------- host batches

class HostBatch:
    """The bytes of one batch as the device holds them: ``buf`` is the whole device buffer (guard bytes included), the
    batch's corpus starts at ``base``; CSR ``offsets`` (relative to the corpus) or ``fixed_len``.  ``lines`` marks a
    batch of text lines (the newline ending a line is not part of it)."""

    def __init__(self, buf, base=0, offsets=None, fixed_len=0, n=None, lines=False):
        self.buf = np.ascontiguousarray(buf, dtype=np.uint8)
        self.base, self.fixed_len, self.lines = int(base), int(fixed_len), lines
        self.offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
        if self.offsets is not None:
            self.n = len(self.offsets) - 1 if n is None else int(n)
        else:
            self.n = int(n)
        self._dev = None
        self.serial = next(_SERIAL)             # the oracle's answers are cached under it

    def corpus(self):
        return self.buf[self.base:]

    def oracle_args(self):
        """(corpus, offsets, fixed_len) of the strings as the oracle sees them."""
        if not self.lines:
            return self.corpus(), self.offsets, self.fixed_len
        b = self.offsets[:-1]
        e = np.maximum(self.offsets[1:].astype(np.int64) - 1, b.astype(np.int64)).astype(np.uint64)
        strings = [bytes(self.corpus()[int(x):int(y)]) for x, y in zip(b, e)]
        corpus, offs = csr(strings)
        return corpus, offs, 0

    def device(self):
        import torch
        if self._dev is None:
            d = torch.from_numpy(self.buf.copy()).to("cuda:0")
            offs = None if self.offsets is None else torch.from_numpy(self.offsets.astype(np.int64)).to("cuda:0")
            self._dev = (d, offs)
        return self._dev

    def corpus_ptr(self):
        return self.device()[0].data_ptr() + self.base

    def offsets_ptr(self):
        offs = self.device()[1]
        return None if offs is None else offs.data_ptr()

    def order(self):
        import torch
        from pire_b200 import _native as N
        offs = self.device()[1]
        order = torch.empty(self.n, dtype=torch.int32, device="cuda:0")
        N.check(N.lib.pire_gpu_length_order(offs.data_ptr(), self.n, order.data_ptr(), 0, _stream()), "pire_gpu_length_order")
        return order


def _stream():
    import torch
    return torch.cuda.current_stream(0).cuda_stream


def fixed_batch(rows, base=0, guard_before=b"", guard_after=b""):
    """n strings of one length (the rows of a 2-D uint8 array) at ``base`` of a buffer whose bytes before ``base`` and
    after the last string are guard bytes (repeated)."""
    n, length = rows.shape
    before = (guard_before * (base + 1))[:base] if guard_before else bytes(base)
    after = (guard_after * 64)[:64] if guard_after else bytes(64)
    buf = np.frombuffer(before + np.ascontiguousarray(rows).tobytes() + after, np.uint8).copy()
    return HostBatch(buf, base=base, fixed_len=length, n=n)


def csr_batch(strings):
    corpus, offs = csr(strings)
    return HostBatch(corpus, offsets=offs)


def lines_batch(text):
    """A text's lines, split on the device (std::getline semantics)."""
    import pire_b200 as P
    import torch
    dev = torch.from_numpy(np.frombuffer(text + bytes(32), np.uint8).copy()).to("cuda:0")
    b = P.Batch.from_text(dev[: len(text)])
    hb = HostBatch(np.frombuffer(text + bytes(32), np.uint8), offsets=b.offsets.cpu().numpy().astype(np.uint64), lines=True)
    hb._dev = (dev, b.offsets)
    return hb


# -------------------------------------------------------------------------------------------------- the comparisons

def _first_diff(got, want, k=5):
    bad = np.argwhere(np.asarray(got) != np.asarray(want))[:k]
    return ", ".join("%s: got %s want %s" % (tuple(int(x) for x in ix), np.asarray(got)[tuple(ix)], np.asarray(want)[tuple(ix)])
                     for ix in bad)


def expect_equal(label, what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, "%s: %s has shape %s, want %s" % (label, what, got.shape, want.shape)
    if not (got == want).all():
        raise AssertionError("%s: %s differs (%d of %d) at %s" % (label, what, int((got != want).sum()), got.size,
                                                                  _first_diff(got, want)))


def _filled(count, value=SENTINEL):
    import torch
    v = value - (1 << 32) if value >= (1 << 31) else value
    return torch.full((count,), v, dtype=torch.int32, device="cuda:0")


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def expect_untouched(label, what, host, valid):
    tail = host[valid:]
    if not (tail == SENTINEL).all():
        k = int(np.nonzero(tail != SENTINEL)[0][0])
        raise AssertionError("%s: %s written past its last entry: [%d] = %#x" % (label, what, valid + k, int(tail[k])))


def unpack_bits(label, words, n):
    """Bits 0..n-1 of a bitmap; the words past (n + 31) / 32 still hold the sentinel, bits past n are zero."""
    nw = (n + 31) // 32
    expect_untouched(label, "match bitmap", words, nw)
    if n % 32:
        assert int(words[nw - 1]) >> (n % 32) == 0, "%s: match bits past n set: %#x" % (label, int(words[nw - 1]))
    return ((words[np.arange(n) // 32] >> (np.arange(n) % 32).astype(np.uint32)) & 1).astype(np.uint8)


class Checker:
    """One scanner (device handle + oracle); caches the oracle's answers per batch and mark combination."""

    def __init__(self, image, name, device_sc=None):
        import pire_b200 as P
        self.image, self.name = image, name
        self.sc = device_sc if device_sc is not None else P.Scanner(image, 0)
        self.orc = Oracle(image)
        self._want = {}

    def want(self, hb, op, *key):
        k = (hb.serial, op) + key
        if k not in self._want:
            corpus, offs, fl = hb.oracle_args()
            if op == "run":
                begin, end = key
                self._want[k] = self.orc.run(corpus, offs, fixed_len=fl, n=hb.n, begin=begin, end=end, shortcuts=False)
            elif op == "prefix":
                shortest, tb, te = key
                self._want[k] = oracle_prefix(self.orc, corpus, offs, fixed_len=fl, n=hb.n, shortest=shortest, through_begin=tb,
                                              through_end=te)
            elif op == "suffix":
                shortest, tb, te = key
                self._want[k] = oracle_suffix(self.orc, corpus, offs, fixed_len=fl, n=hb.n, shortest=shortest, through_end=te,
                                              through_begin=tb)
            else:
                begin, end = key
                self._want[k] = oracle_count(self.orc, corpus, offs, fixed_len=fl, n=hb.n, begin=begin, end=end)
        return self._want[k]

    # ------------------------------------------------------------------ entry points
    def run(self, hb, begin, end, label, ordered=False, n=None):
        """pire_gpu_run_batch / _ordered / _lines; n (<= hb.n) runs the first n strings only."""
        from pire_b200 import _native as N
        n = hb.n if n is None else n
        flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)
        bits, masks, states = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
        order = hb.order() if ordered else None
        if hb.lines:
            rc = N.lib.pire_gpu_run_lines(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), None if order is None else order.data_ptr(), n,
                                          flags, bits.data_ptr(), masks.data_ptr(), states.data_ptr(), _stream())
        elif ordered:
            rc = N.lib.pire_gpu_run_batch_ordered(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), order.data_ptr(), n, flags,
                                                  bits.data_ptr(), masks.data_ptr(), states.data_ptr(), _stream())
        else:
            rc = N.lib.pire_gpu_run_batch(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, n, flags, bits.data_ptr(),
                                          masks.data_ptr(), states.data_ptr(), _stream())
        N.check(rc, "run (%s)" % label)
        f, m, s = (x[:n] for x in self.want(hb, "run", begin, end))
        hm, hs = _host(masks), _host(states)
        expect_untouched(label, "accept masks", hm, n)
        expect_untouched(label, "state indices", hs, n)
        expect_equal(label, "StateIndex", hs[:n], s)
        expect_equal(label, "accept masks", hm[:n], m)
        expect_equal(label, "match bits", unpack_bits(label, _host(bits), n), f)

    def prefix(self, hb, shortest, tb, te, label, suffix=False):
        from pire_b200 import _native as N
        flags = (RUN_BEGIN if tb else 0) | (RUN_END if te else 0) | (RUN_LINES if hb.lines else 0)
        out = _filled(hb.n + EXTRA)
        fn = N.lib.pire_gpu_suffix_batch if suffix else N.lib.pire_gpu_prefix_batch
        N.check(fn(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, hb.n, flags, int(shortest), out.data_ptr(), _stream()),
                "%s (%s)" % ("suffix" if suffix else "prefix", label))
        h = _host(out)
        expect_untouched(label, "lengths", h, hb.n)
        got = h[: hb.n].astype(np.int64)
        got[got == 0xFFFFFFFF] = -1
        what = "%s%s tb=%d te=%d" % ("Shortest" if shortest else "Longest", "Suffix" if suffix else "Prefix", tb, te)
        expect_equal(label, what, got, self.want(hb, "suffix" if suffix else "prefix", shortest, tb, te))

    def count(self, hb, begin, end, mode, label):
        from pire_b200 import _native as N
        self.sc.set_count_mode(mode)
        regs = max(1, self.sc.RegexpsCount())
        flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0) | (RUN_LINES if hb.lines else 0)
        counts, bits = _filled((hb.n + EXTRA) * regs), _filled((hb.n + 31) // 32 + 1)
        N.check(N.lib.pire_gpu_count_batch(self.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, hb.n, flags, counts.data_ptr(),
                                           bits.data_ptr(), _stream()), "count (%s)" % label)
        want, wfin = self.want(hb, "count", begin, end)
        hc = _host(counts)
        expect_untouched(label, "counts", hc, hb.n * regs)
        expect_equal("%s mode=%d" % (label, mode), "counts", hc[: hb.n * regs].reshape(hb.n, regs), want)
        expect_equal("%s mode=%d" % (label, mode), "final bits", unpack_bits(label, _host(bits), hb.n), wfin)

    def all(self, hb, label, marks=MARKS, variants=(1, 2, 3, 4, 5, 6), prefix=True, suffix=True, count_modes=(), ordered=None):
        """Every entry point that applies to the batch, every output against the oracle."""
        if ordered is None:
            ordered = hb.offsets is not None
        for begin, end in marks:
            for v in variants:
                self.sc.set_variant(v)
                lab = "%s [%s begin=%d end=%d variant=%d]" % (label, self.name, begin, end, v)
                self.run(hb, begin, end, lab)
                if ordered:
                    self.run(hb, begin, end, lab + " ordered", ordered=True)
            self.sc.set_variant(0)
            for shortest in (False, True):
                lab = "%s [%s]" % (label, self.name)
                if prefix:
                    self.prefix(hb, shortest, begin, end, lab)
                if suffix:
                    self.prefix(hb, shortest, begin, end, lab, suffix=True)
            for mode in count_modes:
                self.count(hb, begin, end, mode, "%s [%s begin=%d end=%d]" % (label, self.name, begin, end))


# ------------------------------------------------------------------------------------------------------ workloads

def glue10_image():
    from pire_b200 import workloads as W
    return W.load_image("glue10")


GLUE10_ALPHABET = b"(0123456789ABCXYZaefhilmorstuw)-: /GET" + bytes(range(0x20, 0x7F))


def plant_rows(rng, rows, literals, every=3):
    n, length = rows.shape
    for i in range(0, n, every):
        lit = literals[int(rng.integers(len(literals)))][:length]
        where = rng.random()
        at = 0 if where < 0.3 else length - len(lit) if where < 0.7 else int(rng.integers(0, length - len(lit) + 1))
        rows[i, at:at + len(lit)] = np.frombuffer(lit, np.uint8)
    return rows


def random_rows(rng, n, length, alphabet, literals=()):
    rows = rng.choice(np.frombuffer(alphabet, np.uint8), size=(n, length))
    return plant_rows(rng, rows, literals) if literals else rows


def random_strings(rng, alphabet, lengths, literals=()):
    out = []
    a = np.frombuffer(alphabet, np.uint8)
    for k, ln in enumerate(lengths):
        s = bytearray(rng.choice(a, size=int(ln)).tobytes())
        if literals and k % 3 == 0 and ln:
            lit = literals[k % len(literals)][: int(ln)]
            at = 0 if k % 2 else int(ln) - len(lit)
            s[at:at + len(lit)] = lit
        out.append(bytes(s))
    return out


def text_of_lines(rng, alphabet, literals, n_lines, long_every=0):
    lines = []
    for k in range(n_lines):
        ln = int(rng.choice([0, 0, 1, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 300]))
        if long_every and k % long_every == long_every - 1:
            ln = 5000
        lines.append(random_strings(rng, alphabet, [ln], literals)[0].replace(b"\n", b" "))
    return b"\n".join(lines) + b"\n"


# ---------------------------------------------------------------------------------------------- (a) cold starts

COLD_SCANNERS = {
    # name: (image, alphabet, literals)
    "anchored": (lambda: EDGE["anchored"]["image"], ALPHABETS["anchored"], [b"abcd", b"abcde", b"cdabe", b"ababe"]),
    "glued": (lambda: EDGE["glued"]["image"], ALPHABETS["glued"], [b"GET ", b"error", b"x123y"]),
    "glue10": (glue10_image, GLUE10_ALPHABET, [b"GET ", b"error", b"timeout", b"(555) 123-4567", b"https://"]),
}


def host_next(sc, s, data):
    for b in data:
        s = sc.Next(s, b)
    return s


def start_state(sc, begin):
    return sc.Next(sc.Initialize(), BeginMark) if begin else sc.Initialize()


def static_hot(sc, max_hot):
    """The first max_hot rows of the static hot order (dfa_tables.cpp StaticHotOrder), via the host Scanner concept."""
    from test_edge_images import static_hot_order
    return set(static_hot_order(sc, max_hot))


def tune_visits(sc, strings, begin):
    """What VisitCountKernel counts for a tuning sample: the state each byte is read in."""
    visits = {}
    for s in strings:
        st = start_state(sc, begin)
        for b in s:
            visits[st] = visits.get(st, 0) + 1
            st = sc.Next(st, b)
    return visits


def cold_start_cases(sc, strings_for_tune, max_hot, tuned, begin):
    """Whether the run's start state lies outside the hot rows, from the host concept alone.  Static: the start is not
    among the first max_hot rows of the static order.  Tuned (with the opposite Begin mark): the sample never reads a
    byte in the run's start state, and at least max_hot other states are read in, so all the hot rows go to them."""
    start = start_state(sc, begin)
    if not tuned:
        return start not in static_hot(sc, max_hot)
    visits = tune_visits(sc, strings_for_tune, not begin)
    return visits.get(start, 0) == 0 and len(visits) >= max_hot


@pytest.mark.parametrize("name", sorted(COLD_SCANNERS))
def test_cold_starts_and_tiny_hot_sets(name, cuda_device):
    """max_hot 1..3, static and tuned hot rows (tuned with the marks opposite to the run's), every mark combination,
    variants 1-6: uniform batches of one block, two blocks and 1 KiB with 1, 31, 32, 33 and 64k+5 strings, CSR with
    empty strings, a length-binned batch with strings of 8 KiB and more (split kernel), and lines."""
    import pire_b200 as P
    make_image, alphabet, literals = COLD_SCANNERS[name]
    image = make_image()
    host = P.Scanner(image, -1)
    init = host.Initialize()
    assert host.Next(init, BeginMark) != init                  # Begin() moves: a run without it starts elsewhere
    rng = np.random.default_rng(len(name))
    uniform = []
    for length in (32, 64, 1024):
        rows = random_rows(rng, 64 * 3 + 5, length, alphabet, literals)
        rows[1::5] = np.resize(np.frombuffer(literals[0], np.uint8), length)     # rows that stay alive to their end
        uniform.append(fixed_batch(rows))
    ragged = csr_batch(random_strings(rng, alphabet, [0, 0, 1, 0] + list(rng.integers(0, 90, size=300)) + [0], literals))
    long_lens = [8192, 8193, 9000, 12345, 20000] + list(rng.integers(0, 200, size=120))
    binned = csr_batch(random_strings(rng, alphabet, long_lens, literals))
    lines = lines_batch(text_of_lines(rng, alphabet, literals, 1200, long_every=300))
    tune_sample = random_strings(rng, alphabet, [64] * 64, literals)
    tune_batch = P.Batch.from_strings(tune_sample)
    cold_seen = {"static": 0, "tuned": 0, "look2": 0}
    lines_cases = []
    chk = Checker(image, name)
    for max_hot in (1, 2, 3):
        for tuned in (False, True):
            for begin, end in MARKS:
                chk.sc = P.Scanner(image, 0)                   # the static hot order again
                chk.sc.set_max_hot(max_hot)
                if tuned:
                    chk.sc.Tune(tune_batch, len(tune_sample), begin=not begin, end=not end)
                    assert chk.sc.info().tuned == 1
                assert chk.sc.info().hot_rows == max_hot
                cold = cold_start_cases(host, tune_sample, max_hot, tuned, begin)
                if max_hot == 1 and not tuned and not begin:
                    assert cold, "Initialize() is the hot row of a one-row static hot set"
                if cold:
                    cold_seen["tuned" if tuned else "static"] += 1
                    lines_cases.append((max_hot, tuned, begin, end))
                    chk.sc.set_variant(4)
                    if chk.sc.info().variant == 4:              # look-ahead set complete: the LOOK ring kernel runs
                        cold_seen["look2"] += 1
                label = "max_hot=%d %s%s" % (max_hot, "tuned" if tuned else "static", " cold" if cold else "")
                for hb, what in zip(uniform, ("32B", "64B", "1KiB")):
                    for n in (1, 31, 32, 33, hb.n):
                        for v in range(1, 7):
                            chk.sc.set_variant(v)
                            chk.run(hb, begin, end, "%s uniform %s n=%d [%s begin=%d end=%d variant=%d]"
                                    % (label, what, n, name, begin, end, v), n=n)
                    chk.sc.set_variant(0)
                    for shortest in (False, True):
                        chk.prefix(uniform[-1], shortest, begin, end, "%s uniform 1KiB [%s]" % (label, name))
                chk.all(ragged, label + " csr", marks=((begin, end),))
                chk.all(binned, label + " binned", marks=((begin, end),), variants=(1, 2, 4), prefix=False, suffix=False)
                chk.all(lines, label + " lines", marks=((begin, end),), variants=(1, 2))
    assert cold_seen["static"] >= 2 and cold_seen["tuned"] >= 1, cold_seen
    if name == "anchored":
        # tuned on text that dies at once, the hot id 0 is the dead state: the look-ahead set is complete with one hot
        # row, and the LOOK ring kernel starts its lanes cold
        assert cold_seen["look2"] >= 1, cold_seen
    # the lines runs of the cold configurations went through ScanLinesKernel, and those of a hot start through the
    # in-stream ScanTextKernel (LaunchLines)
    from pire_b200 import _native as N
    hot_case = (1, False, True, True)
    for case in lines_cases + [hot_case]:
        max_hot, tuned, begin, end = case
        sc = P.Scanner(image, 0)
        sc.set_max_hot(max_hot)
        if tuned:
            sc.Tune(tune_batch, len(tune_sample), begin=not begin, end=not end)
        bits = _filled((lines.n + 31) // 32 + 1)
        flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)
        launched = kernels_launched(lambda: N.check(N.lib.pire_gpu_run_lines(sc._h, lines.corpus_ptr(), lines.offsets_ptr(), None, lines.n, flags,
                                                                             bits.data_ptr(), None, None, _stream()), "run_lines"))
        want, other = ("ScanTextKernel", "ScanLinesKernel") if case == hot_case else ("ScanLinesKernel", "ScanTextKernel")
        assert want in launched and other not in launched, (case, launched[:2000])


# -------------------------------------------------------------------------------------------- (b) wide tables

def test_wide_tables(cuda_device):
    """More than 65 536 states: 32-bit cells in the complete table.  Text over {a, b} sends lanes through states far
    from the hot rows at once; a few other bytes send them to the dead state."""
    import pire_b200 as P
    e = EDGE["wide"]
    rng = np.random.default_rng(131)
    rows = rng.choice(np.frombuffer(b"ab", np.uint8), size=(64 * 40 + 5, 256))
    rows[::17, 100] = ord("c")
    uniform = fixed_batch(rows)
    ragged = csr_batch(random_strings(rng, b"ab" * 50 + b"c", [0, 1, 16, 17, 33] + list(rng.integers(0, 400, size=1500))))
    binned = csr_batch(random_strings(rng, b"ab", [8192, 9001, 16384, 30000] + list(rng.integers(0, 300, size=200))))
    lines = lines_batch(text_of_lines(rng, b"ab" * 30 + b"c", [], 3000, long_every=1000))
    for max_hot in (255, 2):
        chk = Checker(e["image"], "wide")
        chk.sc.set_max_hot(max_hot)
        info = chk.sc.info()
        assert info.states == e["states"] > 65536
        assert info.table_bytes == info.states * info.letters * 4          # 32-bit cells: ScanTables::wide
        label = "max_hot=%d" % max_hot
        chk.all(uniform, label + " uniform", marks=((True, True), (False, False)))
        chk.all(ragged, label + " csr", marks=((True, True), (False, False)))
        chk.all(binned, label + " binned", marks=((True, True),), variants=(1, 2, 4), prefix=False, suffix=False)
        chk.all(lines, label + " lines", marks=((True, True),), variants=(1, 2))
        # the walks did leave the hot rows: most strings end in a state outside them (before the End mark)
        hot = static_hot(P.Scanner(e["image"], -1), max_hot)
        _, _, states = chk.want(uniform, "run", False, False)
        assert np.mean([int(s) not in hot for s in states]) > 0.9


# ------------------------------------------------------------------------------- (c) non-uniform fixed length

FIXED_LENS = (1, 7, 15, 16, 17, 31, 33, 47, 63, 64, 65, 100, 1027)
BASES = (0, 1, 15, 16, 31)
COUNTS = (1, 31, 33, 2003)


def _guarded_rows(rng, n, length):
    """Strings over the letters of the glued scanner (^GET |error|x[0-9]+y) that end in 'erro' or 'x12', or start with
    'ET ' or 'rror': consuming a guard byte 'r' after them, or 'G' / 'e' before them, would change the answer."""
    rows = random_rows(rng, n, length, ALPHABETS["glued"])
    for i in range(n):
        k = i % 6
        if k == 0:
            lit, at = b"erro", length - 4
        elif k == 1:
            lit, at = b"x12", length - 3
        elif k == 2:
            lit, at = b"ET ", 0
        elif k == 3:
            lit, at = b"rror", 0
        else:
            continue
        lit = lit[max(0, -at):][: length]
        at = max(0, at)
        rows[i, at:at + len(lit)] = np.frombuffer(lit, np.uint8)
    return rows


@pytest.mark.parametrize("length", FIXED_LENS)
def test_non_uniform_fixed_length(length, cuda_device):
    """Fixed-length batches with a length that is not a multiple of 32, or a base that is not 32-byte aligned, go to
    the generic, prefix-ring and count-ring kernels.  Guard bytes before the base and after the last string must not be
    read into any string.  length 64 at base 0 is the uniform control."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    rng = np.random.default_rng(length)
    rows = _guarded_rows(rng, max(COUNTS), length)
    glued = Checker(EDGE["glued"]["image"], "glued")
    hf = Checker(W.load_image("hf_glue10"), "hf_glue10")
    assert hf.sc.RegexpsCount() > 4
    for base in BASES:
        full = fixed_batch(rows, base=base, guard_before=b"Ge", guard_after=b"ry")
        assert is_uniform(full.corpus_ptr(), None, length) == (length % 32 == 0 and base % 32 == 0)
        for n in COUNTS:
            hb = full if n == full.n else fixed_batch(rows[:n], base=base, guard_before=b"Ge", guard_after=b"ry")
            label = "fixed_len=%d base=%d n=%d" % (length, base, n)
            glued.all(hb, label, marks=((True, True), (False, False)), ordered=False, prefix=False, suffix=False)
            for begin, end in MARKS:
                for shortest in (False, True):
                    glued.prefix(hb, shortest, begin, end, label)
                    glued.prefix(hb, shortest, begin, end, label, suffix=True)
            for mode in (1, 2, 3):
                hf.count(hb, True, True, mode, label)
            hf.count(hb, False, False, 1, label)


# ------------------------------------------------------------------------------------------- (d) output bounds

@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 65, 64 * 7 + 33, 64 * 7 + 1])
def test_nothing_written_past_n(n, cuda_device):
    """Every C entry point with outputs one bitmap word and 64 entries larger than needed, pre-filled with a
    sentinel (Checker.run / prefix / count check the tails).  Variant 4 forces the two-strings-per-lane kernel, whose
    last pair of an odd number of units reports its first unit only."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    rng = np.random.default_rng(n)
    chk = Checker(glue10_image(), "glue10")
    assert chk.sc.info().variant == 4                       # AUTO is the look-ahead filter: the look-ahead set is complete
    uniform = fixed_batch(random_rows(rng, n, 64, GLUE10_ALPHABET, [b"error", b"GET ", b"timeout"]))
    ragged = csr_batch(random_strings(rng, GLUE10_ALPHABET, list(rng.integers(0, 100, size=n)), [b"error", b"timeout"]))
    text = b"\n".join(random_strings(rng, GLUE10_ALPHABET, list(rng.integers(0, 80, size=n)), [b"error"])) + b"\n"
    lines = lines_batch(text)
    assert lines.n == n
    for hb, what in ((uniform, "uniform"), (ragged, "csr"), (lines, "lines")):
        chk.all(hb, "n=%d %s" % (n, what), marks=((True, True), (False, True)))
    hf = Checker(W.load_image("count_words5"), "count_words5")
    words = fixed_batch(random_rows(rng, n, 64, b"abc de"))
    for mode in (1, 2, 3):
        hf.count(words, True, True, mode, "n=%d uniform" % n)
        hf.count(csr_batch(random_strings(rng, b"abc de", list(rng.integers(0, 70, size=n)))), True, False, mode, "n=%d csr" % n)


# ----------------------------------------------------------------------------------------- (e) past 4 GiB

def test_strings_past_4_gib(cuda_device):
    """A 4.3 GiB device buffer: a fixed-length batch (1000 bytes, not uniform), a CSR batch whose offsets pass 2^32
    (generic and split kernels, prefix, count) and the lines of the same bytes.  The strings within 64 of the one that
    straddles byte 2^32, and the last 64, are compared with the oracle."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    total = int(4.3 * (1 << 30)) // 1024 * 1024
    dev = torch.empty(total + 64, dtype=torch.uint8, device="cuda:0")
    try:
        W.SynthSpec(total // 1024, 1024, plants=W.GLUE10_PLANTS, plant_every=3).fill_device(dev)
        dev[total:] = ord("r")
        # newlines every 997 bytes, and a planted 'error' before some of them
        nl = torch.arange(996, total, 997, device="cuda:0")
        dev[nl] = 10
        sc = Checker(glue10_image(), "glue10")
        hf = Checker(W.load_image("hf_glue10"), "hf_glue10")

        # fixed length 1000 over the whole buffer
        L = 1000
        n = total // L
        straddle = (1 << 32) // L
        idx = np.concatenate([np.arange(straddle - 64, straddle + 65), np.arange(n - 64, n)])
        bits, masks, states = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
        from pire_b200 import _native as N
        for variant in (0, 2):
            sc.sc.set_variant(variant)
            N.check(N.lib.pire_gpu_run_batch(sc.sc._h, dev.data_ptr(), None, L, n, RUN_BEGIN | RUN_END, bits.data_ptr(), masks.data_ptr(),
                                             states.data_ptr(), _stream()), "run 4 GiB fixed")
            hbits, hm, hs = _host(bits), _host(masks), _host(states)
            expect_untouched("4GiB fixed", "accept masks", hm, n)
            f = unpack_bits("4GiB fixed", hbits, n)
            rows = np.stack([dev[int(i) * L:(int(i) + 1) * L].cpu().numpy() for i in idx])
            hb = fixed_batch(rows)
            wf, wm, ws = sc.want(hb, "run", True, True)
            label = "4GiB fixed_len=1000 variant=%d" % variant
            expect_equal(label, "match bits", f[idx], wf)
            expect_equal(label, "accept masks", hm[idx], wm)
            expect_equal(label, "StateIndex", hs[idx], ws)
        sc.sc.set_variant(0)
        del bits, masks, states

        # CSR: lengths 0..2000 and every 500th string 9000 bytes (the split kernel), offsets past 2^32
        g = torch.Generator(device="cuda:0")
        g.manual_seed(4)
        lens = torch.randint(0, 2000, (total // 900,), generator=g, device="cuda:0", dtype=torch.int64)
        lens[::500] = 9000
        offs = torch.zeros(lens.numel() + 1, dtype=torch.int64, device="cuda:0")
        torch.cumsum(lens, 0, out=offs[1:])
        m = int(torch.searchsorted(offs, torch.tensor([total], device="cuda:0")).item()) - 1
        offs = offs[: m + 1].contiguous()
        assert int(offs[-1]) <= total and int(offs[-1]) > (1 << 32)
        ho = offs.cpu().numpy().astype(np.uint64)
        straddle = int(np.searchsorted(ho, 1 << 32, side="right")) - 1
        assert ho[straddle] <= (1 << 32) < ho[straddle + 1]
        picks = [(max(0, straddle - 64), straddle + 65), (m - 64, m)]

        def host_csr(lo, hi):
            a, b = int(ho[lo]), int(ho[hi])
            return np.concatenate([dev[a:b].cpu().numpy(), np.zeros(32, np.uint8)]), (ho[lo:hi + 1] - ho[lo]).astype(np.uint64)

        samples = [host_csr(lo, hi) for lo, hi in picks]
        for ordered in (False, True):
            bits, masks, states = _filled((m + 31) // 32 + 1), _filled(m + EXTRA), _filled(m + EXTRA)
            if ordered:
                order = torch.empty(m, dtype=torch.int32, device="cuda:0")
                N.check(N.lib.pire_gpu_length_order(offs.data_ptr(), m, order.data_ptr(), 0, _stream()), "order")
                rc = N.lib.pire_gpu_run_batch_ordered(sc.sc._h, dev.data_ptr(), offs.data_ptr(), order.data_ptr(), m, RUN_BEGIN | RUN_END,
                                                      bits.data_ptr(), masks.data_ptr(), states.data_ptr(), _stream())
            else:
                rc = N.lib.pire_gpu_run_batch(sc.sc._h, dev.data_ptr(), offs.data_ptr(), 0, m, RUN_BEGIN | RUN_END, bits.data_ptr(),
                                              masks.data_ptr(), states.data_ptr(), _stream())
            N.check(rc, "run 4 GiB csr")
            f = unpack_bits("4GiB csr", _host(bits), m)
            hm, hs = _host(masks), _host(states)
            expect_untouched("4GiB csr", "state indices", hs, m)
            for (lo, hi), (corpus, o) in zip(picks, samples):
                hb = HostBatch(corpus, offsets=o)
                wf, wm, ws = sc.want(hb, "run", True, True)
                label = "4GiB csr ordered=%d strings %d..%d" % (ordered, lo, hi)
                expect_equal(label, "match bits", f[lo:hi], wf)
                expect_equal(label, "accept masks", hm[lo:hi], wm)
                expect_equal(label, "StateIndex", hs[lo:hi], ws)
            del bits, masks, states
        # prefix and count on the same CSR batch
        out = _filled(m + EXTRA)
        N.check(N.lib.pire_gpu_prefix_batch(sc.sc._h, dev.data_ptr(), offs.data_ptr(), 0, m, RUN_BEGIN, 0, out.data_ptr(), _stream()),
                "prefix 4 GiB")
        hp = _host(out).astype(np.int64)
        hp[hp == 0xFFFFFFFF] = -1
        expect_untouched("4GiB prefix", "lengths", _host(out), m)
        for (lo, hi), (corpus, o) in zip(picks, samples):
            want = oracle_prefix(sc.orc, corpus, o, through_begin=True)
            expect_equal("4GiB csr LongestPrefix strings %d..%d" % (lo, hi), "lengths", hp[lo:hi], want)
        del out
        regs = hf.sc.RegexpsCount()
        counts, cbits = _filled((m + EXTRA) * regs), _filled((m + 31) // 32 + 1)
        N.check(N.lib.pire_gpu_count_batch(hf.sc._h, dev.data_ptr(), offs.data_ptr(), 0, m, RUN_BEGIN | RUN_END, counts.data_ptr(),
                                           cbits.data_ptr(), _stream()), "count 4 GiB")
        hc = _host(counts)
        expect_untouched("4GiB count", "counts", hc, m * regs)
        hc = hc[: m * regs].reshape(m, regs)
        fin = unpack_bits("4GiB count", _host(cbits), m)
        for (lo, hi), (corpus, o) in zip(picks, samples):
            want, wfin = oracle_count(hf.orc, corpus, o)
            expect_equal("4GiB csr count strings %d..%d" % (lo, hi), "counts", hc[lo:hi], want)
            expect_equal("4GiB csr count strings %d..%d" % (lo, hi), "final bits", fin[lo:hi], wfin)
        del counts, cbits, offs, lens

        # the lines of the same bytes
        batch = P.Batch.from_text(dev[:total])
        nl_n = batch.n
        lo_off = batch.offsets.cpu().numpy().astype(np.uint64)
        assert lo_off[-1] > (1 << 32)
        straddle = int(np.searchsorted(lo_off, 1 << 32, side="right")) - 1
        picks = [(straddle - 64, straddle + 65), (nl_n - 64, nl_n)]
        bits, masks, states = _filled((nl_n + 31) // 32 + 1), _filled(nl_n + EXTRA), _filled(nl_n + EXTRA)
        N.check(N.lib.pire_gpu_run_lines(sc.sc._h, dev.data_ptr(), batch.offsets.data_ptr(), None, nl_n, RUN_BEGIN | RUN_END,
                                         bits.data_ptr(), masks.data_ptr(), states.data_ptr(), _stream()), "lines 4 GiB")
        f = unpack_bits("4GiB lines", _host(bits), nl_n)
        hm, hs = _host(masks), _host(states)
        expect_untouched("4GiB lines", "state indices", hs, nl_n)
        for lo, hi in picks:
            a, b = int(lo_off[lo]), int(lo_off[hi])
            hb = HostBatch(np.concatenate([dev[a:b].cpu().numpy(), np.zeros(32, np.uint8)]), offsets=lo_off[lo:hi + 1] - lo_off[lo],
                           lines=True)
            wf, wm, ws = sc.want(hb, "run", True, True)
            label = "4GiB lines %d..%d" % (lo, hi)
            expect_equal(label, "match bits", f[lo:hi], wf)
            expect_equal(label, "accept masks", hm[lo:hi], wm)
            expect_equal(label, "StateIndex", hs[lo:hi], ws)
        del batch, bits, masks, states
    finally:
        del dev
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

