"""pire_gpu_slow_run_batch on the GPU, bit for bit against the reference SlowScanner (its recorded answers in
tests/golden/slow_images.json.xz) and against the numpy walker of synthesized NFAs (tests/synth_nfa.py).

Both kernels and every set width run: the lane path (S <= 256, W = 1, 2, 4, 8) and the warp path (256 < S <= 4096, up to
128 words).  Every output carries sentinel words past its end."""
import ctypes as C

import numpy as np
import pytest

import pire_b200 as P
from pire_b200 import _native as N
from slow_fixtures import SLOW
import synth_nfa as SN

pytestmark = pytest.mark.gpu

SENTINEL = 0x5EA15EA1
PAD = 8
EINVAL = -1


def torch():
    import torch as t
    return t


def csr(strings, align=0):
    """A CSR batch of `strings` whose corpus starts `align` bytes into its buffer."""
    t = torch()
    raw = b"\xAA" * align + b"".join(strings)
    buf = t.tensor(list(raw) or [0], dtype=t.uint8, device="cuda:0")
    offs = np.zeros(len(strings) + 1, np.int64)
    offs[1:] = np.cumsum([len(s) for s in strings])
    return P.Batch(buf[align:] if raw else buf, t.tensor(offs, device="cuda:0"), n=len(strings))


def outputs(n, words):
    t = torch()
    bits = t.full(((n + 31) // 32 + PAD,), SENTINEL, dtype=t.int64, device="cuda:0").to(t.int32)
    sets = t.full((n * words + PAD,), SENTINEL, dtype=t.int64, device="cuda:0").to(t.int32)
    return bits, sets


def run(sc, batch, flags, start_sets=None, want_bits=True, want_sets=True):
    """(match bits as bool[n], sets uint32[n, W]); the sentinels past both outputs checked."""
    t = torch()
    n, w = batch.n, sc.set_words
    bits, sets = outputs(n, w)
    st = None
    if start_sets is not None:
        st = t.tensor(np.ascontiguousarray(start_sets, np.uint32).view(np.int32).reshape(-1), device="cuda:0")
    sc.run_batch(batch, flags, bits if want_bits else None, sets if want_sets else None, start_sets=st)
    t.cuda.synchronize()
    b = bits.cpu().numpy().view(np.uint32)
    s = sets.cpu().numpy().view(np.uint32)
    nw = (n + 31) // 32
    if want_bits:
        assert (b[nw:] == SENTINEL).all(), "match bits past the end"
        if n % 32:
            assert b[nw - 1] >> (n % 32) == 0, "bits past n"
    else:
        assert (b == SENTINEL).all()
    assert (s[n * w:] == SENTINEL).all(), "sets past the end"
    if not want_sets:
        assert (s == SENTINEL).all()
    matches = np.unpackbits(b[:nw].view(np.uint8), bitorder="little")[:n].astype(bool)
    return matches, s[: n * w].reshape(n, w)


FLAGS = {(b, e): (N.RUN_BEGIN if b else 0) | (N.RUN_END if e else 0) for b in (False, True) for e in (False, True)}


@pytest.mark.parametrize("e", SLOW, ids=lambda e: e.name)
def test_fixtures_equal_reference(cuda_device, e):
    sc = P.SlowScanner(e.image, cuda_device)
    for (begin, end, from_sets), (final, sets) in e.runs.items():
        for align in (0, 3) if e.name.startswith("heavy") else (0,):
            got_f, got_s = run(sc, csr(e.strings, align), FLAGS[(begin, end)], e.start_sets if from_sets else None)
            assert (got_f == final).all() and (got_s == sets).all(), (begin, end, from_sets, align)
        if not from_sets:
            r = P.Runner(sc)
            r = r.Begin() if begin else r
            r = r.Run(csr(e.strings))
            r = r.End() if end else r
            assert (r.Matches() == final).all() and (r.Sets() == sets).all()


def synth_strings(rng, n, max_len, empty_every=7):
    return [b"" if k % empty_every == 3 else rng.integers(0, 256, int(rng.integers(0, max_len + 1)), dtype=np.uint8).tobytes()
            for k in range(n)]


def oracle(nfa, strings, begin, end, starts=None):
    f, s = [], []
    for i, d in enumerate(strings):
        ff, ss = nfa.run(d, None if starts is None else nfa.unpack(starts[i]), begin, end)
        f.append(ff)
        s.append(ss)
    return np.array(f, bool), np.array(s, np.uint32).reshape(len(strings), nfa.words)


@pytest.mark.parametrize("fam", [f[0] for f in SN.FAMILIES])
def test_synth_csr_every_mark_and_start(cuda_device, fam):
    nfa = SN.family(fam)
    sc = P.SlowScanner(nfa.image(), cuda_device)
    assert sc.info().set_words == nfa.words
    rng = np.random.default_rng(100 + nfa.states)
    n = 45 if nfa.states < 1000 else 33
    strings = synth_strings(rng, n, 70)
    starts = rng.integers(0, 1 << 32, n * nfa.words, dtype=np.uint64).astype(np.uint32).reshape(n, nfa.words)
    starts &= rng.integers(0, 1 << 32, starts.shape, dtype=np.uint64).astype(np.uint32)
    for (begin, end), flags in FLAGS.items():
        for st in (None, starts):
            want_f, want_s = oracle(nfa, strings, begin, end, st)
            got_f, got_s = run(sc, csr(strings, int(rng.integers(0, 32))), flags, st)
            assert (got_f == want_f).all() and (got_s == want_s).all(), (begin, end, st is None)


@pytest.mark.parametrize("fam", ["s1", "s33", "s100", "s256", "s257", "s1500"])
def test_synth_fixed_length_every_alignment(cuda_device, fam):
    nfa = SN.family(fam)
    sc = P.SlowScanner(nfa.image(), cuda_device)
    rng = np.random.default_rng(7)
    t = torch()
    for fixed in (0, 1, 13, 32, 47):
        n = 37
        data = rng.integers(0, 256, n * fixed + 31, dtype=np.uint8)
        dev = t.tensor(data, device="cuda:0")
        for align in range(0, 32, 5 if fixed else 31):
            strings = [data[align + i * fixed: align + (i + 1) * fixed].tobytes() for i in range(n)]
            want_f, want_s = oracle(nfa, strings, True, True)
            got_f, got_s = run(sc, P.Batch(dev[align:], fixed_len=fixed, n=n), N.RUN_BEGIN | N.RUN_END)
            assert (got_f == want_f).all() and (got_s == want_s).all(), (fixed, align)


@pytest.mark.parametrize("name", ["heavy/a30", "heavy/error200"])
def test_null_output_subsets_and_n_zero(cuda_device, name):
    e = next(x for x in SLOW if x.name == name)
    sc = P.SlowScanner(e.image, cuda_device)
    final, sets = e.runs[(True, True, False)]
    b = csr(e.strings)
    for want_bits in (False, True):
        for want_sets in (False, True):
            got_f, got_s = run(sc, b, N.RUN_BEGIN | N.RUN_END, want_bits=want_bits, want_sets=want_sets)
            if want_bits:
                assert (got_f == final).all()
            if want_sets:
                assert (got_s == sets).all()
    empty = P.Batch(b.corpus, b.offsets[:1].contiguous(), n=0)
    run(sc, empty, N.RUN_BEGIN | N.RUN_END)


@pytest.mark.parametrize("name", ["heavy/foo64bar", "heavy/error200", "approx1"])
def test_stream_chained_in_place(cuda_device, name):
    """Each string cut at random points, the pieces run round after round with d_sets == d_start_sets: the same as one
    call over the whole strings."""
    t = torch()
    e = next(x for x in SLOW if x.name == name)
    sc = P.SlowScanner(e.image, cuda_device)
    rng = np.random.default_rng(5)
    strings = e.strings
    n, w, rounds = len(strings), sc.set_words, 4
    cuts = [sorted(rng.integers(0, len(s) + 1, rounds - 1).tolist()) for s in strings]
    pieces = [[s[([0] + c)[k]: (c + [len(s)])[k]] for s, c in zip(strings, cuts)] for k in range(rounds)]
    state = t.tensor(np.tile(sc.Initialize(), n).view(np.int32), device="cuda:0")
    bits = None
    for k in range(rounds):
        flags = (N.RUN_BEGIN if k == 0 else 0) | (N.RUN_END if k == rounds - 1 else 0)
        bits = t.zeros((n + 31) // 32, dtype=t.int32, device="cuda:0")
        sc.run_batch(csr(pieces[k], k), flags, bits, state, start_sets=state)
    t.cuda.synchronize()
    final, sets = e.runs[(True, True, False)]
    got = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
    assert (got == final).all() and (state.cpu().numpy().view(np.uint32).reshape(n, w) == sets).all()
    # the Python mirror: Runner(slow, sets) chains through SetTensor()
    r = P.Runner(sc).Begin().Run(csr(pieces[0]))
    for k in range(1, rounds):
        r = P.Runner(sc, r.SetTensor()).Run(csr(pieces[k]))
    half = P.Runner(sc).Begin().Run(csr(strings))
    assert (r.Sets() == half.Sets()).all() and (r.Matches() == half.Matches()).all()


def lines_text(rng, alphabet, n_lines, max_len, final_newline=True):
    lines = [bytes(rng.choice(np.frombuffer(alphabet, np.uint8), int(rng.integers(0, max_len + 1))).tolist())
             for _ in range(n_lines)]
    text = b"\n".join(lines) + (b"\n" if final_newline else b"")
    return text, lines


@pytest.mark.parametrize("name", ["heavy/a30", "heavy/d3_50_d3", "heavy/error200", "approx2"])
def test_lines_and_line_stream(cuda_device, name):
    t = torch()
    e = next(x for x in SLOW if x.name == name)
    sc = P.SlowScanner(e.image, cuda_device)
    rng = np.random.default_rng(11)
    alphabet = bytes(sorted(set(b"".join(e.strings)) - {10})) or b"ab"
    for final_nl in (True, False):
        text, lines = lines_text(rng, alphabet, 301, 400, final_nl)
        lb = P.Batch.from_text(t.tensor(list(text), dtype=t.uint8, device="cuda:0"))
        assert lb.n == len(lines)
        got_f, got_s = run(sc, lb, N.RUN_BEGIN | N.RUN_END)
        want_f, want_s = run(sc, csr(lines), N.RUN_BEGIN | N.RUN_END)
        assert (got_f == want_f).all() and (got_s == want_s).all()
        # LineStream frames through small slots: frame by frame, the lines' results
        ls = P.LineStream(cuda_device, 4096)
        host = np.frombuffer(text, np.uint8)
        got, at = [], 0
        for cut in (0, 1000, 1001, 7000, len(host)):
            for f in ls.feed(host[at:cut], last=cut == len(host)):
                assert f.first_line == len(got)
                got += P.Runner(sc).Begin().Run(f).End().Matches().tolist()
            at = cut
        assert got == want_f.tolist()


def test_long_string_both_paths(cuda_device):
    """A 5 MiB string in one call equals the same string cut in three and chained through its set; a30 accepts the
    string that ends with a and 30 more bytes, error200 (anchored at the line start, 5 MiB back) accepts nothing."""
    t = torch()
    rng = np.random.default_rng(3)
    for name, tail in (("heavy/a30", b"a" + b"b" * 30), ("heavy/error200", b"error" + b"x" * 200)):
        e = next(x for x in SLOW if x.name == name)
        sc = P.SlowScanner(e.image, cuda_device)
        body = rng.choice(np.frombuffer(b"abcerox", np.uint8), 5 << 20).tobytes()
        for s in (body, body[: -len(tail)] + tail):
            state = t.tensor(sc.Initialize().view(np.int32), device="cuda:0")
            cuts = [0, 1 << 20, (5 << 20) - 4097, len(s)]
            bits = t.zeros(1, dtype=t.int32, device="cuda:0")
            for k in range(3):
                flags = (N.RUN_BEGIN if k == 0 else 0) | (N.RUN_END if k == 2 else 0)
                sc.run_batch(csr([s[cuts[k]: cuts[k + 1]]], k), flags, bits, state, start_sets=state)
            t.cuda.synchronize()
            for align in (0, 5):
                got_f, got_s = run(sc, csr([s], align), N.RUN_BEGIN | N.RUN_END)
                assert bool(got_f[0]) == bool(bits.cpu().numpy()[0] & 1)
                assert (got_s[0] == state.cpu().numpy().view(np.uint32)).all()
            if s is not body:
                assert bool(got_f[0]) == (name == "heavy/a30")


def test_refusals(cuda_device):
    t = torch()
    sc = P.SlowScanner(SLOW[0].image, cuda_device)
    b = csr([b"abc", b"de"])
    bits, sets = outputs(2, sc.set_words)
    lib, h = N.lib, sc._h
    st = t.zeros(2 * sc.set_words, dtype=t.int32, device="cuda:0")
    assert lib.pire_gpu_slow_run_batch(h, b.corpus.data_ptr(), b.offsets.data_ptr(), 0, 2, N.RUN_LINES, st.data_ptr(),
                                       bits.data_ptr(), sets.data_ptr(), None) == EINVAL
    assert lib.pire_gpu_slow_run_batch(h, b.corpus.data_ptr(), b.offsets.data_ptr(), 0, 2, 8, None, bits.data_ptr(),
                                       sets.data_ptr(), None) == EINVAL
    assert lib.pire_gpu_slow_run_batch(h, None, None, 4, 2, 0, None, bits.data_ptr(), sets.data_ptr(), None) == EINVAL
    assert lib.pire_gpu_slow_run_batch(h, b.corpus.data_ptr(), None, 0, 2, N.RUN_LINES, None, bits.data_ptr(),
                                       sets.data_ptr(), None) == EINVAL
    # n == 0 is a no-op, and empty fixed-length strings need no corpus
    assert lib.pire_gpu_slow_run_batch(h, None, None, 0, 0, 0, None, bits.data_ptr(), sets.data_ptr(), None) == 0
    t.cuda.synchronize()
    assert (bits.cpu().numpy().view(np.uint32) == SENTINEL).all()
    assert lib.pire_gpu_slow_run_batch(h, None, None, 0, 2, 0, None, bits.data_ptr(), sets.data_ptr(), None) == 0
    with pytest.raises(N.PireGpuError):
        P.SlowScanner(SN.random_nfa(14, 4097, 2, 1.0).image(), cuda_device)
    dfa_h = C.c_void_p()
    img = SLOW[0].image
    assert lib.pire_gpu_scanner_create((C.c_char * len(img)).from_buffer_copy(img), len(img), cuda_device, C.byref(dfa_h)) == -2
