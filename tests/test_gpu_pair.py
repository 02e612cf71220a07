"""Two scanners over one batch (pire_gpu_run_pair_batch, Pire::Run(sc1, sc2, ...) / Runner(ScannerPair)): every one of the
six outputs must equal, bit for bit, what each scanner gets alone on the same bytes -- pire_gpu_run_batch_from with that
scanner's starts, or pire_gpu_run_batch when its start array is NULL -- with 64 sentinel words past n in every output.
A sample is also checked against the oracle's run from any state (tests/string_oracle.py).  Covers glued, counting,
headline, edge and many-regexp images in pairs, one handle twice, the largest pair of hot tables, small hot sets
(without a look-ahead set), tuned handles, uniform batches of 32 to 4096 bytes, CSR / unaligned / odd-length batches (the
unfused path), all mark combinations, starts NULL / random / outside one scanner, rounds chained in place, NoExit in
one scanner only, NULL outputs, bad arguments, and the Python and C++ front ends."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from refpire import Oracle
from string_oracle import run_from
from test_count_images import COUNT_IMAGES
from test_edge_images import ALPHABETS, EDGE
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, MARKS, SENTINEL, _filled, _host, _stream, csr_batch, expect_equal, expect_untouched,
                            fixed_batch, is_uniform, random_rows, random_strings)

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
LITERALS = [b"GET ", b"error", b"timeout", b"(555) 123-4567", b"https://", b"hello  world", b"fatal", b"foo"]
UNIFORM = [(32, 1), (32, 31), (64, 32 * 3 + 5), (1024, 32 * 2 + 1), (4096, 33)]


def _i32(values):
    import torch
    v = np.asarray(values, dtype=np.uint64).astype(np.uint32).view(np.int32)
    return torch.from_numpy(v.copy()).to("cuda:0")


def _flags(begin, end):
    return (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)


def _starts(values, n):
    """n start words and the sentinels after them, or None."""
    return None if values is None else _i32(list(values[:n]) + [SENTINEL] * EXTRA)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _outputs(n, want=(True, True, True)):
    return [_filled((n + 31) // 32 + 1) if want[0] else None, _filled(n + EXTRA) if want[1] else None,
            _filled(n + EXTRA) if want[2] else None]


def _read(label, outs, n):
    """Host copies of (bits, masks, states); the words past each one's end must still hold the sentinel."""
    res = []
    for k, (t, valid) in enumerate(zip(outs, ((n + 31) // 32, n, n))):
        if t is None:
            res.append(None)
            continue
        h = _host(t)
        expect_untouched(label, ("match bitmap", "accept masks", "state indices")[k], h, valid)
        res.append(h[:valid].copy())
    return res


def single(sc, hb, flags, starts, n=None, want=(True, True, True)):
    """One scanner alone: pire_gpu_run_batch_from with starts, pire_gpu_run_batch without."""
    from pire_b200 import _native as N
    n = hb.n if n is None else n
    outs = _outputs(n, want)
    if starts is None:
        N.check(N.lib.pire_gpu_run_batch(sc._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, n, flags, *map(_ptr, outs), _stream()),
                "pire_gpu_run_batch")
    else:
        N.check(N.lib.pire_gpu_run_batch_from(sc._h, hb.corpus_ptr(), hb.offsets_ptr(), None, hb.fixed_len, n, flags, starts.data_ptr(),
                                              *map(_ptr, outs), _stream()), "pire_gpu_run_batch_from")
    return _read("single", outs, n)


def pair_call(sc1, sc2, hb, flags, st1, st2, n=None, want=(True,) * 6, outs=None):
    from pire_b200 import _native as N
    n = hb.n if n is None else n
    if outs is None:
        outs = _outputs(n, want[:3]) + _outputs(n, want[3:])
    rc = N.lib.pire_gpu_run_pair_batch(sc1._h, sc2._h, hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len, n, flags, _ptr(st1), _ptr(st2),
                                       *map(_ptr, outs), _stream())
    N.check(rc, "pire_gpu_run_pair_batch")
    return _read("pair", outs[:3], n) + _read("pair", outs[3:], n)


def check_pair(sc1, sc2, hb, flags, starts1, starts2, label, want=(True,) * 6):
    """The pair's six outputs against the two single-scanner calls on the same bytes."""
    st1, st2 = _starts(starts1, hb.n), _starts(starts2, hb.n)
    got = pair_call(sc1, sc2, hb, flags, st1, st2, want=want)
    ref = single(sc1, hb, flags, st1, want=want[:3]) + single(sc2, hb, flags, st2, want=want[3:])
    for k in range(6):
        if want[k]:
            expect_equal(label, ("bits", "masks", "states")[k % 3] + str(k // 3 + 1), got[k], ref[k])
        else:
            assert got[k] is None
    return got


def random_starts(rng, size, n, outside=True):
    st = rng.integers(0, max(size, 1), size=n).astype(np.uint64)
    if outside and n >= 3:
        st[1::11] = size                        # Size(): outside the scanner
        st[2::13] = 0xFFFFFFFF
    return st


def image_of(name):
    from pire_b200 import workloads as W
    if name in EDGE:
        return EDGE[name]["image"]
    if name in COUNT_IMAGES:
        return COUNT_IMAGES[name]["image"]
    golden = [c for c in GOLDEN if c.name == name]
    if golden:
        return golden[0].image
    return W.load_image(name)


def scanner(name, max_hot=None):
    import pire_b200 as P
    sc = P.Scanner(image_of(name), 0)
    if max_hot is not None:
        sc.set_max_hot(max_hot)
    return sc


def look_ok(sc):
    """Whether the handle has a look-ahead set: pinned to LOOK, a handle without one resolves to PRED."""
    from pire_b200 import _native as N
    sc.set_variant(N.VARIANT_LOOK)
    ok = sc.info().variant == N.VARIANT_LOOK
    sc.set_variant(N.VARIANT_AUTO)
    return ok


def batches(rng, alphabet):
    out = []
    for length, n in UNIFORM:
        hb = fixed_batch(random_rows(rng, n, length, alphabet, LITERALS))
        assert is_uniform(hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len)
        out.append(("uniform len=%d n=%d" % (length, n), hb))
    return out


def run_pairs(sc1, sc2, name, rng, alphabet, start_sets=None):
    for label, hb in batches(rng, alphabet):
        s1, s2 = random_starts(rng, sc1.Size(), hb.n), random_starts(rng, sc2.Size(), hb.n)
        sets = start_sets or ((None, None), (s1, None), (None, s2), (s1, s2))
        for starts1, starts2 in sets:
            for begin, end in MARKS:
                check_pair(sc1, sc2, hb, _flags(begin, end), starts1, starts2,
                           "%s %s begin=%d end=%d starts=%d%d" % (name, label, begin, end, starts1 is not None, starts2 is not None))


# ------------------------------------------------------------------------------------------------------------- pairs

ALPHA_ALL = GLUE10_ALPHABET + b"hello world foo"


@pytest.mark.parametrize("names", [("AppendixA", "glue10"), ("glue10", "AppendixA"), ("headline", "headline_iu"), ("glue10", "headline")])
def test_pairs_of_scanners(names, cuda_device):
    rng = np.random.default_rng(sum(map(len, names)))
    sc1, sc2 = scanner(names[0]), scanner(names[1])
    run_pairs(sc1, sc2, "+".join(names), rng, ALPHA_ALL)


def test_one_handle_twice(cuda_device):
    rng = np.random.default_rng(2)
    sc = scanner("glue10")
    run_pairs(sc, sc, "glue10 twice", rng, ALPHA_ALL)


def test_largest_hot_tables(cuda_device):
    """glue10 + hf_glue10 (255 and 211 hot rows) and two glue10 handles (255 + 255: the most shared memory a pair takes)."""
    rng = np.random.default_rng(3)
    g1, g2, hf = scanner("glue10"), scanner("glue10"), scanner("hf_glue10")
    assert g1.info().hot_rows == 255 and g2.info().hot_rows == 255 and hf.info().hot_rows == 211
    run_pairs(g1, hf, "glue10+hf_glue10", rng, ALPHA_ALL)
    run_pairs(hf, g1, "hf_glue10+glue10", rng, ALPHA_ALL)
    run_pairs(g1, g2, "glue10+glue10", rng, ALPHA_ALL)


EDGE_NAMES = ["EmptyScanner@784", "all_final", "wide", "absorbing", "none_hot", "anchored"]


def test_edge_images_among_themselves(cuda_device):
    """The empty scanner (no regexps), one state, 32-bit table cells and a scanner with no hot rows beyond the sink, in pairs."""
    rng = np.random.default_rng(4)
    scs = {name: scanner(name) for name in EDGE_NAMES}
    assert scs["EmptyScanner@784"].RegexpsCount() == 0 and scs["all_final"].Size() == 1 and scs["wide"].Size() > 65536
    alphabet = b"".join(ALPHABETS.values())
    for a, b in [("EmptyScanner@784", "all_final"), ("all_final", "wide"), ("wide", "EmptyScanner@784"), ("none_hot", "wide"),
                 ("absorbing", "anchored"), ("anchored", "none_hot")]:
        run_pairs(scs[a], scs[b], "%s+%s" % (a, b), rng, alphabet)


def test_past_32_regexps(cuda_device):
    """An image of 300 regexps beside glue10: the masks hold ids below 32, the states name the rest (pire_gpu_accept_sets)."""
    from pire_b200 import _native as N
    rng = np.random.default_rng(5)
    many, g = scanner("w300"), scanner("glue10")
    ids = rng.integers(0, 300, size=32 * 4 + 3)
    ids[:8] = [0, 31, 32, 33, 63, 64, 255, 299]
    rows = rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvxyz", np.uint8), size=(len(ids), 64))
    for i, k in enumerate(ids):
        rows[i, 60:] = np.frombuffer(b"w%03d" % k, np.uint8)              # every string ends in a match of regexp k
    hb = fixed_batch(rows)
    for begin, end in MARKS:
        check_pair(many, g, hb, _flags(begin, end), None, None, "w300+glue10 begin=%d end=%d" % (begin, end))
    got = check_pair(many, g, hb, 0, None, None, "w300+glue10 no marks")      # EndMark leaves `[a-z]*w%03d`
    words = N.lib.pire_gpu_accept_words(many._h)
    assert words == 10
    states = _i32(got[2])
    sets = _filled(hb.n * words + EXTRA)
    N.check(N.lib.pire_gpu_accept_sets(many._h, states.data_ptr(), hb.n, sets.data_ptr(), _stream()), "accept_sets")
    rows_ = _host(sets)[: hb.n * words].reshape(hb.n, words)
    high = 0
    for i in range(hb.n):
        ids = [r for r in range(words * 32) if (int(rows_[i, r // 32]) >> (r % 32)) & 1]
        assert ids == many.AcceptedRegexps(int(got[2][i])), i
        high += any(r >= 32 for r in ids)
    assert high > 0


def test_small_hot_sets_and_tuned_handles(cuda_device):
    """set_max_hot(2) and (6): one of them has no look-ahead set, so its chain reads the table on every byte; then handles
    after Tune and AutoSelect."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    rng = np.random.default_rng(6)
    small = [scanner("glue10", 2), scanner("glue10", 6), scanner("AppendixA", 2), scanner("headline", 6)]
    assert not all(look_ok(sc) for sc in small), "no handle without a look-ahead set"
    run_pairs(small[0], small[1], "glue10/2+glue10/6", rng, ALPHA_ALL)
    run_pairs(small[2], small[3], "AppendixA/2+headline/6", rng, ALPHA_ALL)
    run_pairs(small[0], scanner("glue10"), "glue10/2+glue10", rng, ALPHA_ALL)
    spec = W.SynthSpec(4096, 1024, plants=W.GLUE10_PLANTS)
    dev = torch.empty(spec.total_bytes(), dtype=torch.uint8, device="cuda:0")
    spec.fill_device(dev)
    sample = P.Batch(dev, fixed_len=1024, n=4096)
    tuned = [scanner("glue10"), scanner("headline")]
    for sc in tuned:
        sc.Tune(sample, 1024)
        sc.AutoSelect(sample)
        assert sc.info().tuned
    run_pairs(tuned[0], tuned[1], "tuned glue10+headline", rng, ALPHA_ALL)


# ----------------------------------------------------------------------------------------------------------- batches

def test_unfused_batches(cuda_device):
    """CSR with empty strings, a fixed length that is not a multiple of 32 and an unaligned corpus: the single launches."""
    rng = np.random.default_rng(7)
    sc1, sc2 = scanner("glue10"), scanner("AppendixA")
    lengths = [0, 0, 1, 31, 32, 33, 1000] + [int(x) for x in rng.integers(0, 3000, size=90)] + [0]
    cases = [("CSR", csr_batch(random_strings(rng, ALPHA_ALL, lengths, LITERALS))),
             ("fixed 100", fixed_batch(random_rows(rng, 77, 100, ALPHA_ALL, LITERALS))),
             ("unaligned 64", fixed_batch(random_rows(rng, 70, 64, ALPHA_ALL, LITERALS), base=1)),
             ("unaligned 1024", fixed_batch(random_rows(rng, 40, 1024, ALPHA_ALL, LITERALS), base=16))]
    for label, hb in cases:
        assert not is_uniform(hb.corpus_ptr(), hb.offsets_ptr(), hb.fixed_len)
        s1, s2 = random_starts(rng, sc1.Size(), hb.n), random_starts(rng, sc2.Size(), hb.n)
        for starts1, starts2 in ((None, None), (s1, None), (None, s2), (s1, s2)):
            for begin, end in MARKS:
                check_pair(sc1, sc2, hb, _flags(begin, end), starts1, starts2, "%s begin=%d end=%d" % (label, begin, end))


def test_sizes_of_n(cuda_device):
    """n = 0 writes nothing; n = 1, 31, 32 * k + r on a uniform buffer longer than the batch."""
    rng = np.random.default_rng(8)
    sc1, sc2 = scanner("glue10"), scanner("headline")
    hb = fixed_batch(random_rows(rng, 32 * 9 + 13, 64, ALPHA_ALL, LITERALS))
    outs = _outputs(8) + _outputs(8)
    pair_call(sc1, sc2, hb, 3, None, None, n=0, outs=outs)
    for t in outs:
        assert (_host(t) == SENTINEL).all()
    for n in (1, 31, 32, 33, 32 * 9 + 13):
        st1 = _starts(random_starts(rng, sc1.Size(), n), n)
        got = pair_call(sc1, sc2, hb, 3, st1, None, n=n)
        ref = single(sc1, hb, 3, st1, n=n) + single(sc2, hb, 3, None, n=n)
        for k in range(6):
            expect_equal("n=%d" % n, "output %d" % k, got[k], ref[k])


def test_against_the_oracle(cuda_device):
    rng = np.random.default_rng(9)
    names = ("AppendixA", "glue10")
    scs = [scanner(n) for n in names]
    orcs = [Oracle(image_of(n)) for n in names]
    rows = random_rows(rng, 32 * 2 + 7, 256, ALPHA_ALL, LITERALS)
    hb = fixed_batch(rows)
    starts = [random_starts(rng, sc.Size(), hb.n) for sc in scs]
    for begin, end in MARKS:
        got = check_pair(scs[0], scs[1], hb, _flags(begin, end), starts[0], None, "oracle begin=%d end=%d" % (begin, end))
        for i in range(0, hb.n, 3):
            for k, (orc, st) in enumerate(zip(orcs, (int(starts[0][i]), None))):
                want = run_from(orc, rows[i], st, begin, end)
                bit = (int(got[3 * k][i // 32]) >> (i % 32)) & 1
                assert (bit, int(got[3 * k + 1][i]), int(got[3 * k + 2][i])) == tuple(int(x) for x in want), (names[k], i, begin, end)


def test_rounds_chained_in_place(cuda_device):
    """Four uniform rounds, each scanner's states updated in place (d_state_idx == d_start), equal one call over the whole
    strings."""
    rng = np.random.default_rng(10)
    sc1, sc2 = scanner("glue10"), scanner("AppendixA")
    n, length, rounds = 32 * 13 + 5, 1024, 4
    rows = random_rows(rng, n, length, ALPHA_ALL, LITERALS)
    whole = fixed_batch(rows)
    pieces = [fixed_batch(np.ascontiguousarray(rows[:, r * length // rounds:(r + 1) * length // rounds])) for r in range(rounds)]
    want = pair_call(sc1, sc2, whole, 3, None, None)
    s1, s2 = _starts([sc1.Initialize()] * n, n), _starts([sc2.Initialize()] * n, n)
    outs = _outputs(n) + _outputs(n)
    outs[2], outs[5] = s1, s2
    for r, hb in enumerate(pieces):
        last = r == rounds - 1
        flags = (RUN_BEGIN if r == 0 else 0) | (RUN_END if last else 0)
        use = outs if last else [None, None, s1, None, None, s2]
        got = pair_call(sc1, sc2, hb, flags, s1, s2, outs=use)
    for k in range(6):
        expect_equal("chained", "output %d" % k, got[k], want[k])


def test_noexit_in_one_scanner_only(cuda_device):
    """Every lane of a warp reaches a NoExit state of one scanner early (`foo` absorbs, `.*` is one state), while the
    other scanner's answer depends on the end of the strings: a warp that left when only one scanner was NoExit would
    get the other one's results wrong.  Both orders, and both NoExit at different times."""
    rng = np.random.default_rng(11)
    n, length = 32 * 6, 1024
    rows = random_rows(rng, n, length, b"abcdxyz hel")
    rows[:, 3:6] = np.frombuffer(b"foo", np.uint8)                      # absorbing: NoExit from byte 6
    tail = b"hello  world"
    rows[::2, length - len(tail):] = np.frombuffer(tail, np.uint8)      # AppendixA: decided by the last bytes
    late = rows.copy()
    late[:, 3:6] = np.frombuffer(b"xyz", np.uint8)
    late[:, 700:703] = np.frombuffer(b"foo", np.uint8)                  # absorbing from byte 703 only
    absorbing, appendix, all_final = scanner("absorbing"), scanner("AppendixA"), scanner("all_final")
    for label, r in (("early", rows), ("late", late)):
        hb = fixed_batch(r)
        for a, b, name in ((absorbing, appendix, "absorbing+AppendixA"), (appendix, absorbing, "AppendixA+absorbing"),
                           (all_final, appendix, "all_final+AppendixA"), (all_final, absorbing, "all_final+absorbing")):
            for begin, end in MARKS:
                got = check_pair(a, b, hb, _flags(begin, end), None, None, "%s %s begin=%d end=%d" % (label, name, begin, end))
                if name == "absorbing+AppendixA" and end:
                    # every string matches `foo`; AppendixA matches the even strings only
                    assert (got[0] == 0xFFFFFFFF).all() and (got[3] == 0x55555555).all(), (label, got[0][:2], got[3][:2])


def test_null_outputs(cuda_device):
    rng = np.random.default_rng(12)
    sc1, sc2 = scanner("glue10"), scanner("headline")
    hb = fixed_batch(random_rows(rng, 32 * 2 + 9, 128, ALPHA_ALL, LITERALS))
    st1 = random_starts(rng, sc1.Size(), hb.n)
    for subset in range(64):
        want = tuple(bool(subset >> k & 1) for k in range(6))
        check_pair(sc1, sc2, hb, 3, st1, None, "outputs %s" % (want,), want=want)
    csr = csr_batch(random_strings(rng, ALPHA_ALL, [0, 5, 100, 40], LITERALS))
    for subset in (0, 5, 42, 63):
        want = tuple(bool(subset >> k & 1) for k in range(6))
        check_pair(sc1, sc2, csr, 3, None, None, "CSR outputs %s" % (want,), want=want)


def test_bad_arguments(cuda_device):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    rng = np.random.default_rng(13)
    sc1, sc2 = scanner("glue10"), scanner("headline")
    hb = fixed_batch(random_rows(rng, 40, 64, ALPHA_ALL))
    out = _filled(64)

    def call(h1, h2, corpus, offs, fl, n, flags):
        o = out.data_ptr()
        return N.lib.pire_gpu_run_pair_batch(h1, h2, corpus, offs, fl, n, flags, None, None, o, o, o, o, o, o, _stream())

    assert call(sc1._h, sc2._h, hb.corpus_ptr(), None, 64, 40, 3) == 0
    assert call(sc1._h, sc2._h, hb.corpus_ptr(), None, 64, 40, RUN_LINES | 1) == -1
    assert call(sc1._h, sc2._h, hb.corpus_ptr(), None, 64, 40, 8) == -1
    assert call(sc1._h, sc2._h, None, None, 64, 40, 3) == -1
    assert call(None, sc2._h, hb.corpus_ptr(), None, 64, 40, 3) == -1
    assert call(sc1._h, None, hb.corpus_ptr(), None, 64, 40, 3) == -1
    host = P.Scanner(image_of("glue10"), -1)
    assert call(host._h, sc2._h, hb.corpus_ptr(), None, 64, 40, 3) == -4
    assert call(sc1._h, host._h, hb.corpus_ptr(), None, 64, 40, 3) == -4
    torch.cuda.synchronize()
    before = _host(out).copy()
    assert call(sc1._h, sc2._h, None, None, 0, 0, 3) == 0
    torch.cuda.synchronize()
    assert (_host(out) == before).all()
    pair = P.ScannerPair(sc1, sc2)
    with pytest.raises(ValueError):
        P.Runner(pair).Run(P.Batch.from_text(torch.tensor(list(b"a\nb\n"), dtype=torch.uint8, device="cuda:0"))).Matches()
    if torch.cuda.device_count() >= 2:
        other = P.Scanner(image_of("headline"), 1)
        assert call(sc1._h, other._h, hb.corpus_ptr(), None, 64, 40, 3) == -1


# -------------------------------------------------------------------------------------------------------- front ends

def test_python_pair_runner(cuda_device):
    """ScannerPair + Runner: Matches() is the OR, First() / Second() equal each scanner's own Runner, and rounds chain
    through (states1, states2) with either None."""
    import torch
    import pire_b200 as P
    rng = np.random.default_rng(14)
    sc1, sc2 = scanner("glue10"), scanner("AppendixA")
    pair = P.ScannerPair(sc1, sc2)
    n, length = 32 * 7 + 3, 512
    rows = random_rows(rng, n, length, ALPHA_ALL, LITERALS)
    dev = torch.from_numpy(rows.reshape(-1).copy()).to("cuda:0")
    batch = P.Batch(dev, fixed_len=length, n=n)
    r = P.Runner(pair).Begin().Run(batch).End()
    one, two = P.Runner(sc1).Begin().Run(batch).End(), P.Runner(sc2).Begin().Run(batch).End()
    for half, ref in ((r.First(), one), (r.Second(), two)):
        assert (half.Matches() == ref.Matches()).all() and (half.States() == ref.States()).all()
        assert (half.AcceptMasks() == ref.AcceptMasks()).all()
        assert half.AcceptedRegexps(0) == ref.AcceptedRegexps(0)
    assert (r.Matches() == (one.Matches() | two.Matches())).all() and r.Matches().any()
    # two rounds; the second scanner starts its first round from Initialize() (None)
    halves = [P.Batch(torch.from_numpy(np.ascontiguousarray(rows[:, k * 256:(k + 1) * 256]).reshape(-1)).to("cuda:0"), fixed_len=256, n=n)
              for k in (0, 1)]
    first = P.Runner(pair, (torch.full((n,), sc1.Initialize(), dtype=torch.int32, device="cuda:0"), None)).Begin().Run(halves[0])
    second = P.Runner(pair, (first.First().StateTensor(), first.Second().StateTensor())).Run(halves[1]).End()
    assert (second.First().States() == one.States()).all() and (second.Second().States() == two.States()).all()
    assert (second.Matches() == r.Matches()).all()
    # a ragged batch takes the unfused path through the same classes
    strings = random_strings(rng, ALPHA_ALL, [int(x) for x in rng.integers(0, 900, size=50)], LITERALS)
    rb = P.Batch.from_strings(strings)
    rr = P.Runner(pair).Begin().Run(rb).End()
    assert (rr.First().States() == P.Runner(sc1).Begin().Run(rb).End().States()).all()
    assert (rr.Second().States() == P.Runner(sc2).Begin().Run(rb).End().States()).all()


def test_cpp_pair_runner(tmp_path, cuda_device):
    """tests/cpp/pair_check.cpp through include/pire_gpu.hpp: Runner(pair) and Run(sc1, sc2, ...) against BatchRunner."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "pair_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pair_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    images = []
    for name in ("glue10", "headline"):
        p = tmp_path / (name + ".pire")
        p.write_bytes(W.load_image(name))
        images.append(str(p))
    for n, length, rounds in ((20_003, 1024, 4), (33, 256, 2), (1, 32, 1)):
        out = subprocess.run([exe, images[0], images[1], str(n), str(length), str(rounds), "7"], capture_output=True, text=True,
                             timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ", 0 mismatches" in out.stdout, out.stdout
