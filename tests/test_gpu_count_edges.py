"""The counting entry points off the default shapes, against the in-repo oracle: pire_gpu_count_batch (CountKernel) and
pire_gpu_count_string (CountStringKernel) on the edge images of tests/golden/edge_images.json.xz (32-bit tables, cold
starts, one-row hot sets, all-final and never-hot scanners, NoExit starts), on line batches, and on the scanners of
more than 256 regexps of tests/golden/count_images.json.xz.  The edge images are plain Scanners; the count entry
points and the oracle's count both apply TakeAction to whatever image they are given, so they are counted as they are.

As in tests/test_gpu_edges.py, every group first asserts the precondition that puts it on its path, and every output
buffer is larger than the call may write and pre-filled with a sentinel that must survive."""
import numpy as np
import pytest

from count_oracle import count_from
from refpire import oracle_count
from test_count_images import COUNT_IMAGES, count_rows_max, w_strings, want_counts
from test_edge_images import ALPHABETS, EDGE
from test_gpu_count_string import Counter
from test_gpu_edges import (EXTRA, MARKS, RUN_BEGIN, RUN_END, RUN_LINES, SENTINEL, BeginMark, Checker, HostBatch, _filled, _host,
                            _stream, cold_start_cases, csr_batch, expect_equal, expect_untouched, fixed_batch, lines_batch,
                            random_rows, random_strings, static_hot, text_of_lines, unpack_bits)
from test_gpu_parity import _text_of
from test_gpu_string import BLOCK, MIN_BLOCKS, text_buffer

pytestmark = pytest.mark.gpu

# strings drawn from each image's alphabet carry these, so that the walks reach final states
LITERALS = {
    "wide": [],
    "anchored": [b"abcd", b"abcde", b"cdabe", b"ababe"],
    "glued": [b"GET ", b"error", b"x123y"],
    "all_final": [],
    "none_hot": [b"ab" * 140, b"cd" * 139 + b"ab"],
    "absorbing": [b"foo"],
}
HOTS = {"wide": (255, 2)}
FLAG_MARKS = [0, RUN_BEGIN, RUN_END, RUN_BEGIN | RUN_END]


def reachable(sc):
    todo, seen = [sc.Initialize()], {sc.Initialize()}
    while todo:
        s = todo.pop()
        for c in list(range(256)) + [BeginMark, BeginMark + 1]:
            t = sc.Next(s, c)
            if t not in seen:
                seen.add(t)
                todo.append(t)
    return seen


def noexit(sc, s):
    """dfa_tables.cpp's noexit predicate: every byte leads back to s."""
    return all(sc.Next(s, b) == s for b in range(256))


def check_edge_precondition(name, sc, host, max_hot, tuned):
    info = sc.info()
    if name == "wide":
        assert info.states > 65536 and info.table_bytes == info.states * info.letters * 4       # 32-bit cells
    if name == "all_final":
        assert all(host.Final(s) for s in reachable(host))                                    # first_final_hot == 0
    if name == "none_hot" and not tuned:
        assert info.hot_rows == min(max_hot, 255)
        assert not any(host.Final(s) for s in static_hot(host, max_hot))                       # finals entered through the sink


def count_batches(name, rng):
    alphabet, literals = ALPHABETS[name], LITERALS[name]
    out = []
    for length in (32, 64, 1024):
        rows = random_rows(rng, 64 * 3 + 5, length, alphabet, literals)
        if literals:
            rows[1::5] = np.resize(np.frombuffer(literals[0], np.uint8), length)      # rows that stay alive to their end
        out.append(("uniform %dB" % length, fixed_batch(rows)))
    rows = random_rows(rng, 101, 47, alphabet, literals)
    out.append(("fixed_len=47 base=1", fixed_batch(rows, base=1, guard_before=alphabet[:2], guard_after=alphabet[:2])))
    strings = random_strings(rng, alphabet, [0, 0, 1, 0] + list(rng.integers(0, 400, size=300)) + [0], literals)
    out.append(("csr", csr_batch(strings + [lit for lit in literals for _ in range(3)])))       # whole matches of anchored patterns
    out.append(("lines", lines_batch(text_of_lines(rng, alphabet, literals, 600, long_every=200))))
    return out


# --------------------------------------------------------------------------- (a) count_batch on the edge images

@pytest.mark.parametrize("name", sorted(EDGE))
def test_count_batch_edge_images(name, cuda_device):
    """Uniform 32 B / 64 B / 1 KiB, a non-uniform fixed length at base 1, ragged CSR with empty strings and lines; every
    mark combination; count modes 1-3 (and 0 after Tune); max_hot 255, 3, 2, 1, static and tuned with the opposite
    marks (255 and 2 for the 32-bit table)."""
    import pire_b200 as P
    image = EDGE[name]["image"]
    host = P.Scanner(image, -1)
    rng = np.random.default_rng(sum(name.encode()) + 7)
    batches = count_batches(name, rng)
    tune_sample = random_strings(rng, ALPHABETS[name], [64] * 64, LITERALS[name])
    tune_batch = P.Batch.from_strings(tune_sample)
    chk = Checker(image, name)
    cold = {"static": 0, "tuned": 0}
    counted = 0
    for max_hot in HOTS.get(name, (255, 3, 2, 1)):
        for tuned in (False, True):
            for begin, end in MARKS:
                if not tuned and (begin, end) == MARKS[0] or tuned:
                    chk.sc = P.Scanner(image, 0)
                    chk.sc.set_max_hot(max_hot)
                    if tuned:
                        chk.sc.Tune(tune_batch, len(tune_sample), begin=not begin, end=not end)
                        assert chk.sc.info().tuned == 1
                check_edge_precondition(name, chk.sc, host, max_hot, tuned)
                if name in ("anchored", "glued") and cold_start_cases(host, tune_sample, max_hot, tuned, begin):
                    cold["tuned" if tuned else "static"] += 1
                label = "max_hot=%d %s [%s begin=%d end=%d]" % (max_hot, "tuned" if tuned else "static", name, begin, end)
                for what, hb in batches:
                    for mode in ((0, 1, 2, 3) if tuned else (1, 2, 3)):
                        chk.count(hb, begin, end, mode, "%s %s" % (what, label))
                    counted += int(chk.want(hb, "count", begin, end)[0].sum())
    assert counted > 0                                      # final states were entered
    if name in ("anchored", "glued"):
        assert cold["static"] >= 2 and cold["tuned"] >= 1, cold
    if name == "none_hot":
        want, _ = chk.want(batches[2][1], "count", False, False)
        assert want.sum() > 0                               # 1 KiB rows reach the final state, outside the hot rows


# -------------------------------------------------------------------------- (b) count_string on the edge images

def count_in_rows(c, dev, cases, flags):
    """Every case counted into a row of one buffer, launched without a synchronise; the column past the counters and
    the words past the two outputs hold the sentinel."""
    import torch
    regs = c.regs()
    counts = torch.zeros((len(cases), regs + 1), dtype=torch.int64, device="cuda:0")
    counts[:, regs] = SENTINEL
    words = torch.full((len(cases), 3), SENTINEL, dtype=torch.int32, device="cuda:0")
    for k, (off, n) in enumerate(cases):
        c.launch(dev, off, n, flags, counts[k], words[k])
    hc, hw = counts.cpu().numpy(), words.cpu().numpy().view(np.uint32)
    assert (hc[:, regs] == SENTINEL).all() and (hw[:, 2] == SENTINEL).all(), "written past the counters or the words"
    return hc[:, :regs], hw[:, :2]


def edge_text(name, size, seed):
    """Bytes of the image's alphabet with its short literals every 37 bytes; the texts from offset 0 start with a whole
    match of the anchored patterns (`abcde`, 280 bytes of `ab`)."""
    import torch
    _, host = text_buffer(size, ALPHABETS[name], [x for x in LITERALS[name] if len(x) < 32], every=37, seed=seed)
    lead = {"anchored": b"abcde", "none_hot": b"ab" * 300}.get(name, b"")
    host[:len(lead)] = np.frombuffer(lead, np.uint8)
    return torch.from_numpy(host).to("cuda:0"), host


@pytest.mark.parametrize("name", sorted(EDGE))
def test_count_string_edge_images(name, cuda_device):
    """Lengths 0..300 at alignments 0, 1, 7, 16 and 31 and one length past the one-CTA piece boundary, every mark
    combination and count mode: against the oracle's count, count_batch with n = 1 and run_string's words."""
    import pire_b200 as P
    image = EDGE[name]["image"]
    c = Counter(image)
    check_edge_precondition(name, c.sc, P.Scanner(image, -1), 255, False)
    step = 32 * BLOCK * MIN_BLOCKS
    long_n = step + 32 + 5
    dev, host = edge_text(name, long_n + 64, seed=len(name))
    cases = [(off, n) for off in (0, 1, 7, 16, 31) for n in range(0, 301, 1 if off in (0, 1) else 7)]
    corpus = np.concatenate([host[off:off + n] for off, n in cases])
    offs = np.concatenate([[0], np.cumsum([n for _, n in cases])]).astype(np.uint64)
    counted = 0
    for flags in FLAG_MARKS:
        begin, end = bool(flags & RUN_BEGIN), bool(flags & RUN_END)
        want, wfin = oracle_count(c.orc, corpus, offs, begin=begin, end=end)
        counted += int(want.sum())
        for k in range(0, len(cases), 101):
            off, n = cases[k]
            assert count_from(c.orc, host[off:off + n], None, begin, end)[0] == want[k].tolist()
        lw, lfin = oracle_count(c.orc, host[3:3 + long_n], np.array([0, long_n], np.uint64), begin=begin, end=end)
        for mode in (0, 1, 2, 3):
            c.sc.set_count_mode(mode)
            got_c, got_w = count_in_rows(c, dev, cases, flags)
            label = (name, mode, flags)
            expect_equal(str(label), "counts", got_c, want)
            expect_equal(str(label), "match words", got_w[:, 0], wfin)
            for k in range(0, len(cases), 37):
                off, n = cases[k]
                assert c.check_count(dev, off, n, flags, what=label)[1:] == (int(got_w[k, 0]), int(got_w[k, 1]))
            got = c.check_count(dev, 3, long_n, flags, what=label + ("long",))
            assert got[0] == lw[0].tolist() and got[1] == int(lfin[0]), label
    assert counted > 0


RESUME_ALL = ("anchored", "glued", "all_final", "absorbing")


@pytest.mark.parametrize("name", RESUME_ALL + ("wide",))
def test_count_string_resume_edge_images(name, cuda_device):
    """Resumed from every state (about 200 sampled states of the 32-bit table): against count_from.  Among the starts
    is a hot NoExit state, which makes the kernel skip phase 1 and count every piece from the start."""
    import pire_b200 as P
    image = EDGE[name]["image"]
    c = Counter(image)
    host = P.Scanner(image, -1)
    hot = set(static_hot(host, c.sc.info().hot_rows))
    if name == "wide":
        states = sorted(set(np.random.default_rng(5).integers(0, host.Size(), size=200).tolist()) | set(sorted(hot)[:20]))
    else:
        states = list(range(host.Size()))
    if name in ("all_final", "absorbing"):
        skipping = [s for s in states if s in hot and noexit(host, s)]
        assert skipping and any(host.Final(s) for s in skipping), "no hot NoExit start: the skip path is not reached"
    dev, text = edge_text(name, 400, seed=len(name) + 50)
    for mode in ((1, 2) if name != "wide" else (2,)):
        c.sc.set_count_mode(mode)
        for st in states:
            for flags in FLAG_MARKS:
                for off, n in ((0, 0), (3, 7), (5, 333)):
                    want, res = count_from(c.orc, text[off:off + n], st, bool(flags & RUN_BEGIN), bool(flags & RUN_END))
                    got = c.count(dev, off, n, flags, start=st)
                    assert got == (want, res[0], res[2]), (name, mode, st, flags, n, got, want, res)


# ------------------------------------------------------------------------------------------- (c) line batches

def lines_at(text, shift):
    """The lines of `text` placed `shift` bytes into a device buffer: (HostBatch, P.Batch over the same bytes)."""
    import torch
    import pire_b200 as P
    buf = np.frombuffer(bytes(shift) + text + bytes(32), np.uint8).copy()
    dev = torch.from_numpy(buf).to("cuda:0")
    b = P.Batch.from_text(dev[shift:shift + len(text)])
    hb = HostBatch(buf, base=shift, offsets=b.offsets.cpu().numpy().astype(np.uint64), lines=True)
    hb._dev = (dev, b.offsets)
    return hb, b


def edge_lines_text(rng, name, n_lines, ending):
    lines = [s.replace(b"\n", b" ") for s in random_strings(rng, ALPHABETS[name], list(rng.integers(0, 120, size=n_lines)), LITERALS[name])]
    lines[n_lines // 3] = random_strings(rng, ALPHABETS[name], [1500], LITERALS[name])[0].replace(b"\n", b" ")
    lines[n_lines // 2] = random_strings(rng, ALPHABETS[name], [40000], LITERALS[name])[0].replace(b"\n", b" ")
    for k in range(n_lines // 4, n_lines // 4 + 50):
        lines[k] = b""
    return b"\n".join(lines) + ending


def run_batch_lines(chk, hb, begin, end, label):
    """pire_gpu_run_batch with PIRE_GPU_RUN_LINES: the generic kernel, one line per lane, against the oracle."""
    from pire_b200 import _native as N
    flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0) | RUN_LINES
    bits, masks, states = _filled((hb.n + 31) // 32 + 1), _filled(hb.n + EXTRA), _filled(hb.n + EXTRA)
    N.check(N.lib.pire_gpu_run_batch(chk.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), 0, hb.n, flags, bits.data_ptr(), masks.data_ptr(),
                                     states.data_ptr(), _stream()), "run_batch lines (%s)" % label)
    f, m, s = chk.want(hb, "run", begin, end)
    hm, hs = _host(masks), _host(states)
    expect_untouched(label, "accept masks", hm, hb.n)
    expect_untouched(label, "state indices", hs, hb.n)
    expect_equal(label, "StateIndex", hs[: hb.n], s)
    expect_equal(label, "accept masks", hm[: hb.n], m)
    expect_equal(label, "match bits", unpack_bits(label, _host(bits), hb.n), f)


LINE_IMAGES = ("hf_glue10", "count_words5", "none_hot", "all_final")


@pytest.mark.parametrize("name", LINE_IMAGES)
def test_line_batches(name, cuda_device):
    """count_batch with PIRE_GPU_RUN_LINES through the C ABI and HalfFinalCount(sc, Batch.from_text(t)); on the same
    batches suffix scans, run_batch (the generic kernel) and run_lines, and run_lines after AutoSelect on the lines.
    Texts with and without a last newline, at shifts 0, 1, 7, 16 and 31, with runs of empty lines and lines longer than
    1 KiB and 32 KiB."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    image = EDGE[name]["image"] if name in EDGE else W.load_image(name)
    rng = np.random.default_rng(sum(name.encode()))
    chk = Checker(image, name)
    if name in EDGE:
        check_edge_precondition(name, chk.sc, P.Scanner(image, -1), 255, False)
    for ending in (b"\n", b""):
        text = edge_lines_text(rng, name, 600, ending) if name in EDGE else _text_of(rng, 600, ending)[0]
        assert max(len(x) for x in text.split(b"\n")) > 32 * 1024
        for shift in (0, 1, 7, 16, 31):
            hb, batch = lines_at(text, shift)
            assert hb.n == text.count(b"\n") + (0 if text.endswith(b"\n") else 1)
            label = "%s ending=%r shift=%d" % (name, ending, shift)
            for begin, end in MARKS:
                lab = "%s [begin=%d end=%d]" % (label, begin, end)
                for mode in (1, 2, 3):
                    chk.count(hb, begin, end, mode, lab)
                for shortest in (False, True):
                    chk.prefix(hb, shortest, begin, end, lab, suffix=True)
                for v in (1, 2, 4):
                    chk.sc.set_variant(v)
                    run_batch_lines(chk, hb, begin, end, "%s variant=%d" % (lab, v))
                    chk.run(hb, begin, end, "%s variant=%d" % (lab, v))
                chk.sc.set_variant(0)
            chk.sc.set_count_mode(0)
            for begin, end in ((True, True), (False, False)):
                res = P.HalfFinalCount(chk.sc, batch, begin=begin, end=end)
                want, wfin = chk.want(hb, "count", begin, end)
                expect_equal(label + " HalfFinalCount", "counts", res.counts, want)
                expect_equal(label + " HalfFinalCount", "final", res.final, wfin.astype(bool))
    # AutoSelect times the variants on the line batch (pire_gpu_run_batch with RUN_LINES); run_lines keeps its results
    hb, batch = lines_at(text, 7)
    sc = P.Scanner(image, 0)
    sc.AutoSelect(batch)
    chk.sc = sc
    for begin, end in MARKS:
        chk.run(hb, begin, end, "%s after AutoSelect variant=%d" % (name, sc.info().variant))


# ---------------------------------------------------------------------------------- (d) past 256 regexps

def w_buffer(rng, size, plants):
    """Lowercase bytes with 'w' + id written at each (offset, id) of `plants`: (device tensor, host array)."""
    import torch
    host = rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8), size=size)
    for at, i in plants:
        host[at:at + 4] = np.frombuffer(b"w%03d" % i, np.uint8)
    return torch.from_numpy(host).to("cuda:0"), host


@pytest.mark.parametrize("name", sorted(COUNT_IMAGES))
def test_many_regexps(name, cuda_device):
    """256, 257 and 300 regexps: count_string (its u32 rows per warp up to kCountRowsMax regexps, the u64 counters
    directly past it) in rows, chained and over 2 MB, modes AUTO and PACKED (the accept lists above 16 regexps);
    count_batch on a CSR batch (rows of 257 and more u32); accept_sets of 9 and more words; run_batch accept masks."""
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    e = COUNT_IMAGES[name]
    k = e["regexps"]
    c = Counter(e["image"])
    assert c.regs() == k and c.sc.info().regexps == k
    shared_rows = k <= count_rows_max()
    rng = np.random.default_rng(k)

    # count_string: many short texts, each ending one match, launched into rows without a synchronise
    ids = [k - 1, 0, 1, 2, 3, 4, 31, 32, 255] + ([256] if k > 256 else []) + list(rng.integers(0, k, size=60))
    gaps = rng.integers(4, 9000, size=len(ids))
    gaps[::7] = 150_000
    pos = np.cumsum(gaps + 4)
    plants = list(zip(pos.tolist(), ids))
    dev, host = w_buffer(rng, int(pos[-1]) + 64 + 64, plants)
    cases = [(int(prev) + 4, int(at) + 4 + int(x) - (int(prev) + 4)) for (prev, at, x) in
             zip([0] + pos[:-1].tolist(), pos.tolist(), rng.integers(0, 3, size=len(ids)))]
    corpus = np.concatenate([host[off:off + n] for off, n in cases])
    offs = np.concatenate([[0], np.cumsum([n for _, n in cases])]).astype(np.uint64)
    want, wfin = oracle_count(c.orc, corpus, offs, begin=False, end=False)
    assert (want.sum(axis=1) == 1).all() and want[:, 256:].any() == (k > 256)          # one match each, ids past 255 too
    # a 2 MB text whose only match lies deep in the grid's pieces
    big_n = 2_000_003
    big_dev, big = w_buffer(rng, big_n + 64, [(1_999_000, k - 1)])
    big_want, big_fin = oracle_count(c.orc, big[1:1 + big_n], np.array([0, big_n], np.uint64), begin=False, end=False)
    assert big_want[0, k - 1] == 1
    for mode in (0, 2):
        c.sc.set_count_mode(mode)
        label = "%s mode=%d shared_rows=%d" % (name, mode, shared_rows)
        got_c, got_w = count_in_rows(c, dev, cases, 0)
        expect_equal(label, "counts", got_c, want)
        expect_equal(label, "match words", got_w[:, 0], wfin)
        for j in range(0, len(cases), 9):
            off, n = cases[j]
            assert c.check_count(dev, off, n, 0, what=label)[0] == want[j].tolist()
        for j in (1, 2, 3):
            off, n = cases[j]
            assert count_from(c.orc, host[off:off + n], None, False, False)[0] == want[j].tolist()
            mid = c.sc.Initialize()
            for b in host[off:off + n // 2]:
                mid = c.sc.Next(mid, int(b))
            rest, res = count_from(c.orc, host[off + n // 2:off + n], mid, False, True)
            assert c.count(dev, off + n // 2, n - n // 2, RUN_END, start=mid) == (rest, res[0], res[2]), (label, j)
        one = c.check_count(big_dev, 1, big_n, 0, what=label + " 2 MB")
        assert one[0] == big_want[0].tolist() and one[1] == int(big_fin[0])
        assert c.check_count(big_dev, 1, big_n, RUN_BEGIN | RUN_END, what=label + " 2 MB marks")[0] == \
            oracle_count(c.orc, big[1:1 + big_n], np.array([0, big_n], np.uint64))[0][0].tolist()
        # chained through one state word and one counts buffer, cut inside the match too
        for cuts in ([0, 1_000_000, 1_999_001, 1_999_003, big_n], [0, 17, 17, 500_000, 1_999_000, big_n]):
            counts = torch.zeros(k + 1, dtype=torch.int64, device="cuda:0")
            counts[k] = SENTINEL
            words = torch.full((64,), SENTINEL, dtype=torch.int32, device="cuda:0")
            state = words.data_ptr() + 4
            for j in range(len(cuts) - 1):
                N.check(N.lib.pire_gpu_count_string(c.sc._h, big_dev.data_ptr() + 1 + cuts[j], cuts[j + 1] - cuts[j], 0,
                                                    None if j == 0 else state, counts.data_ptr(), words.data_ptr(), state, _stream()),
                        "pire_gpu_count_string")
            hc, w = counts.cpu().numpy(), words.cpu().numpy().view(np.uint32)
            assert hc[k] == SENTINEL and (w[2:] == SENTINEL).all()
            assert (hc[:k].tolist(), int(w[0]), int(w[1])) == one, (label, cuts)

    # count_batch, run_batch and accept_sets on a CSR batch
    strings = w_strings(rng, k, 3000, 120)
    hb = csr_batch(strings)
    chk = Checker(e["image"], name)
    want_b, _ = chk.want(hb, "count", False, False)
    assert (want_b == want_counts(strings, k)).all() and want_b[:, 256:].any() == (k > 256)
    for mode in (0, 1, 2, 3):
        chk.count(hb, False, False, mode, "%s csr" % name)
    chk.count(hb, True, True, 1, "%s csr" % name)
    chk.run(hb, False, False, "%s csr" % name)                   # masks against the oracle's (ids below 32)
    words_per = (k + 31) // 32
    assert N.lib.pire_gpu_accept_words(c.sc._h) == words_per and (words_per >= 9) == (k > 256)
    masks, states = _filled(hb.n + EXTRA), _filled(hb.n + EXTRA)
    N.check(N.lib.pire_gpu_run_batch(c.sc._h, hb.corpus_ptr(), hb.offsets_ptr(), 0, hb.n, 0, None, masks.data_ptr(), states.data_ptr(),
                                     _stream()), "run_batch")
    sets = _filled(hb.n * words_per + EXTRA)
    N.check(N.lib.pire_gpu_accept_sets(c.sc._h, states.data_ptr(), hb.n, sets.data_ptr(), _stream()), "accept_sets")
    hs, hm, hset = _host(states)[: hb.n], _host(masks)[: hb.n], _host(sets)
    expect_untouched(name, "accept sets", hset, hb.n * words_per)
    rows = hset[: hb.n * words_per].reshape(hb.n, words_per)
    high = 0
    for i in range(hb.n):
        got = [r for r in range(words_per * 32) if (int(rows[i, r // 32]) >> (r % 32)) & 1]
        acc = c.sc.AcceptedRegexps(int(hs[i]))
        assert got == acc, (name, i, got, acc)
        assert int(hm[i]) == sum(1 << r for r in acc if r < 32), (name, i, int(hm[i]), acc)
        high += any(r >= 32 for r in acc)
    assert high > 0                                           # strings whose only accepted id is past the mask's 32 bits
