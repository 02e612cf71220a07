"""pire_gpu_match_ends_string: where the HalfFinalScanner matches end in one string over the whole grid.

The independent answer is a positions walk on the in-repo oracle (ends_from below): count_oracle.count_from's loop,
recording (position, id) at each TakeAction instead of counting it.  Large texts are checked against
pire_gpu_count_string, an entry point tested on its own: the per-id histogram of all entries, and of the entries up to
a cut point against a count of the text up to there.  Every output buffer carries sentinels below the incoming
*d_found and past the capacity, and they must survive."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN_COUNTS, ROOT
from string_oracle import BEGIN_MARK, END_MARK, StringWalk
from test_count_images import COUNT_IMAGES, w_text
from test_edge_images import ALPHABETS, EDGE
from test_gpu_count_string import MARKS, RUN_BEGIN, RUN_END, Counter, _start_word, _stream
from test_gpu_string import PRINTABLE, SENTINEL, glue10, text_buffer

pytestmark = pytest.mark.gpu

SENTINEL64 = 0x5A5A5A5A5A5A5A5A
GUARD = 64                      # sentinel entries past the capacity
LITERALS = {"anchored": [b"abcd", b"abcde"], "glued": [b"GET ", b"error", b"x123y"], "none_hot": [b"ab" * 140],
            "absorbing": [b"foo"]}


def ends_from(orc, text, start=None, begin=True, end=True, base=0):
    """count_oracle.count_from's walk recording (base + bytes consumed, id) at every TakeAction, in walk order: the
    entries pire_gpu_match_ends_string must write.  Returns (ends u64, ids u32, StringWalk result)."""
    w = StringWalk(orc, start)
    ends, ids = [], []
    if not w.valid:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint32), w.result()
    lib, sc = w._lib, w._sc
    buf = (C.c_uint64 * 4096)()
    lists = {}

    def take(st, pos):
        lst = lists.get(st)
        if lst is None:
            lst = [int(buf[i]) for i in range(min(lib.pire_oracle_accepted(sc, st, buf, 4096), 4096))] \
                if lib.pire_oracle_final(sc, st) else []
            lists[st] = lst
        for i in lst:
            ends.append(base + pos)
            ids.append(i)

    if start is None:
        take(w._st, 0)
    if begin:
        w._st = lib.pire_oracle_step(sc, w._st, BEGIN_MARK)
        take(w._st, 0)
    text = np.asarray(text, dtype=np.uint8)
    for k, ch in enumerate(text.tolist()):
        w._st = lib.pire_oracle_step(sc, w._st, ch)
        take(w._st, k + 1)
    if end:
        w._st = lib.pire_oracle_step(sc, w._st, END_MARK)
        take(w._st, len(text))
    return np.array(ends, np.uint64), np.array(ids, np.uint32), w.result()


class Ends(Counter):
    """Counter (count_string, run_string) with the match-ends entry point."""

    def launch_ends(self, dev, off, n, flags, ends, ids, capacity, found, words=None, start_ptr=None, base=0, stream=None):
        from pire_b200 import _native as N
        text = None if dev is None else dev.data_ptr() + off
        N.check(N.lib.pire_gpu_match_ends_string(self.sc._h, text, n, flags, start_ptr, base,
                                                 None if ends is None else ends.data_ptr(), None if ids is None else ids.data_ptr(),
                                                 capacity, found.data_ptr(), None if words is None else words.data_ptr(),
                                                 None if words is None else words.data_ptr() + 4, stream or _stream()),
                "pire_gpu_match_ends_string")

    def ends(self, dev, off, n, flags, start=None, base=0, capacity=None, below=3):
        """One call into buffers whose first `below` entries precede the incoming *d_found, with GUARD sentinel entries
        past `capacity` (default: room for all).  -> (ends, ids, found, match, state); the sentinels must survive."""
        import torch
        if capacity is None:
            capacity = below + self.total(dev, off, n, flags, start)
        ends = torch.full((capacity + GUARD,), SENTINEL64, dtype=torch.int64, device="cuda:0")
        ids = torch.full((capacity + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0")
        found = torch.tensor([below], dtype=torch.int64, device="cuda:0")
        words = torch.full((64,), SENTINEL, dtype=torch.int32, device="cuda:0")
        st = None if start is None else _start_word(start)
        self.launch_ends(dev, off, n, flags, ends, ids, capacity, found, words, None if st is None else st.data_ptr(), base)
        e = ends.cpu().numpy().view(np.uint64)
        i = ids.cpu().numpy().view(np.uint32)
        w = words.cpu().numpy().view(np.uint32)
        got = int(found.item()) - below
        top = min(below + got, capacity)
        assert (e[:below] == SENTINEL64).all() and (i[:below] == SENTINEL).all(), "written below the incoming *d_found"
        assert (e[top:] == SENTINEL64).all() and (i[top:] == SENTINEL).all(), "written past the entries or the capacity"
        assert (w[2:] == SENTINEL).all(), "written past the match and state words"
        return e[below:top], i[below:top], got, int(w[0]), int(w[1])

    def total(self, dev, off, n, flags, start=None):
        """The number of entries, from count_string."""
        return sum(self.count(dev, off, n, flags, start)[0])

    def check(self, dev, host, off, n, flags, start=None, base=0, what=""):
        """One call against the oracle walk, count_string and run_string."""
        e, i, found, match, state = self.ends(dev, off, n, flags, start, base)
        we, wi, res = ends_from(self.orc, host[off:off + n], start, bool(flags & RUN_BEGIN), bool(flags & RUN_END), base)
        assert found == len(we) and (e == we).all() and (i == wi).all(), (what, off, n, flags, start, found, len(we))
        assert (match, state) == (res[0], res[2]), (what, off, n, flags, start)
        counts, cmatch, cstate = self.count(dev, off, n, flags, start)
        assert np.bincount(i, minlength=self.regs()).tolist() == counts and (match, state) == (cmatch, cstate), what
        return e, i


# --------------------------------------------------------------------------- (a) golden counts

def test_golden_counts(cuda_device):
    """The count_ut.cpp HalfFinal strings: entries equal the oracle walk, and their histogram the fixture counts."""
    import torch
    for case in GOLDEN_COUNTS:
        for max_hot in (255, 3):
            c = Ends(case.image, max_hot=max_hot)
            for s, want, fin in zip(case.strings, case.counts, case.final):
                dev = torch.frombuffer(bytearray(s + b"\0" * 32), dtype=torch.uint8).to("cuda:0")
                host = np.frombuffer(s, np.uint8)
                e, i = c.check(dev, host, 0, len(s), RUN_BEGIN | RUN_END, what=(case, max_hot, s))
                assert np.bincount(i, minlength=c.regs()).tolist() == want and c.ends(dev, 0, len(s), 3)[3] == fin


# --------------------------------------------------------------------------- (b) short lengths and alignments

def test_short_lengths_all_alignments(cuda_device):
    """Lengths 0..300 at all 32 alignments, the four mark combinations, on hf_glue10: every case appended to one buffer
    through one *d_found with no synchronise, case k at base 1000 k."""
    import torch
    from pire_b200 import workloads as W
    c = Ends(W.load_image("hf_glue10"))
    _, plants = glue10()
    dev, host = text_buffer(400, PRINTABLE, plants, every=41, seed=41)
    cases = [(off, n) for off in range(32) for n in range(0, 301, 1 if off in (0, 1, 17) else 7)]
    for flags in MARKS:
        want = [ends_from(c.orc, host[off:off + n], None, bool(flags & RUN_BEGIN), bool(flags & RUN_END), 1000 * k)
                for k, (off, n) in enumerate(cases)]
        total = sum(len(w[0]) for w in want)
        ends = torch.full((total + GUARD,), SENTINEL64, dtype=torch.int64, device="cuda:0")
        ids = torch.full((total + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0")
        found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
        words = torch.full((len(cases), 2), SENTINEL, dtype=torch.int32, device="cuda:0")
        for k, (off, n) in enumerate(cases):
            c.launch_ends(dev, off, n, flags, ends, ids, total, found, words[k], base=1000 * k)
        e = ends.cpu().numpy().view(np.uint64)
        i = ids.cpu().numpy().view(np.uint32)
        w = words.cpu().numpy().view(np.uint32)
        assert int(found.item()) == total
        assert (e[:total] == np.concatenate([x[0] for x in want])).all(), flags
        assert (i[:total] == np.concatenate([x[1] for x in want])).all(), flags
        assert (e[total:] == SENTINEL64).all() and (i[total:] == SENTINEL).all()
        assert w.tolist() == [[x[2][0], x[2][2]] for x in want]
        assert total > 100                                  # matches were found


# --------------------------------------------------------------------------- (c) every state as a start

@pytest.mark.parametrize("name", ["golden", "absorbing", "glued"])
def test_every_state_as_start(name, cuda_device):
    """From every state of a small scanner, hot NoExit starts (which skip the locate phase) among them; starts at or
    past Size() write nothing, leave *d_found as it was and report 0 / 0xFFFFFFFF."""
    from test_gpu_count_edges import noexit
    image = GOLDEN_COUNTS[0].image if name == "golden" else EDGE[name]["image"]
    alphabet = PRINTABLE + b"aaaabbbb" if name == "golden" else ALPHABETS[name] + b"".join(LITERALS[name])
    c = Ends(image)
    dev, host = text_buffer(400, alphabet, seed=42)
    if name != "golden":                                    # every state hot, one of them NoExit
        assert c.sc.info().hot_rows >= c.sc.Size() and any(noexit(c.sc, s) for s in range(c.sc.Size()))
    for st in range(c.sc.Size()):
        for flags in MARKS:
            for off, n in ((0, 0), (3, 7), (5, 333)):
                c.check(dev, host, off, n, flags, start=st, base=17, what=(name, st))
    for st in (c.sc.Size(), c.sc.Size() + 1, 0xFFFFFFFF):
        for flags in MARKS:
            e, i, found, match, state = c.ends(dev, 0, 300, flags, start=st, capacity=8)
            assert (len(e), found, match, state) == (0, 0, 0, 0xFFFFFFFF)


# --------------------------------------------------------------------------- (d) chains

def test_chains_equal_one_call(cuda_device):
    """Pieces of 0, 1, 31, 33 and a few thousand bytes, running base, no synchronise: byte for byte the arrays of one
    call over the concatenation; also through StringMatchEnds, resumed from a state, and against count_string."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    _, plants = glue10()
    dev, host = text_buffer(3_000_064, PRINTABLE, plants, every=307, seed=43)
    for name in ("hf_glue10", "count_words5"):
        c = Ends(W.load_image(name))
        n = 1_000_003 if name == "hf_glue10" else 200_001
        cuts = [0, 0, 1, 32, 32, 65, 3000, 7777, n // 2, n]
        for flags in (RUN_BEGIN | RUN_END, 0, RUN_END):
            one_e, one_i, total, match, state = c.ends(dev, 1, n, flags, below=0)
            ends = torch.full((total + GUARD,), SENTINEL64, dtype=torch.int64, device="cuda:0")
            ids = torch.full((total + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0")
            found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
            words = torch.full((2,), SENTINEL, dtype=torch.int32, device="cuda:0")
            state_ptr = words.data_ptr() + 4
            for k in range(len(cuts) - 1):
                f = (flags & RUN_BEGIN if k == 0 else 0) | (flags & RUN_END if k == len(cuts) - 2 else 0)
                c.launch_ends(dev, 1 + cuts[k], cuts[k + 1] - cuts[k], f, ends, ids, total, found, words,
                              None if k == 0 else state_ptr, base=cuts[k])
            e = ends.cpu().numpy().view(np.uint64)
            i = ids.cpu().numpy().view(np.uint32)
            assert int(found.item()) == total and (e[:total] == one_e).all() and (i[:total] == one_i).all(), (name, flags)
            assert (e[total:] == SENTINEL64).all() and (i[total:] == SENTINEL).all()
            assert [int(x) for x in words.cpu().numpy().view(np.uint32)] == [match, state]
            assert np.bincount(one_i, minlength=c.regs()).tolist() == c.count(dev, 1, n, flags)[0]
        # the Python front end: the same pieces, and a run resumed from the state the first half reached
        e0, i0, total0, match0, state0 = c.ends(dev, 1, n, RUN_BEGIN | RUN_END, below=0)
        m = P.StringMatchEnds(c.sc, total0).Begin()
        for lo, hi in zip(cuts, cuts[1:]):
            m.Run(dev[1 + lo:1 + hi])
        m.End()
        assert m.Found() == total0 and (m.Ends() == e0).all() and (m.Ids() == i0).all() and (m.Final(), m.State()) == (bool(match0), state0)
        assert m.EndsTensor().shape[0] == total0 and m.IdsTensor().dtype == torch.int32 and m.FoundTensor().dtype == torch.int64
        half = P.StringMatchEnds(c.sc, total0).Begin().Run(dev[1:1 + n // 2])
        rest = P.StringMatchEnds(c.sc, total0, half.State()).Run(dev[1 + n // 2:1 + n]).End()
        assert (np.concatenate([half.Ends(), rest.Ends() + n // 2]) == e0).all()
        assert (np.concatenate([half.Ids(), rest.Ids()]) == i0).all() and rest.State() == state0


# --------------------------------------------------------------------------- (e) scale

def planted(nbytes):
    """tools/string_bench.py's text: 1 KiB synthetic strings with the glue10 and headline plants, back to back."""
    import torch
    from pire_b200 import workloads as W
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(nbytes // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    return dev


def device_ends(c, dev, n, flags, capacity, base=0, start_ptr=None):
    """One call into device buffers of `capacity`; -> (ends, ids, found) as device tensors (no sentinels: large)."""
    import torch
    ends = torch.empty(capacity, dtype=torch.int64, device="cuda:0")
    ids = torch.empty(capacity, dtype=torch.int32, device="cuda:0")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    c.launch_ends(dev, 0, n, flags, ends, ids, capacity, found, start_ptr=start_ptr, base=base)
    return ends, ids, int(found.item())


@pytest.mark.parametrize("mib", [64, 1024])
def test_planted_text_at_scale(mib, cuda_device):
    """64 MiB and 1 GiB of planted text with hf_glue10, count_words5 and headline: the ends ascend, the histogram is
    count_string's, the entries up to random cut points are count_string's of the text up to there, and the first
    300 KB equal the oracle walk."""
    import torch
    from pire_b200 import workloads as W
    n = mib * 2 ** 20 - 5
    text = planted(mib * 2 ** 20)
    head = text[:300_000].cpu().numpy()
    rng = np.random.default_rng(44 + mib)
    base = 123_456_789_012
    for name in ("hf_glue10", "count_words5", "headline"):
        c = Ends(W.load_image(name))
        counts = c.count(text, 0, n, RUN_BEGIN | RUN_END)
        total = sum(counts[0])
        assert total > 0 or name == "headline"              # hello\s+w.+d$ matches only a text that begins with it
        ends, ids, found = device_ends(c, text, n, RUN_BEGIN | RUN_END, total, base)
        assert found == total
        ends -= base
        assert bool((ends[1:] >= ends[:-1]).all()) and bool((ends >= 0).all()) and bool((ends <= n).all())
        assert torch.bincount(ids.long(), minlength=c.regs()).tolist() == counts[0]
        for p in [int(x) for x in rng.integers(1, n, size=4)] + [300_000]:
            k = int(torch.searchsorted(ends, torch.tensor([p], dtype=torch.int64, device="cuda:0"), right=True).item())
            want = c.count(text, 0, p, RUN_BEGIN)[0]
            assert torch.bincount(ids[:k].long(), minlength=c.regs()).tolist() == want, (name, p)
        we, wi, _ = ends_from(c.orc, head, None, True, False)
        k = len(we)
        assert (ends[:k].cpu().numpy().view(np.uint64) == we).all() and (ids[:k].cpu().numpy().view(np.uint32) == wi).all()
        assert k == len(ends) or int(ends[k]) > 300_000
        del ends, ids
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------- (f) overflow

def test_capacity_below_total(cuda_device):
    """The written entries are the first `capacity` of a full-capacity call, and *d_found is the full total; the
    sentinels past the capacity survive."""
    from pire_b200 import workloads as W
    text = planted(16 * 2 ** 20)
    host = text.cpu().numpy()
    for name in ("hf_glue10", "count_words5"):
        c = Ends(W.load_image(name))
        n = len(host) - 3
        full_e, full_i, total, match, state = c.ends(text, 3, n, RUN_BEGIN | RUN_END, below=0)
        for capacity in (0, 1, 7, total // 3, total - 1):
            e, i, found, m, s = c.ends(text, 3, n, RUN_BEGIN | RUN_END, capacity=capacity, below=min(capacity, 2))
            below = min(capacity, 2)
            assert found == total and (m, s) == (match, state)
            assert (e == full_e[: capacity - below]).all() and (i == full_i[: capacity - below]).all(), (name, capacity)


def test_past_2_32_entries(cuda_device):
    """count_words5 on 4 GiB of planted text with 2^20 entries of room: the u64 total passes 2^32 and equals the sum of
    count_string's counters, and the entries written are the first of the answer (checked against a 1 MiB call)."""
    import torch
    from pire_b200 import workloads as W
    n = 4 * 2 ** 30
    text = planted(n)
    try:
        c = Ends(W.load_image("count_words5"))
        total = sum(c.count(text, 0, n, RUN_BEGIN | RUN_END)[0])
        ends, ids, found = device_ends(c, text, n, RUN_BEGIN | RUN_END, 2 ** 20)
        assert found == total and found > 2 ** 32, found
        small_e, small_i, small = device_ends(c, text, 2 ** 20, RUN_BEGIN, 2 ** 20)
        k = min(small, 2 ** 20)
        assert bool((ends[:k] == small_e[:k]).all()) and bool((ids[:k] == small_i[:k]).all())
    finally:
        del text
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------- (g) edge and large scanners

@pytest.mark.parametrize("name", sorted(EDGE))
def test_edge_images(name, cuda_device):
    """The edge images (32-bit tables, cold starts, one-row hot sets, the all-final scanner where every step emits) with
    hot sets of 255, 2 and 1 rows, against the oracle walk."""
    rng = np.random.default_rng(sum(name.encode()))
    alphabet = ALPHABETS[name]
    host = rng.choice(np.frombuffer(alphabet, np.uint8), size=70_000)
    for k, at in enumerate(range(100, len(host) - 300, 997)):
        lits = LITERALS.get(name)
        if lits:
            lit = np.frombuffer(lits[k % len(lits)], np.uint8)
            host[at:at + len(lit)] = lit
    import torch
    dev = torch.from_numpy(host).to("cuda:0")
    for max_hot in (255, 2, 1):
        c = Ends(EDGE[name]["image"], max_hot=max_hot)
        for off, n in ((0, 0), (1, 17), (5, 300), (3, 66_000)):
            for flags in (RUN_BEGIN | RUN_END, 0):
                e, _ = c.check(dev, host, off, n, flags, base=max_hot, what=(name, max_hot))
                if name == "all_final" and n:
                    assert len(e) >= n and set(range(1, n + 1)) <= set((e - max_hot).tolist())


@pytest.mark.parametrize("name", sorted(COUNT_IMAGES))
def test_many_regexps(name, cuda_device):
    """256, 257 and 300 regexps: ids past 255 come out right."""
    import torch
    image = COUNT_IMAGES[name]
    k = image["regexps"]
    rng = np.random.default_rng(k)
    c = Ends(image["image"])
    assert c.regs() == k
    seen = []
    # a text's [a-z]* prefix ends at most one match: short texts each planted with one id, and one whose only match lies
    # in the last pieces of the grid
    texts = [(int(rng.integers(0, 3000)), [i]) for i in [k - 1, 0, 255, 31, 32] + list(range(256, k, 7)) + list(rng.integers(0, k, 20))]
    for length, ids in texts + [(300_000, [k - 1])]:
        host = w_text(rng, length + 4 + 40, ids, plant_at=[length])
        dev = torch.from_numpy(host).to("cuda:0")
        for flags in (RUN_BEGIN | RUN_END, 0):
            _, i = c.check(dev, host, 0, len(host), flags, what=(name, length, ids))
            seen += i.tolist()
    assert (max(seen) >= 256) == (k > 256) and k - 1 in seen


# --------------------------------------------------------------------------- (h) bad arguments and the front ends

def test_arguments_and_zero_bytes(cuda_device):
    import torch
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    c = Ends(W.load_image("hf_glue10"))
    dev = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    ends = torch.full((8,), SENTINEL64, dtype=torch.int64, device="cuda:0")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    f = N.lib.pire_gpu_match_ends_string
    for flags in (4, 8, 1 << 31, RUN_BEGIN | 4):
        assert f(c.sc._h, dev.data_ptr(), 10, flags, None, 0, ends.data_ptr(), None, 8, found.data_ptr(), None, None, _stream()) == -1
    assert f(c.sc._h, dev.data_ptr(), 10, 0, None, 0, ends.data_ptr(), None, 8, None, None, None, _stream()) == -1
    assert f(c.sc._h, None, 1, 0, None, 0, ends.data_ptr(), None, 8, found.data_ptr(), None, None, _stream()) == -1
    assert f(None, dev.data_ptr(), 1, 0, None, 0, ends.data_ptr(), None, 8, found.data_ptr(), None, None, _stream()) == -1
    assert int(found.item()) == 0 and (ends.cpu().numpy().view(np.uint64) == SENTINEL64).all()
    host = np.zeros(64, np.uint8)
    for flags in MARKS:
        c.check(None, host, 0, 0, flags, base=5, what="empty")
        c.check(dev, host, 0, 0, flags, what="empty")
    # NULL ends or ids: the other array is still written, and *d_found counts
    _, plants = glue10()
    dev, host = text_buffer(100_064, PRINTABLE, plants, every=211, seed=45)
    want_e, want_i, total, _, _ = c.ends(dev, 0, 100_000, 3, below=0)
    for keep in ("ends", "ids"):
        arr = torch.full((total,), -1, dtype=torch.int64 if keep == "ends" else torch.int32, device="cuda:0")
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda:0")
        c.launch_ends(dev, 0, 100_000, 3, arr if keep == "ends" else None, arr if keep == "ids" else None, total, cnt)
        got = arr.cpu().numpy().view(np.uint64 if keep == "ends" else np.uint32)
        assert int(cnt.item()) == total and (got == (want_e if keep == "ends" else want_i)).all()


def test_two_streams_one_handle(cuda_device):
    import torch
    from pire_b200 import workloads as W
    _, plants = glue10()
    c = Ends(W.load_image("hf_glue10"))
    n = 16 * 2 ** 20
    texts = [text_buffer(n + 64, PRINTABLE, p, every=e, seed=s)[0] for p, e, s in ((plants, 10_007, 46), (plants[::-1], 7_777, 47))]
    want = [c.ends(t, 0, n, RUN_BEGIN | RUN_END, below=0) for t in texts]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    bufs = [(torch.empty(2 * len(w[0]), dtype=torch.int64, device="cuda:0"), torch.empty(2 * len(w[0]), dtype=torch.int32, device="cuda:0"),
             torch.zeros(1, dtype=torch.int64, device="cuda:0")) for w in want]
    torch.cuda.synchronize()
    for rep in range(2):
        for s, t, (e, i, f), w in zip(streams, texts, bufs, want):
            c.launch_ends(t, 0, n, RUN_BEGIN | RUN_END, e, i, 2 * len(w[0]), f, base=rep * n, stream=s.cuda_stream)
    torch.cuda.synchronize()
    for (e, i, f), w in zip(bufs, want):
        assert int(f.item()) == 2 * len(w[0])
        assert (e.cpu().numpy().view(np.uint64) == np.concatenate([w[0], w[0] + n])).all()
        assert (i.cpu().numpy().view(np.uint32) == np.concatenate([w[1], w[1]])).all()


def test_cpp_string_match_ends(tmp_path, cuda_device):
    """tests/cpp/match_ends_check.cpp through include/pire_gpu.hpp's StringMatchEnds: one call, a chain and a resumed
    run write the same entries, and their histogram is StringCounter's."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "match_ends_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "match_ends_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    for name in ("hf_glue10", "count_words5"):
        image = tmp_path / (name + ".pire")
        image.write_bytes(W.load_image(name))
        for n, seed in ((10_000_019, 1), (1000, 2), (0, 3)):
            out = subprocess.run([exe, str(image), str(n), str(seed)], capture_output=True, text=True, timeout=300)
            assert out.returncode == 0, out.stdout + out.stderr
            assert ": 0 mismatches" in out.stdout
