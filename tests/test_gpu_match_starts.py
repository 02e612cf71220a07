"""pire_gpu_match_starts_string / _batch: the leftmost start of every match-ends entry, walked leftwards through a
reversed scanner.

The independent answer is the in-repo oracle's LongestSuffix (oracle_suffix, pinned to the reference) on the entry's
own regexp's reversed image alone, over [lower_k, end_k): BeginMark when lower_k is the text's start under BEGIN, and
for an entry at the text's end under END the longer of the walks without and with EndMark.  With d_ids == NULL it is
plain LongestSuffix on the glued reversed image.  The open flag is checked by walking the same image with
pire_oracle_run and asking whether a final state is still reachable (pire_oracle_step over every letter).  The ends come
from pire_gpu_match_ends_string / _batch_from on the forward images.  Every output buffer carries sentinels below
*d_first and past the processed range, and they must survive."""
import ctypes as C

import numpy as np
import pytest

from refpire import Oracle, oracle_suffix
from start_images import START_IMAGES
from string_oracle import BEGIN_MARK, END_MARK, _lib

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
NO_START = 0xFFFFFFFFFFFFFFFF
SENT64 = 0x5A5A5A5A5A5A5A5A
SENT8 = 0xA5
GUARD = 16
ALPHABET = b"abxyzEeGTrorkz0123456789 \t-:/.()ABCDEFGHIJKLMNOPQRSTUVWXYZhlowdeftiupsmn"
PLANTS = {
    "glue10": [b"ABCDEFGHIJKLMNOPQRSTUVWXYZ", b"XABCDEFGHIJKLMNOPQRSTUVWXYZ", b"(555) 123-4567", b"hello \t world",
               b"error", b"fatal", b"https://", b"GET ", b"timeout", b"http://"],
    "edges": [b"GET ", b"timeout", b"error", b"errorerror"],
    "never": [b"a", b"b", b"ab", b"\n"],
    "empty": [b"xxx", b"x"],
    "utf8_ci": ["привет".encode("utf-8"), b"ERROR", b"eRrOr"],
    "lit40": [b"k%02dz" % i for i in range(40)],
    "words": [b"abc", b"hello", b"zz"],
}


def _scanner(image):
    import pire_b200 as P
    return P.Scanner(image, 0)


class Case:
    """One pattern set: GPU handles of its forward and glued reversed images, oracles of the reversed ones."""
    _cache = {}

    def __new__(cls, name):
        if name not in cls._cache:
            c = object.__new__(cls)
            e = START_IMAGES[name]
            c.name = name
            c.fwd = _scanner(e["forward"])
            c.rev = _scanner(e["reversed"])
            c.glued = Oracle(e["reversed"])
            c.single = [Oracle(img) for img in e["per_regexp"]]
            c._live = {}
            cls._cache[name] = c
        return cls._cache[name]

    def live(self, orc):
        """The oracle states of `orc` from which some continuation (bytes and marks) reaches a final state."""
        key = id(orc)
        if key not in self._live:
            lib, sc = _lib(), C.byref(orc._sc)
            init = lib.pire_oracle_initial(sc)
            succ, todo = {}, [init]
            while todo:
                s = todo.pop()
                if s in succ:
                    continue
                succ[s] = {lib.pire_oracle_step(sc, s, ch) for ch in list(range(256)) + [BEGIN_MARK, END_MARK]}
                todo.extend(t for t in succ[s] if t not in succ)
            live = {s for s in succ if lib.pire_oracle_final(sc, s)}
            grew = True
            while grew:
                grew = False
                for s, ts in succ.items():
                    if s not in live and ts & live:
                        live.add(s)
                        grew = True
            self._live[key] = live
        return self._live[key]


def text_of(name, size, seed):
    rng = np.random.default_rng(seed)
    host = rng.choice(np.frombuffer(ALPHABET, np.uint8), size=size)
    plants = PLANTS[name]
    at = 3
    while at < size - 40:
        lit = np.frombuffer(plants[int(rng.integers(len(plants)))], np.uint8)
        host[at:at + len(lit)] = lit
        at += len(lit) + int(rng.integers(0, 40))
    return host


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def match_ends(case, text_dev, base, flags, capacity=None):
    """pire_gpu_match_ends_string on the forward image: (ends, ids, found) device tensors."""
    import torch
    from pire_b200 import _native as N
    n = text_dev.numel()
    cap = capacity if capacity is not None else max(16, 4 * n + 16)
    ends = torch.empty(cap, dtype=torch.int64, device="cuda:0")
    ids = torch.empty(cap, dtype=torch.int32, device="cuda:0")
    found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    rc = N.lib.pire_gpu_match_ends_string(case.fwd._h, text_dev.data_ptr() if n else None, n, flags, None, base,
                                          ends.data_ptr(), ids.data_ptr(), cap, found.data_ptr(), None, None, _stream())
    assert rc == 0, N.lib.pire_gpu_last_error()
    return ends, ids, found


def out_buffers(cap):
    import torch
    starts = torch.full((cap + GUARD,), SENT64, dtype=torch.int64, device="cuda:0")
    opened = torch.full((cap + GUARD,), SENT8, dtype=torch.uint8, device="cuda:0")
    return starts, opened


def starts_string(case, text_dev, base, flags, max_back, ends, ids, first, found, cap, starts, opened, use_ids=True):
    import torch
    from pire_b200 import _native as N
    dfirst = None
    if first is not None:
        dfirst = torch.tensor([first], dtype=torch.int64, device="cuda:0")
    n = text_dev.numel()
    rc = N.lib.pire_gpu_match_starts_string(case.rev._h, text_dev.data_ptr() if n else None, n, base, flags, max_back,
                                            ends.data_ptr(), ids.data_ptr() if use_ids else None,
                                            None if dfirst is None else dfirst.data_ptr(), found.data_ptr(), cap,
                                            starts.data_ptr(), None if opened is None else opened.data_ptr(), _stream())
    torch.cuda.synchronize()
    return rc


def want_entry(case, win, wstart, e, rid, begin, end, max_back, use_ids=True):
    """(start, open) of one entry by the oracle; None when its end is outside the window."""
    wend = wstart + len(win)
    if e < wstart or e > wend:
        return None
    lower = e - max_back if max_back and e - wstart > max_back else wstart
    tb = begin and lower == wstart
    orc = case.single[rid] if use_ids else case.glued
    offs = np.array([lower - wstart, e - wstart], np.uint64)
    best, opened = -1, False
    lib, sc = _lib(), C.byref(orc._sc)
    seg = np.ascontiguousarray(win[lower - wstart:e - wstart][::-1])
    for te in ((False, True) if end and e == wend else (False,)):
        best = max(best, int(oracle_suffix(orc, win, offsets=offs, through_end=te, through_begin=tb)[0]))
        if not tb:
            st = lib.pire_oracle_initial(sc)
            if te:
                st = lib.pire_oracle_step(sc, st, END_MARK)
            if seg.size:
                st = lib.pire_oracle_run(sc, st, seg.ctypes.data, seg.ctypes.data + seg.size)
            if use_ids:
                opened = opened or st in case.live(orc)
            else:
                lib.pire_oracle_dead.argtypes = [C.POINTER(type(orc._sc)), C.c_uint64]
                opened = opened or not lib.pire_oracle_dead(sc, st)
    return (NO_START if best < 0 else e - best), opened


def check(case, win, wstart, ends_h, ids_h, got_s, got_o, lo, hi, begin, end, max_back, use_ids=True, ks=None):
    """Entries [lo, hi) (or the indices ks) against the oracle; entries outside the window keep their sentinels."""
    bad = []
    for k in (range(lo, hi) if ks is None else ks):
        w = want_entry(case, win, wstart, int(ends_h[k]), int(ids_h[k]), begin, end, max_back, use_ids)
        if w is None:
            if got_s[k] != SENT64 or (got_o is not None and got_o[k] != SENT8):
                bad.append((k, "written outside the window"))
            continue
        if int(got_s[k]) != w[0] or (got_o is not None and bool(got_o[k]) != w[1]):
            bad.append((k, int(ends_h[k]), int(ids_h[k]), hex(int(got_s[k])), hex(w[0]), int(got_o[k]) if got_o is not None else None, w[1]))
    assert not bad, (case.name, len(bad), bad[:5])


def host(t, dtype):
    return t.cpu().numpy().view(dtype)


@pytest.mark.parametrize("name", sorted(START_IMAGES))
@pytest.mark.parametrize("flags", [0, RUN_BEGIN, RUN_END, RUN_BEGIN | RUN_END])
@pytest.mark.parametrize("use_ids", [True, False])
def test_string_form(name, flags, use_ids):
    import torch
    case = Case(name)
    size = 3000
    host_text = text_of(name, size + 16, seed=flags * 7 + len(name))
    buf = torch.from_numpy(host_text).to("cuda:0")
    skew = 5 + flags                                      # an unaligned window
    text = buf[skew:skew + size]
    win = host_text[skew:skew + size]
    base = 1000003
    ends, ids, found = match_ends(case, text, base, flags)
    nf = int(found.item())
    cap = ends.numel()
    assert 0 < nf <= cap
    starts, opened = out_buffers(cap)
    assert starts_string(case, text, base, flags, 0, ends, ids, None, found, cap, starts, opened, use_ids) == 0
    s, o = host(starts, np.uint64), host(opened, np.uint8)
    assert (s[nf:] == SENT64).all() and (o[nf:] == SENT8).all()
    check(case, win, base, host(ends, np.uint64), host(ids, np.uint32), s, o, 0, nf, bool(flags & RUN_BEGIN),
          bool(flags & RUN_END), 0, use_ids)
    got = s[:nf]
    assert (got != SENT64).all()
    assert ((got == NO_START) | (got <= host(ends, np.uint64)[:nf])).all()


@pytest.mark.parametrize("name", ["glue10", "never", "edges", "lit40"])
@pytest.mark.parametrize("max_back", [1, 7, 64])
def test_max_back_first_and_capacity(name, max_back):
    case = Case(name)
    import torch
    host_text = text_of(name, 2000, seed=max_back)
    text = torch.from_numpy(host_text).to("cuda:0")
    flags = RUN_BEGIN | RUN_END
    ends, ids, found = match_ends(case, text, 0, flags)
    nf = int(found.item())
    first, cap = 3, nf - 2
    starts, opened = out_buffers(ends.numel())
    assert starts_string(case, text, 0, flags, max_back, ends, ids, first, found, cap, starts, opened) == 0
    s, o = host(starts, np.uint64), host(opened, np.uint8)
    assert (s[:first] == SENT64).all() and (o[:first] == SENT8).all()
    assert (s[cap:] == SENT64).all() and (o[cap:] == SENT8).all()
    check(case, host_text, 0, host(ends, np.uint64), host(ids, np.uint32), s, o, first, cap, True, True, max_back)
    # an empty range writes nothing
    starts2, opened2 = out_buffers(ends.numel())
    assert starts_string(case, text, 0, flags, max_back, ends, ids, cap, found, cap, starts2, opened2) == 0
    assert (host(starts2, np.uint64) == SENT64).all() and (host(opened2, np.uint8) == SENT8).all()


@pytest.mark.parametrize("name", ["glue10", "never", "edges", "empty"])
def test_chunked_windows(name):
    """One entry array over the whole text, processed window by window with overlap: each call writes the entries
    inside its window and nothing else, each as the oracle says for that window; and an entry whose start differs from
    the whole text's answer had its open flag set."""
    import torch
    case = Case(name)
    size = 4096
    host_text = text_of(name, size, seed=11)
    full = torch.from_numpy(host_text).to("cuda:0")
    flags = RUN_BEGIN | RUN_END
    ends, ids, found = match_ends(case, full, 0, flags)
    nf = int(found.item())
    ends_h, ids_h = host(ends, np.uint64), host(ids, np.uint32)
    whole, whole_open = out_buffers(ends.numel())
    assert starts_string(case, full, 0, flags, 0, ends, ids, None, found, ends.numel(), whole, whole_open) == 0
    whole_h = host(whole, np.uint64)
    for a, b in ((0, 1500), (1000, 2600), (2500, 4096), (777, 781), (4096, 4096)):
        starts, opened = out_buffers(ends.numel())
        win = full[a:b]
        rc = starts_string(case, win, a, (RUN_BEGIN if a == 0 else 0) | (RUN_END if b == size else 0), 0, ends, ids, None,
                           found, ends.numel(), starts, opened)
        assert rc == 0
        s, o = host(starts, np.uint64), host(opened, np.uint8)
        check(case, host_text[a:b], a, ends_h, ids_h, s, o, 0, nf, a == 0, b == size, 0)
        inside = (ends_h[:nf] >= a) & (ends_h[:nf] <= b)
        moved = inside & (s[:nf] != whole_h[:nf])
        assert (o[:nf][moved] == 1).all(), (a, b)


def _batch_ends(case, batch, n, rounds, flags_first, flags_last):
    import pire_b200 as P
    me = P.BatchMatchEnds(case.fwd, n, 64 * sum(b.payload_bytes() for b in rounds) + 64)
    if flags_first & RUN_BEGIN:
        me.Begin()
    for b in rounds:
        me.Run(b)
    if flags_last & RUN_END:
        me.End()
    return me


@pytest.mark.parametrize("name", ["glue10", "edges", "never", "lit40"])
@pytest.mark.parametrize("layout", ["fixed", "csr"])
def test_batch_form(name, layout):
    """Two rounds of BatchMatchEnds, then the starts of the entries of the second round's window, with the d_pos the
    ends left behind; entries of the first round are outside every window and keep their sentinels.  A batch of one
    round with d_pos == NULL and BEGIN is compared too, and d_strings == NULL on a one-string batch."""
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    case = Case(name)
    n = 67
    rng = np.random.default_rng(5)
    lens = np.full(n, 96) if layout == "fixed" else rng.integers(0, 200, size=n)
    texts = [[text_of(name, int(l) + 48, seed=1000 * r + i)[:int(l)] for i, l in enumerate(lens)] for r in range(2)]

    def batch_of(strs):
        if layout == "fixed":
            return P.Batch(torch.from_numpy(np.concatenate(strs)).to("cuda:0"), fixed_len=int(lens[0]), n=n)
        return P.Batch.from_strings([s.tobytes() for s in strs])

    rounds = [batch_of(texts[0]), batch_of(texts[1])]
    me = _batch_ends(case, None, n, rounds, RUN_BEGIN, RUN_END)
    nf = me.Found()
    assert nf <= me.capacity
    cap = me.capacity
    starts, opened = out_buffers(cap)
    win = rounds[1]
    rc = N.lib.pire_gpu_match_starts_batch(case.rev._h, win.corpus.data_ptr(), None if win.offsets is None else win.offsets.data_ptr(),
                                           win.fixed_len, n, me.PosTensor().data_ptr(), RUN_END, 0,
                                           me.StringsTensor().data_ptr(), me.EndsTensor().data_ptr(), me.IdsTensor().data_ptr(),
                                           None, me.FoundTensor().data_ptr(), cap, starts.data_ptr(), opened.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc == 0
    s, o = host(starts, np.uint64), host(opened, np.uint8)
    strs, ends_h, ids_h = me.Strings(), me.Ends(), me.Ids()
    assert (s[nf:] == SENT64).all() and (o[nf:] == SENT8).all()
    for i in range(n):                                    # string i's entries of both rounds
        check(case, texts[1][i], int(lens[i]), ends_h, ids_h, s, o, 0, 0, False, True, 0, ks=np.nonzero(strs == i)[0])

    # one round, d_pos == NULL: ends are offsets within each string
    me1 = _batch_ends(case, None, n, rounds[:1], RUN_BEGIN, RUN_END)
    s1, o1 = out_buffers(me1.capacity)
    w1 = rounds[0]
    rc = N.lib.pire_gpu_match_starts_batch(case.rev._h, w1.corpus.data_ptr(), None if w1.offsets is None else w1.offsets.data_ptr(),
                                           w1.fixed_len, n, None, RUN_BEGIN | RUN_END, 0, me1.StringsTensor().data_ptr(),
                                           me1.EndsTensor().data_ptr(), me1.IdsTensor().data_ptr(), None,
                                           me1.FoundTensor().data_ptr(), me1.capacity, s1.data_ptr(), o1.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc == 0
    s1h, o1h = host(s1, np.uint64), host(o1, np.uint8)
    strs1, ends1, ids1 = me1.Strings(), me1.Ends(), me1.Ids()
    for i in range(n):
        check(case, texts[0][i], 0, ends1, ids1, s1h, o1h, 0, 0, True, True, 0, ks=np.nonzero(strs1 == i)[0])

    # d_strings == NULL: every entry belongs to string 0 of a one-string batch
    one = P.Batch.from_strings([texts[0][0].tobytes()])
    me0 = _batch_ends(case, None, 1, [one], RUN_BEGIN, RUN_END)
    s0, o0 = out_buffers(me0.capacity)
    rc = N.lib.pire_gpu_match_starts_batch(case.rev._h, one.corpus.data_ptr(), one.offsets.data_ptr(), 0, 1, None,
                                           RUN_BEGIN | RUN_END, 0, None, me0.EndsTensor().data_ptr(), me0.IdsTensor().data_ptr(),
                                           None, me0.FoundTensor().data_ptr(), me0.capacity, s0.data_ptr(), o0.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc == 0
    check(case, texts[0][0], 0, me0.Ends(), me0.Ids(), host(s0, np.uint64), host(o0, np.uint8), 0, me0.Found(), True, True, 0)


def test_python_face_and_two_calls_identical():
    import torch
    import pire_b200 as P
    case = Case("glue10")
    host_text = text_of("glue10", 50000, seed=3)
    t = torch.from_numpy(host_text).to("cuda:0")
    cap = 1 << 16
    r1 = P.MatchStarts(case.rev, P.StringMatchEnds(case.fwd, cap).Begin().Run(t).End(), t)
    r2 = P.MatchStarts(case.rev, P.StringMatchEnds(case.fwd, cap).Begin().Run(t).End(), t)
    a, b = r1.Starts(), r2.Starts()
    assert len(a) > 100 and (a == b).all() and (r1.Open() == r2.Open()).all()
    assert torch.equal(r1.StartsTensor(), r2.StartsTensor()) and torch.equal(r1.OpenTensor(), r2.OpenTensor())
    assert not r1.Open().any()                            # the whole text, BEGIN: every walk is settled
    ends, ids, found = match_ends(case, t, 0, RUN_BEGIN | RUN_END, cap)
    starts, opened = out_buffers(cap)
    assert starts_string(case, t, 0, RUN_BEGIN | RUN_END, 0, ends, ids, None, found, cap, starts, opened) == 0
    assert (host(starts, np.uint64)[:len(a)] == a).all()
    check(case, host_text, 0, host(ends, np.uint64), host(ids, np.uint32), host(starts, np.uint64),
          host(opened, np.uint8), 0, min(len(a), 3000), True, True, 0)


def test_batch_python_face():
    import torch
    import pire_b200 as P
    case = Case("edges")
    n, L = 40, 64
    strs = [text_of("edges", L + 48, seed=i)[:L] for i in range(n)]
    batch = P.Batch(torch.from_numpy(np.concatenate(strs)).to("cuda:0"), fixed_len=L, n=n)
    me = P.BatchMatchEnds(case.fwd, n, 4096).Begin().Run(batch).End()
    r = P.MatchStarts(case.rev, me, batch)
    s, e, ids, st = r.Starts(), me.Ends(), me.Ids(), me.Strings()
    for k in range(len(s)):
        w = want_entry(case, strs[st[k]], 0, int(e[k]), int(ids[k]), True, True, 0)
        assert int(s[k]) == w[0]


def test_walk_past_4_gib():
    """One window just past 2^32 bytes and one a.*b entry whose reversed walk crosses all of it: 64-bit lengths."""
    import torch
    case = Case("never")
    size = (1 << 32) + 4099
    text = torch.full((size,), ord("c"), dtype=torch.uint8, device="cuda:0")
    text[2] = ord("a")
    text[size - 3] = ord("b")
    ends = torch.tensor([size - 2, 7, size - 2], dtype=torch.int64, device="cuda:0")
    ids = torch.zeros(3, dtype=torch.int32, device="cuda:0")
    found = torch.tensor([3], dtype=torch.int64, device="cuda:0")
    starts, opened = out_buffers(3)
    base = 1 << 33
    ends += base
    assert starts_string(case, text, base, RUN_BEGIN | RUN_END, 0, ends, ids, None, found, 3, starts, opened) == 0
    s, o = host(starts, np.uint64), host(opened, np.uint8)
    assert int(s[0]) == base + 2 and int(s[2]) == base + 2 and o[0] == 0
    assert int(s[1]) == NO_START                         # no 'b' ends at 7
    # the same walk cut by max_back: no 'a' within reach, and open
    starts, opened = out_buffers(3)
    assert starts_string(case, text, base, RUN_BEGIN | RUN_END, 1 << 20, ends, ids, None, found, 3, starts, opened) == 0
    s, o = host(starts, np.uint64), host(opened, np.uint8)
    assert int(s[0]) == NO_START and o[0] == 1
    del text
    torch.cuda.empty_cache()


def test_refusals():
    import torch
    from pire_b200 import _native as N
    case = Case("edges")
    t = torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    ends = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    found = torch.ones(1, dtype=torch.int64, device="cuda:0")
    starts, opened = out_buffers(4)
    f = N.lib.pire_gpu_match_starts_string
    assert f(case.rev._h, t.data_ptr(), 16, 0, RUN_LINES, 0, ends.data_ptr(), None, None, found.data_ptr(), 4, starts.data_ptr(), None, None) == -1
    assert f(case.rev._h, t.data_ptr(), 16, 0, 8, 0, ends.data_ptr(), None, None, found.data_ptr(), 4, starts.data_ptr(), None, None) == -1
    assert f(case.rev._h, t.data_ptr(), 16, 0, 0, 0, None, None, None, found.data_ptr(), 4, starts.data_ptr(), None, None) == -1
    assert f(case.rev._h, t.data_ptr(), 16, 0, 0, 0, ends.data_ptr(), None, None, None, 4, starts.data_ptr(), None, None) == -1
    assert f(case.rev._h, t.data_ptr(), 16, 0, 0, 0, ends.data_ptr(), None, None, found.data_ptr(), 4, None, None, None) == -1
    assert f(case.rev._h, None, 16, 0, 0, 0, ends.data_ptr(), None, None, found.data_ptr(), 4, starts.data_ptr(), None, None) == -1
    torch.cuda.synchronize()
    assert (host(starts, np.uint64) == SENT64).all()


def test_cpp_match_starts(tmp_path):
    """tests/cpp/match_starts_check.cpp through include/pire_gpu.hpp: ends plus starts over a text fed in pieces, each
    piece's entries walked in a window of the piece and the 4 KiB before it, equal the one call over the whole text once
    the open entries are walked again from the text's start."""
    import os
    import shutil
    import subprocess
    from refpire import ROOT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "match_starts_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "match_starts_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    images = []
    for name in ("glue10", "words"):
        for kind in ("forward", "reversed"):
            images.append(tmp_path / ("%s_%s.pire" % (name, kind)))
            images[-1].write_bytes(START_IMAGES[name][kind])
    for fwd, rev in ((images[0], images[1]), (images[2], images[3])):
        for n, seed in ((3_000_017, 1), (1000, 2), (0, 3)):
            out = subprocess.run([exe, str(fwd), str(rev), str(n), str(seed)], capture_output=True, text=True, timeout=300)
            assert out.returncode == 0, out.stdout + out.stderr
            assert ": 0 mismatches" in out.stdout
