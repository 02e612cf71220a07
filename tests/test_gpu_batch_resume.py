"""A batch of strings resumed from per-string states (pire_gpu_run_batch_from), against the oracle's run from any state
(tests/string_oracle.py): match bits, accept masks and StateIndex of every string, with 64 sentinel words past n in every
output.  Covers every variant pinned on uniform and CSR batches, length-ordered batches long enough for the split kernel,
cold starts (small hot sets, tuned tables, 32-bit tables), every state of AppendixA as a start, starts outside the
scanner, rounds chained in place through one state buffer, bad arguments, and the Python and C++ front ends."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from refpire import Oracle
from string_oracle import run_from
from test_edge_images import ALPHABETS, EDGE
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, MARKS, SENTINEL, HostBatch, _filled, _host, _stream, csr_batch, expect_equal,
                            expect_untouched, fixed_batch, glue10_image, random_rows, random_strings, unpack_bits)
from test_string_images import STRING_IMAGES

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
LITERALS = [b"GET ", b"error", b"timeout", b"(555) 123-4567", b"https://"]


def _i32(values):
    import torch
    v = np.asarray(values, dtype=np.uint64).astype(np.uint32).view(np.int32)
    return torch.from_numpy(v.copy()).to("cuda:0")


def strings_of(hb):
    corpus, offs, fl = hb.oracle_args()
    if offs is None:
        return [bytes(corpus[i * fl:(i + 1) * fl]) for i in range(hb.n)]
    return [bytes(corpus[int(offs[i]):int(offs[i + 1])]) for i in range(hb.n)]


def want_from(orc, strings, starts, begin, end):
    res = [run_from(orc, np.frombuffer(s, np.uint8), int(st), begin, end) for s, st in zip(strings, starts)]
    return tuple(np.array([r[k] for r in res], dtype=np.uint32) for k in range(3))


def run_from_batch(sc, hb, starts, begin, end, order=None, n=None, state_buf=None):
    """pire_gpu_run_batch_from; returns (bits, masks, states) on the host, with the sentinels past n checked."""
    from pire_b200 import _native as N
    n = hb.n if n is None else n
    flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)
    bits, masks = _filled((n + 31) // 32 + 1), _filled(n + EXTRA)
    if state_buf is None:
        state_buf = _filled(n + EXTRA)
        start_buf = _i32(list(starts) + [SENTINEL] * EXTRA)
    else:
        start_buf = state_buf
    N.check(N.lib.pire_gpu_run_batch_from(sc._h, hb.corpus_ptr(), hb.offsets_ptr(), None if order is None else order.data_ptr(),
                                          hb.fixed_len, n, flags, start_buf.data_ptr(), bits.data_ptr(), masks.data_ptr(),
                                          state_buf.data_ptr(), _stream()), "pire_gpu_run_batch_from")
    hb_bits, hm, hs = _host(bits), _host(masks), _host(state_buf)
    expect_untouched("run_from", "accept masks", hm, n)
    expect_untouched("run_from", "state indices", hs, n)
    return unpack_bits("run_from", hb_bits, n), hm[:n], hs[:n]


def check(sc, orc, hb, starts, begin, end, label, order=None, cache=None):
    strings = strings_of(hb)
    key = (hb.serial, tuple(int(s) for s in starts), begin, end)
    if cache is not None and key in cache:
        want = cache[key]
    else:
        want = want_from(orc, strings, starts, begin, end)
        if cache is not None:
            cache[key] = want
    f, m, s = run_from_batch(sc, hb, starts, begin, end, order=order)
    expect_equal(label, "StateIndex", s, want[2])
    expect_equal(label, "accept masks", m, want[1])
    expect_equal(label, "match bits", f, want[0])


def random_starts(rng, size, n, invalid=True):
    st = rng.integers(0, size, size=n).astype(np.uint64)
    if invalid and n >= 3:
        st[1::11] = size                        # Size(): outside the scanner
        st[2::13] = 0xFFFFFFFF
    return st


def csr_at(strings, base):
    """A CSR batch whose corpus starts `base` bytes into its buffer (offsets relative to the corpus)."""
    hb = csr_batch(strings)
    buf = np.concatenate([np.full(base, 0x41, np.uint8), hb.buf, np.zeros(32, np.uint8)])
    return HostBatch(buf, base=base, offsets=hb.offsets)


# ------------------------------------------------------------------------------------------------ variants and shapes

UNIFORM_SHAPES = [(32, 1), (64, 31), (96, 33), (1024, 64), (1024, 65), (32, 32 * 5 + 3), (256, 32 * 9 + 7), (65536, 5)]


@pytest.mark.parametrize("max_hot", [255, 2])
def test_every_variant_on_uniform_and_csr_batches(max_hot, cuda_device):
    import pire_b200 as P
    rng = np.random.default_rng(100 + max_hot)
    image = glue10_image()
    sc, orc = P.Scanner(image, 0), Oracle(image)
    sc.set_max_hot(max_hot)
    size = sc.Size()
    cache = {}
    batches = [("uniform len=%d n=%d" % (ln, n), fixed_batch(random_rows(rng, n, ln, GLUE10_ALPHABET, LITERALS)))
               for ln, n in UNIFORM_SHAPES]
    for base in (0, 1, 17, 31):
        lengths = [0, 1, 15, 16, 31, 32, 33, 100] + [int(x) for x in rng.integers(0, 2000, size=90)]
        batches.append(("CSR base=%d" % base, csr_at(random_strings(rng, GLUE10_ALPHABET, lengths, LITERALS), base)))
    starts = {label: random_starts(rng, size, hb.n) for label, hb in batches}
    for variant in range(1, 8):
        sc.set_variant(variant)
        for label, hb in batches:
            for begin, end in MARKS:
                check(sc, orc, hb, starts[label], begin, end, "%s variant=%d begin=%d end=%d" % (label, variant, begin, end),
                      cache=cache)


def test_ordered_batches_with_split_strings(cuda_device):
    import pire_b200 as P
    rng = np.random.default_rng(7)
    image = glue10_image()
    sc, orc = P.Scanner(image, 0), Oracle(image)
    lengths = [8192, 9000, 20000, 65536 + 17, 100000] + [int(x) for x in rng.integers(0, 3000, size=200)]
    hb = csr_at(random_strings(rng, GLUE10_ALPHABET, lengths, LITERALS), 5)
    starts = random_starts(rng, sc.Size(), hb.n)
    cache = {}
    for variant in (1, 2, 4):
        sc.set_variant(variant)
        for begin, end in MARKS:
            check(sc, orc, hb, starts, begin, end, "ordered variant=%d begin=%d end=%d" % (variant, begin, end), order=hb.order(),
                  cache=cache)


# ----------------------------------------------------------------------------------------------------------- scanners

def test_scanners_hot_sets_and_tables(cuda_device):
    import pire_b200 as P
    from pire_b200 import workloads as W
    rng = np.random.default_rng(3)
    tune_sample = random_strings(rng, GLUE10_ALPHABET, [1024] * 64, [b"GET ", b"error"])
    for name in ("glue10", "headline"):
        image = W.load_image(name)
        orc = Oracle(image)
        uni = fixed_batch(random_rows(rng, 32 * 3 + 5, 256, GLUE10_ALPHABET, LITERALS))
        ragged = csr_batch(random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(0, 700, size=70)], LITERALS))
        cache = {}
        for tuned in (False, True):
            for max_hot in (255, 6, 2, 1):
                sc = P.Scanner(image, 0)
                sc.set_max_hot(max_hot)
                if tuned:
                    sc.Tune(P.Batch.from_strings(tune_sample), len(tune_sample))
                for variant in (1, 2, 4, 7):
                    sc.set_variant(variant)
                    for hb in (uni, ragged):
                        starts = random_starts(np.random.default_rng(hb.serial), sc.Size(), hb.n)
                        for begin, end in MARKS:
                            check(sc, orc, hb, starts, begin, end, "%s tuned=%d max_hot=%d variant=%d begin=%d end=%d"
                                  % (name, tuned, max_hot, variant, begin, end), cache=cache)
    # 32-bit table cells, and the string images
    images = [("wide", EDGE["wide"]["image"], ALPHABETS["wide"])] + [(k, e["image"], bytes(range(0x20, 0x7F))) for k, e in STRING_IMAGES.items()]
    for name, image, alphabet in images:
        orc = Oracle(image)
        sc = P.Scanner(image, 0)
        hb = fixed_batch(random_rows(rng, 32 * 2 + 3, 128, alphabet))
        ragged = csr_batch(random_strings(rng, alphabet, [int(x) for x in rng.integers(0, 300, size=40)]))
        for max_hot in (255, 2):
            sc.set_max_hot(max_hot)
            for variant in (1, 2, 4, 7):
                sc.set_variant(variant)
                for b in (hb, ragged):
                    starts = random_starts(rng, sc.Size(), b.n)
                    for begin, end in MARKS:
                        check(sc, orc, b, starts, begin, end, "%s max_hot=%d variant=%d begin=%d end=%d" % (name, max_hot, variant,
                                                                                                           begin, end))


def test_every_state_of_appendix_a_as_a_start(cuda_device):
    import pire_b200 as P
    case = next(c for c in GOLDEN if c.name == "AppendixA")
    sc, orc = P.Scanner(case.image, 0), Oracle(case.image)
    size = sc.Size()
    strings = list(case.strings) + [b"hello world", b"hello  wd", b"", b"x" * 40]
    # every (state, string) pair, plus Size() and 0xFFFFFFFF
    states = list(range(size)) + [size, 0xFFFFFFFF]
    pairs = [(s, st) for st in states for s in strings]
    hb = csr_batch([p[0] for p in pairs])
    starts = np.array([p[1] for p in pairs], dtype=np.uint64)
    uni_rows = np.frombuffer((b"hello   world, say hello world!!" * 2), np.uint8)[None, :].repeat(len(states), 0)
    uni = fixed_batch(uni_rows)
    for variant in range(1, 8):
        sc.set_variant(variant)
        for begin, end in MARKS:
            check(sc, orc, hb, starts, begin, end, "AppendixA CSR variant=%d begin=%d end=%d" % (variant, begin, end))
            check(sc, orc, uni, np.array(states, dtype=np.uint64), begin, end,
                  "AppendixA uniform variant=%d begin=%d end=%d" % (variant, begin, end))


# ----------------------------------------------------------------------------------------------------------- identity

def test_initialize_starts_give_run_batch_words(cuda_device):
    """Starts = Initialize() give the words of pire_gpu_run_batch / _ordered, on a large batch, whatever the variant."""
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    spec = W.SynthSpec((1 << 16) + 5, 1024, plants=W.GLUE10_PLANTS)
    dev = torch.empty(spec.total_bytes(), dtype=torch.uint8, device="cuda:0")
    spec.fill_device(dev)
    batch = P.Batch(dev, fixed_len=1024, n=spec.n_strings)
    sc = P.Scanner(W.load_image("glue10"), 0)
    sc.Tune(batch, 1 << 14)
    n = batch.n
    init = torch.full((n,), sc.Initialize(), dtype=torch.int32, device="cuda:0")
    rng = np.random.default_rng(5)
    lengths = [int(x) for x in rng.integers(0, 20000, size=4000)]
    ragged = P.Batch.from_strings(random_strings(rng, GLUE10_ALPHABET, lengths, LITERALS)).bin_by_length()
    for variant in range(0, 8):
        sc.set_variant(variant)
        for flags in (RUN_BEGIN | RUN_END, 0):
            for b in (batch, ragged):
                outs = []
                for start in (None, init[: b.n]):
                    bits = torch.zeros((b.n + 31) // 32, dtype=torch.int32, device="cuda:0")
                    masks = torch.zeros(b.n, dtype=torch.int32, device="cuda:0")
                    states = torch.zeros(b.n, dtype=torch.int32, device="cuda:0")
                    sc.run_batch(b, flags, bits, masks, states, start_idx=start)
                    outs.append((bits.cpu().numpy(), masks.cpu().numpy(), states.cpu().numpy()))
                for k, what in enumerate(("match bits", "accept masks", "StateIndex")):
                    expect_equal("variant=%d flags=%d %s" % (variant, flags, "ordered" if b.order is not None else "uniform"), what,
                                 outs[1][k], outs[0][k])
    sc.set_variant(N.VARIANT_AUTO)


# ----------------------------------------------------------------------------------------------------------- chaining

def _chain_case(sc, rounds, whole_hb, piece_hbs, ordered, variant):
    """k rounds in place through one state buffer; the final words against one pire_gpu_run_batch over the whole strings."""
    from pire_b200 import _native as N
    import torch
    sc.set_variant(variant)
    n = whole_hb.n
    state = _filled(n + EXTRA)
    bits, masks = _filled((n + 31) // 32 + 1), _filled(n + EXTRA)
    state[:n] = sc.Initialize()
    for r, hb in enumerate(piece_hbs):
        flags = (RUN_BEGIN if r == 0 else 0) | (RUN_END if r == rounds - 1 else 0)
        order = hb.order() if ordered else None
        last = r == rounds - 1
        N.check(N.lib.pire_gpu_run_batch_from(sc._h, hb.corpus_ptr(), hb.offsets_ptr(), None if order is None else order.data_ptr(),
                                              hb.fixed_len, n, flags, state.data_ptr(), bits.data_ptr() if last else None,
                                              masks.data_ptr() if last else None, state.data_ptr(), _stream()), "round %d" % r)
    wb, wm, ws = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
    N.check(N.lib.pire_gpu_run_batch(sc._h, whole_hb.corpus_ptr(), whole_hb.offsets_ptr(), whole_hb.fixed_len, n, RUN_BEGIN | RUN_END,
                                     wb.data_ptr(), wm.data_ptr(), ws.data_ptr(), _stream()), "whole")
    torch.cuda.synchronize()
    label = "chain variant=%d ordered=%d rounds=%d" % (variant, ordered, rounds)
    expect_untouched(label, "state indices", _host(state), n)
    expect_equal(label, "StateIndex", _host(state), _host(ws))
    expect_equal(label, "accept masks", _host(masks), _host(wm))
    expect_equal(label, "match bits", _host(bits), _host(wb))


def test_rounds_chained_in_place(cuda_device):
    import pire_b200 as P
    rng = np.random.default_rng(11)
    sc = P.Scanner(glue10_image(), 0)
    # uniform: the two-string ring kernel (LOOK pinned), the one-string ring kernel and the plain walk
    n, length, rounds = 32 * 41 + 9, 1024, 4
    rows = random_rows(rng, n, length, GLUE10_ALPHABET, LITERALS)
    whole = fixed_batch(rows)
    pieces = [fixed_batch(np.ascontiguousarray(rows[:, r * length // rounds:(r + 1) * length // rounds])) for r in range(rounds)]
    for variant in (4, 7, 1, 2):
        _chain_case(sc, rounds, whole, pieces, False, variant)
    # CSR: ragged pieces (some empty), in order and length-ordered with strings long enough for the split kernel
    lengths = [20000, 70000, 9000] + [int(x) for x in rng.integers(0, 5000, size=300)]
    strings = random_strings(rng, GLUE10_ALPHABET, lengths, LITERALS)
    cuts = [sorted(int(c) for c in rng.integers(0, len(s) + 1, size=2)) for s in strings]
    parts = [[s[:c[0]], s[c[0]:c[1]], s[c[1]:]] for s, c in zip(strings, cuts)]
    whole = csr_batch(strings)
    pieces = [csr_at([p[r] for p in parts], 3 * r) for r in range(3)]
    for variant in (1, 2, 4):
        _chain_case(sc, 3, whole, pieces, False, variant)
        _chain_case(sc, 3, whole, pieces, True, variant)


# ------------------------------------------------------------------------------------------------------ bad arguments

def test_bad_arguments(cuda_device):
    import pire_b200 as P
    from pire_b200 import _native as N
    sc = P.Scanner(glue10_image(), 0)
    hb = fixed_batch(random_rows(np.random.default_rng(1), 40, 64, GLUE10_ALPHABET))
    csr = csr_batch([b"abc", b"GET x"])
    start = _i32([sc.Initialize()] * 64)
    out = _filled(64)
    lib = N.lib

    def call(h, corpus, offs, order, fl, n, flags, st):
        return lib.pire_gpu_run_batch_from(h, corpus, offs, order, fl, n, flags, st, out.data_ptr(), out.data_ptr(), out.data_ptr(),
                                           _stream())
    ok = call(sc._h, hb.corpus_ptr(), None, None, 64, 40, 3, start.data_ptr())
    assert ok == 0
    assert call(sc._h, hb.corpus_ptr(), None, None, 64, 40, 3, None) == -1                       # null d_start
    assert call(sc._h, hb.corpus_ptr(), None, None, 64, 40, RUN_LINES | 1, start.data_ptr()) == -1
    assert call(sc._h, hb.corpus_ptr(), None, None, 64, 40, 8, start.data_ptr()) == -1           # unknown flag
    assert call(sc._h, None, None, None, 64, 40, 3, start.data_ptr()) == -1                      # null corpus
    order = csr.order()
    assert call(sc._h, hb.corpus_ptr(), None, order.data_ptr(), 64, 2, 3, start.data_ptr()) == -1   # order, fixed length
    assert call(None, hb.corpus_ptr(), None, None, 64, 40, 3, start.data_ptr()) == -1
    host = P.Scanner(glue10_image(), -1)
    assert call(host._h, hb.corpus_ptr(), None, None, 64, 40, 3, start.data_ptr()) == -4         # PIRE_GPU_ENODEVICE
    before = _host(out).copy()
    assert call(sc._h, None, None, None, 0, 0, 3, None) == 0                                     # n == 0: a no-op
    import torch
    torch.cuda.synchronize()
    assert (_host(out) == before).all()
    assert call(sc._h, csr.corpus_ptr(), csr.offsets_ptr(), order.data_ptr(), 0, 2, 3, start.data_ptr()) == 0
    with pytest.raises(ValueError):
        sc.run_batch(P.Batch.from_text(torch.tensor(list(b"a\nb\n"), dtype=torch.uint8, device="cuda:0")), 3,
                     start_idx=start)


# -------------------------------------------------------------------------------------------------------- front ends

def test_python_runner_chain(cuda_device):
    """Runner(sc, prev.StateTensor()) round after round equals one Runner over the whole strings; with d_order too."""
    import torch
    import pire_b200 as P
    rng = np.random.default_rng(21)
    sc = P.Scanner(glue10_image(), 0)
    n, length, rounds = 32 * 17 + 3, 512, 4
    rows = random_rows(rng, n, length, GLUE10_ALPHABET, LITERALS)
    whole = P.Runner(sc).Begin().Run(P.Batch(torch.from_numpy(rows.reshape(-1).copy()).to("cuda:0"), fixed_len=length, n=n)).End()
    prev = None
    for r in range(rounds):
        piece = np.ascontiguousarray(rows[:, r * length // rounds:(r + 1) * length // rounds])
        b = P.Batch(torch.from_numpy(piece.reshape(-1)).to("cuda:0"), fixed_len=piece.shape[1], n=n)
        cur = P.Runner(sc) if prev is None else P.Runner(sc, prev.StateTensor())
        if r == 0:
            cur.Begin()
        cur.Run(b)
        if r == rounds - 1:
            cur.End()
        prev = cur
    assert (prev.States() == whole.States()).all()
    assert (prev.AcceptMasks() == whole.AcceptMasks()).all()
    assert (prev.Matches() == whole.Matches()).all()
    # a ragged batch, length-ordered, from given states
    strings = random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(0, 12000, size=200)], LITERALS)
    starts = random_starts(rng, sc.Size(), len(strings))
    r = P.Runner(sc, _i32(starts)).Begin().Run(P.Batch.from_strings(strings).bin_by_length()).End()
    want = want_from(Oracle(glue10_image()), strings, starts, True, True)
    expect_equal("python ordered", "StateIndex", r.States(), want[2])
    expect_equal("python ordered", "accept masks", r.AcceptMasks(), want[1])
    expect_equal("python ordered", "match bits", r.Matches().astype(np.uint32), want[0])


def test_cpp_batch_runner(tmp_path, cuda_device):
    """tests/cpp/batch_resume_check.cpp through include/pire_gpu.hpp's BatchRunner::From: rounds chained in place equal one
    pire_gpu_run_batch over the whole strings."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "batch_resume_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "batch_resume_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    image = tmp_path / "glue10.pire"
    image.write_bytes(W.load_image("glue10"))
    for n, length, rounds in ((100_003, 1024, 4), (33, 256, 8), (1, 32, 1)):
        out = subprocess.run([exe, str(image), str(n), str(length), str(rounds), "7"], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ", 0 mismatches" in out.stdout, out.stdout
