"""pire_gpu_count_string: HalfFinalScanner counts of one string over the whole grid, from Initialize() or resumed.

Every case compares the u64 counters with pire_gpu_count_batch on the same bytes (CSR, n = 1) or with the in-repo
oracle, and the match word and StateIndex with pire_gpu_run_string.  Output buffers are 64 words long and pre-filled
with a sentinel past the words the call may change."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, GOLDEN_COUNTS, ROOT
from refpire import Oracle, oracle_count
from count_oracle import count_from
from test_gpu_string import BLOCK, MIN_BLOCKS, PRINTABLE, SENTINEL, Checker, ctas, full_grid, glue10, text_buffer

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END = 1, 2
MARKS = [0, RUN_BEGIN, RUN_END, RUN_BEGIN | RUN_END]


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _start_word(start):
    import torch
    word = start & 0xFFFFFFFF
    return torch.tensor([word - (1 << 32) if word >= 1 << 31 else word], dtype=torch.int32, device="cuda:0")


class Counter(Checker):
    """Checker with the counting entry points: count_string launches into rows of one buffer without a synchronise."""

    def regs(self):
        return max(1, self.sc.RegexpsCount())

    def launch(self, dev, off, n, flags, counts, words, start_ptr=None, stream=None):
        from pire_b200 import _native as N
        text = None if dev is None else dev.data_ptr() + off
        N.check(N.lib.pire_gpu_count_string(self.sc._h, text, n, flags, start_ptr, counts.data_ptr(), words.data_ptr(),
                                            words.data_ptr() + 4, stream or _stream()), "pire_gpu_count_string")

    def count(self, dev, off, n, flags, start=None):
        """-> (counts as a list, match word, state); nothing past the counters and words 0 may change."""
        import torch
        counts = torch.zeros(self.regs() + 64, dtype=torch.int64, device="cuda:0")
        counts[self.regs():] = SENTINEL
        words = torch.full((64,), SENTINEL, dtype=torch.int32, device="cuda:0")
        st = None if start is None else _start_word(start)
        self.launch(dev, off, n, flags, counts, words, None if st is None else st.data_ptr())
        c = counts.cpu().numpy()
        w = words.cpu().numpy().view(np.uint32)
        assert (c[self.regs():] == SENTINEL).all(), "counters written past max(1, regexps)"
        assert (w[2:] == SENTINEL).all(), "written past the match and state words"
        return [int(x) for x in c[: self.regs()]], int(w[0]), int(w[1])

    def count_batch(self, dev, off, n, flags):
        import torch
        from pire_b200 import _native as N
        counts = torch.zeros(self.regs(), dtype=torch.int32, device="cuda:0")
        bits = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        offs = torch.tensor([off, off + n], dtype=torch.int64, device="cuda:0")
        N.check(N.lib.pire_gpu_count_batch(self.sc._h, dev.data_ptr(), offs.data_ptr(), 0, 1, flags, counts.data_ptr(), bits.data_ptr(),
                                           _stream()), "pire_gpu_count_batch")
        return [int(x) for x in counts.cpu().numpy().view(np.uint32)], int(bits.cpu().numpy().view(np.uint32)[0])

    def check_count(self, dev, off, n, flags, what=""):
        """count_string against count_batch (n = 1) and run_string on the same bytes."""
        got = self.count(dev, off, n, flags)
        counts, bit = self.count_batch(dev, off, n, flags)
        match, _, state = self.string(dev, off, n, flags)
        assert got == (counts, match, state), (what, off, n, flags, got, counts, match, state)
        assert bit == match
        return got


def test_golden_counts(cuda_device):
    """The numbers of count_ut.cpp HalfFinal@553 (committed fixtures), every string counted alone."""
    import torch
    for case in GOLDEN_COUNTS:
        for max_hot, mode in ((255, 0), (255, 1), (255, 2), (255, 3), (3, 1), (3, 2), (3, 3)):
            c = Counter(case.image, max_hot=max_hot)
            c.sc.set_count_mode(mode)
            for s, want, fin in zip(case.strings, case.counts, case.final):
                dev = torch.frombuffer(bytearray(s + b"\0" * 32), dtype=torch.uint8).to("cuda:0")
                got = c.count(dev, 0, len(s), RUN_BEGIN | RUN_END)
                assert got[0] == want and got[1] == fin, (case, max_hot, mode, s)


def test_short_lengths_all_alignments(cuda_device):
    """Lengths 0..300 at all 32 alignments, the four mark combinations, the three counter forms."""
    import torch
    from pire_b200 import workloads as W
    c = Counter(W.load_image("hf_glue10"))
    _, plants = glue10()
    dev, host = text_buffer(400, PRINTABLE, plants, every=41, seed=21)
    for mode in (1, 2, 3):
        c.sc.set_count_mode(mode)
        for flags in MARKS:
            cases = [(off, n) for off in range(32) for n in range(0, 301, 1 if off in (0, 1, 17) else 7)]
            regs = c.regs()
            counts = torch.zeros((len(cases), regs), dtype=torch.int64, device="cuda:0")
            words = torch.full((len(cases), 2), SENTINEL, dtype=torch.int32, device="cuda:0")
            for k, (off, n) in enumerate(cases):
                c.launch(dev, off, n, flags, counts[k], words[k])
            got_c = counts.cpu().numpy()
            got_w = words.cpu().numpy().view(np.uint32)
            orc = c.orc
            corpus = np.concatenate([host[off:off + n] for off, n in cases])
            offs = np.concatenate([[0], np.cumsum([n for _, n in cases])]).astype(np.uint64)
            want, wfin = oracle_count(orc, corpus, offs, begin=bool(flags & RUN_BEGIN), end=bool(flags & RUN_END))
            assert (got_c == want).all(), (mode, flags, np.argwhere(got_c != want)[:4])
            assert (got_w[:, 0] == wfin).all()
            for k in range(0, len(cases), 97):
                off, n = cases[k]
                assert c.check_count(dev, off, n, flags, what="short")[1:] == (int(got_w[k, 0]), int(got_w[k, 1]))


def test_piece_boundaries(cuda_device):
    """Lengths one block either side of the piece boundaries of a one-CTA grid, a few CTAs and the full grid."""
    from pire_b200 import workloads as W
    c = Counter(W.load_image("hf_glue10"))
    _, plants = glue10()
    full = full_grid(c.sc.info().hot_rows)
    step = 32 * BLOCK * MIN_BLOCKS
    assert ctas(step, full) == 1 and ctas(step + 32, full) == 2
    lens = [32 * BLOCK - 32, 32 * BLOCK, 32 * BLOCK + 32, step - 32, step, step + 32, 3 * step - 32, 3 * step + 32,
            full * step - 32, full * step, full * step + 32, 2 * full * step + 32]
    dev, host = text_buffer(max(lens) + 64, PRINTABLE, plants, every=4093, seed=22)
    for mode in (0, 1, 2, 3):
        c.sc.set_count_mode(mode)
        for n in lens:
            for off in (0, 13):
                c.check_count(dev, off, n, RUN_BEGIN | RUN_END if off else 0, what=("length", mode))


def test_images_modes_and_hot_sets(cuda_device):
    """hf_glue10, headline and count_words5; count modes AUTO / LISTS / PACKED / EVERY_CHUNK; static, tuned and tiny hot
    sets (H = 2, 6)."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    _, plants = glue10()
    dev, host = text_buffer(2_000_128, PRINTABLE, plants + [b"hello world", b"the cat"], every=1013, seed=23)
    for name in ("hf_glue10", "headline", "count_words5"):
        for tuned in (False, True):
            c = Counter(W.load_image(name))
            if tuned:
                c.sc.Tune(P.Batch(dev[: len(host) // 4096 * 4096], fixed_len=4096))
            for max_hot in (255, 6, 2):
                c.sc.set_max_hot(max_hot)
                for mode in (0, 1, 2, 3):
                    c.sc.set_count_mode(mode)
                    for flags in (RUN_BEGIN | RUN_END, 0):
                        c.check_count(dev, 3, 2_000_003, flags, what=(name, tuned, max_hot, mode))


def test_many_regexps(cuda_device, ref):
    """The 21-counter glued scanner of test_half_final_counts_vs_reference: more than 16 regexps, the accept lists."""
    from refpire import Oracle as O
    scs = [ref.compile_half_final(b"ab+", "un", mode) for mode in (1, 2, 3, 4, 5)]
    glued = scs[0]
    for sc in scs[1:] + [scs[3], scs[1]]:
        glued = ref.glue_half_final(glued, sc)
    many = glued
    for _ in range(2):
        many = ref.glue_half_final(many, glued)
    assert many.regexps == 21
    c = Counter(many.save())
    dev, host = text_buffer(1_000_064, b"abcde z", seed=24)
    for mode in (0, 2):
        c.sc.set_count_mode(mode)
        for n in (0, 31, 5000, 1_000_001):
            for flags in (RUN_BEGIN | RUN_END, 0):
                got = c.check_count(dev, 7, n, flags, what=("21", mode))
                want, _ = oracle_count(O(many.save()), host[7:7 + n], np.array([0, n], np.uint64), begin=bool(flags & 1),
                                       end=bool(flags & 2))
                assert got[0] == want[0].tolist()


def test_planted_64_mib(cuda_device):
    """64 MiB of planted text, hf_glue10 untuned and tuned, against the oracle."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    image = W.load_image("hf_glue10")
    _, plants = glue10()
    n = 64 * 2 ** 20
    dev, host = text_buffer(n + 64, PRINTABLE, plants, every=1009, seed=25)
    want, wfin = oracle_count(Oracle(image), host[5:5 + n], np.array([0, n], np.uint64))
    for tuned in (False, True):
        c = Counter(image)
        if tuned:
            c.sc.Tune(P.Batch(dev[:n], fixed_len=4096))
        got = c.count(dev, 5, n, RUN_BEGIN | RUN_END)
        assert got[0] == want[0].tolist() and got[1] == int(wfin[0]), tuned
        assert got[1:] == c.string(dev, 5, n, RUN_BEGIN | RUN_END)[::2]


def test_resume_chained_in_place(cuda_device):
    """A text cut at many points (empty chunks and cuts inside a 32-byte block), chained through one state word and one
    counts buffer with no synchronise: the sum equals the one-shot count."""
    import torch
    from pire_b200 import workloads as W
    rng = np.random.default_rng(26)
    _, plants = glue10()
    c = Counter(W.load_image("hf_glue10"))
    n = 3_000_017
    dev, host = text_buffer(n + 64, PRINTABLE, plants, every=7919, seed=27)
    for mode in (1, 2, 3):
        c.sc.set_count_mode(mode)
        one = c.check_count(dev, 1, n, RUN_BEGIN | RUN_END, what="one call")
        for trial in range(3):
            cuts = np.sort(np.concatenate([[0, n], rng.integers(0, n, size=8), rng.integers(0, 40, size=3)]))
            cuts = np.concatenate([cuts[:3], cuts[2:3], cuts[3:]])          # an empty chunk
            counts = torch.zeros(c.regs(), dtype=torch.int64, device="cuda:0")
            words = torch.full((64,), SENTINEL, dtype=torch.int32, device="cuda:0")
            state = words.data_ptr() + 4
            from pire_b200 import _native as N
            for k in range(len(cuts) - 1):
                flags = (RUN_BEGIN if k == 0 else 0) | (RUN_END if k == len(cuts) - 2 else 0)
                N.check(N.lib.pire_gpu_count_string(c.sc._h, dev.data_ptr() + 1 + int(cuts[k]), int(cuts[k + 1] - cuts[k]), flags,
                                                    None if k == 0 else state, counts.data_ptr(), words.data_ptr(), state, _stream()),
                        "pire_gpu_count_string")
            w = words.cpu().numpy().view(np.uint32)
            assert (w[2:] == SENTINEL).all()
            assert ([int(x) for x in counts.cpu().numpy()], int(w[0]), int(w[1])) == one, (mode, trial, cuts)


def test_resume_from_every_state(cuda_device):
    """From every state of a small HalfFinalScanner (the golden glue of five counters), against the oracle's count walk;
    starts outside the scanner count nothing."""
    case = GOLDEN_COUNTS[0]
    c = Counter(case.image)
    dev, host = text_buffer(400, PRINTABLE + b"aaaabbbb", seed=28)
    for mode in (1, 2):
        c.sc.set_count_mode(mode)
        for st in range(c.sc.Size()):
            for flags in MARKS:
                for off, n in ((0, 0), (3, 7), (5, 333)):
                    want, res = count_from(c.orc, host[off:off + n], st, bool(flags & 1), bool(flags & 2))
                    got = c.count(dev, off, n, flags, start=st)
                    assert got == (want, res[0], res[2]), (mode, st, flags, n, got, want, res)
    for st in (c.sc.Size(), c.sc.Size() + 1, 0xFFFFFFFF):
        for flags in MARKS:
            assert c.count(dev, 0, 300, flags, start=st) == ([0] * c.regs(), 0, 0xFFFFFFFF)


def test_past_4_gib_and_2_32_counts(cuda_device, ref):
    """`a` (surrounded) over 4.5 GiB of `a`: every byte ends a match, so the count is n_bytes plus what the mark steps
    add (taken from the oracle's count of 64 a's) -- past 2^32 in one counter, with u64 offsets, and no oracle over the
    whole text.  The image is compiled by the reference (oracle/_ref)."""
    import torch
    import refpire
    if not refpire.have_ref():
        pytest.skip("needs the reference build (oracle/_ref) to compile the `a` HalfFinalScanner")
    c = Counter(ref.compile_half_final(b"a", "", 0).save())
    n = 4 * 2 ** 30 + 2 ** 29 + 13
    dev = torch.full((n + 64,), ord("a"), dtype=torch.uint8, device="cuda:0")
    try:
        for flags in (0, RUN_BEGIN | RUN_END):
            small, _ = count_from(c.orc, np.full(64, ord("a"), np.uint8), None, bool(flags & 1), bool(flags & 2))
            assert small[0] >= 64
            got = c.count(dev, 0, n, flags)
            assert got[0] == [small[0] - 64 + n], (flags, got, small)
            assert got[1:] == c.string(dev, 0, n, flags)[::2]
    finally:
        del dev
        torch.cuda.empty_cache()


def test_two_streams_one_handle(cuda_device):
    import torch
    from pire_b200 import workloads as W
    _, plants = glue10()
    c = Counter(W.load_image("hf_glue10"))
    n = 64 * 2 ** 20
    dev_a, host_a = text_buffer(n + 64, PRINTABLE, plants, every=100_003, seed=29)
    dev_b, host_b = text_buffer(n + 64, PRINTABLE, plants[::-1], every=77_777, seed=30)
    want = [c.count(d, 0, n, RUN_BEGIN | RUN_END) for d in (dev_a, dev_b)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    counts = [torch.zeros(c.regs(), dtype=torch.int64, device="cuda:0") for _ in range(2)]
    words = [torch.full((2,), SENTINEL, dtype=torch.int32, device="cuda:0") for _ in range(2)]
    torch.cuda.synchronize()
    for rep in range(3):
        for s, dev, cn, w in zip(streams, (dev_a, dev_b), counts, words):
            c.launch(dev, 0, n, RUN_BEGIN | RUN_END, cn, w, stream=s.cuda_stream)
    torch.cuda.synchronize()
    for cn, w, wa in zip(counts, words, want):
        assert [int(x) for x in cn.cpu().numpy()] == [3 * x for x in wa[0]]
        assert (int(w[0].item()), int(w[1].item()) & 0xFFFFFFFF) == wa[1:]


def test_arguments_empty_scanner_and_zero_bytes(cuda_device):
    import torch
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    c = Counter(W.load_image("hf_glue10"))
    dev = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    counts = torch.zeros(c.regs(), dtype=torch.int64, device="cuda:0")
    for flags in (4, 8, 1 << 31, RUN_BEGIN | 4):
        assert N.lib.pire_gpu_count_string(c.sc._h, dev.data_ptr(), 10, flags, None, counts.data_ptr(), None, None, _stream()) == -1
    assert N.lib.pire_gpu_count_string(c.sc._h, dev.data_ptr(), 10, 0, None, None, None, None, _stream()) == -1
    assert N.lib.pire_gpu_count_string(c.sc._h, None, 1, 0, None, counts.data_ptr(), None, None, _stream()) == -1
    assert N.lib.pire_gpu_count_string(None, dev.data_ptr(), 1, 0, None, counts.data_ptr(), None, None, _stream()) == -1
    assert not counts.any().item()
    for flags in MARKS:
        want, res = count_from(c.orc, np.zeros(0, np.uint8), None, bool(flags & 1), bool(flags & 2))
        assert c.count(None, 0, 0, flags) == (want, res[0], res[2])
        assert c.check_count(dev, 0, 0, flags)[0] == want
    empty = next(x for x in GOLDEN if x.name == "EmptyScanner@784")
    e = Counter(empty.image)
    dev, host = text_buffer(100_064, PRINTABLE, seed=31)
    for flags in MARKS:
        for n in (0, 5, 100_000):
            e.check_count(dev, 0, n, flags, what="empty scanner")


def test_python_string_counter(cuda_device):
    import pire_b200 as P
    from pire_b200 import workloads as W
    _, plants = glue10()
    c = Counter(W.load_image("hf_glue10"))
    n = 5_000_003
    dev, host = text_buffer(n + 64, PRINTABLE, plants, every=100_003, seed=32)
    want = c.count(dev, 0, n, RUN_BEGIN | RUN_END)
    cuts = [0, 0, 1, 33, 1_000_000, 1_000_000, 4_000_001, n]
    r = P.StringCounter(c.sc).Begin()
    for lo, hi in zip(cuts, cuts[1:]):
        r.Run(dev[lo:hi])
    r.End()
    assert [r.Result(i) for i in range(c.regs())] == want[0] and (int(r.Final()), r.State()) == want[1:]
    assert r.AcceptedRegexps() == [i for i, x in enumerate(want[0]) if x]
    # resumed from the state the first half reached: its start is not counted again
    half = P.StringCounter(c.sc).Begin().Run(dev[: n // 2])
    rest = P.StringCounter(c.sc, half.State()).Run(dev[n // 2: n]).End()
    assert [half.Result(i) + rest.Result(i) for i in range(c.regs())] == want[0] and rest.State() == want[2]
    assert P.StringCounter(c.sc, c.sc.Size()).Begin().Run(dev[:100]).End().State() == 0xFFFFFFFF


def test_cpp_string_counter(tmp_path, cuda_device):
    """tests/cpp/count_string_check.cpp through include/pire_gpu.hpp's StringCounter: one call, a chain and
    pire_gpu_count_batch agree."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "count_string_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "count_string_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    image = tmp_path / "hf_glue10.pire"
    image.write_bytes(W.load_image("hf_glue10"))
    for n, seed in ((30_000_017, 1), (1000, 2), (0, 3)):
        out = subprocess.run([exe, str(image), str(n), str(seed)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ": 0 mismatches" in out.stdout
