"""pire_gpu_run_string: one string over the whole grid, from Initialize() or from a given state.

Every case compares match word, accept mask and StateIndex with the oracle (tests/string_oracle.py: the in-repo C
oracle run from a state), and -- when the string starts from Initialize() -- with pire_gpu_run_batch on the same
bytes (CSR, n = 1).  Every output buffer is 64 words long and pre-filled with a sentinel; only word 0 may change."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from refpire import Oracle
from string_oracle import StringWalk, run_from
from test_edge_images import ALPHABETS, EDGE, static_hot_order
from test_string_images import STRING_IMAGES

pytestmark = pytest.mark.gpu

RUN_BEGIN, RUN_END = 1, 2
MARKS = [0, RUN_BEGIN, RUN_END, RUN_BEGIN | RUN_END]
SENTINEL = 0x5A5A5A5A
PRINTABLE = bytes(range(0x20, 0x7F))

# Python copy of the piece rule of LaunchString / ScanStringKernel (pire_b200/csrc/scan_kernels.cu)
BLOCK = 512                   # kBlock: lanes per CTA
MIN_BLOCKS = 16               # kStringMinBlocks: 32-byte blocks per lane before the grid gets fewer CTAs
MARK_BYTES = BLOCK * 32       # kSplitMarkBytes


def full_grid(hot):
    """The occupancy query's grid on an H100: two CTAs per SM (the kernel's launch bound) unless shared memory allows
    fewer."""
    import torch
    props = torch.cuda.get_device_properties(0)
    shared = ((hot + 1 + 3) // 4 * 4) * 292 + 512 + 256 + 16 + MARK_BYTES
    per_sm = min(2, (228 * 1024) // (shared + 1024))
    return props.multi_processor_count * per_sm


def ctas(n, full):
    want = -(-(n // 32) // (BLOCK * MIN_BLOCKS))
    return max(1, min(want, full))


def pieces(n, off, full):
    """(CTAs, blocks of the shortest piece, lanes with one block more) for n bytes at an address = off mod 32."""
    head = (32 - off % 32) % 32
    body = (n - head) // 32 if n >= head else 0
    g = ctas(n, full)
    return g, body // (g * BLOCK), body % (g * BLOCK)


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


class Checker:
    def __init__(self, image, max_hot=None, variant=None):
        import pire_b200 as P
        self.sc = P.Scanner(image, 0)
        if max_hot is not None:
            self.sc.set_max_hot(max_hot)
        if variant is not None:
            self.sc.set_variant(variant)
        self.orc = Oracle(image)

    def string(self, dev, off, n, flags, start=None, start_ptr=None, stream=None):
        """pire_gpu_run_string -> (match word, mask, state); the other 63 words of every output must stay untouched."""
        import torch
        from pire_b200 import _native as N
        out = torch.full((3, 64), SENTINEL, dtype=torch.int32, device="cuda:0")
        if start is not None:
            word = start & 0xFFFFFFFF
            st = torch.tensor([word - (1 << 32) if word >= 1 << 31 else word], dtype=torch.int32, device="cuda:0")
            start_ptr = st.data_ptr()
        text = None if dev is None else dev.data_ptr() + off
        N.check(N.lib.pire_gpu_run_string(self.sc._h, text, n, flags, start_ptr, out[0].data_ptr(), out[1].data_ptr(),
                                          out[2].data_ptr(), stream or _stream()), "pire_gpu_run_string")
        o = out.cpu().numpy().view(np.uint32)
        assert (o[:, 1:] == SENTINEL).all(), "written past word 0"
        return tuple(int(x) for x in o[:, 0])

    def batch(self, dev, off, n, flags):
        import torch
        from pire_b200 import _native as N
        out = torch.full((3, 64), SENTINEL, dtype=torch.int32, device="cuda:0")
        offs = torch.tensor([off, off + n], dtype=torch.int64, device="cuda:0")
        N.check(N.lib.pire_gpu_run_batch(self.sc._h, dev.data_ptr(), offs.data_ptr(), 0, 1, flags, out[0].data_ptr(),
                                         out[1].data_ptr(), out[2].data_ptr(), _stream()), "pire_gpu_run_batch")
        o = out.cpu().numpy().view(np.uint32)
        return tuple(int(x) for x in o[:, 0])

    def check(self, dev, host, off, n, flags, start=None, what=""):
        got = self.string(dev, off, n, flags, start)
        want = run_from(self.orc, host[off:off + n], start, bool(flags & RUN_BEGIN), bool(flags & RUN_END))
        assert got == want, (what, off, n, flags, start, got, want)
        if start is None:
            assert self.batch(dev, off, n, flags) == got, (what, off, n, flags)
        return got


def text_buffer(size, alphabet, plants=(), every=997, seed=1):
    """Random bytes of `alphabet` with `plants` written every `every` bytes; (device tensor, host array)."""
    import torch
    rng = np.random.default_rng(seed)
    host = rng.choice(np.frombuffer(alphabet, np.uint8), size=size)
    for k, at in enumerate(range(every // 2, size - 64, every) if plants else ()):
        lit = np.frombuffer(plants[k % len(plants)], np.uint8)
        host[at:at + len(lit)] = lit
    return torch.from_numpy(host).to("cuda:0"), host


def glue10():
    from pire_b200 import workloads as W
    return W.load_image("glue10"), [p.lstrip(b"^$") for p in W.GLUE10_PLANTS]


def test_lengths_and_alignments(cuda_device):
    """Short lengths around the 16- and 32-byte edges, and lengths one block either side of the piece boundaries of a
    one-CTA grid, a few CTAs and the full grid (the piece rule's Python copy is asserted on each)."""
    image, plants = glue10()
    c = Checker(image)
    full = full_grid(c.sc.info().hot_rows)
    step = 32 * BLOCK * MIN_BLOCKS                        # bytes of body per CTA at the minimum piece length
    lens = [0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 8191, 8192, 8193]
    # one CTA: the body's 512 lanes get one block each, then two
    for n in (32 * BLOCK, 2 * 32 * BLOCK):
        assert pieces(n, 0, full)[:3] == (1, n // (32 * BLOCK), 0)
        assert pieces(n - 32, 0, full)[2] == BLOCK - 1 and pieces(n + 32, 0, full)[2] == 1
        lens += [n - 32, n, n + 32]
    # from one CTA to two, and three CTAs with pieces of exactly MIN_BLOCKS blocks
    assert ctas(step, full) == 1 and ctas(step + 32, full) == 2
    assert pieces(3 * step, 0, full) == (3, MIN_BLOCKS, 0) and pieces(3 * step + 32, 0, full)[0] == 4
    lens += [step - 32, step, step + 32, 3 * step - 32, 3 * step, 3 * step + 32]
    # the full grid, and past it (pieces grow instead of CTAs)
    assert ctas(full * step, full) == full and ctas(full * step - 32 * BLOCK * MIN_BLOCKS, full) == full - 1
    assert pieces(2 * full * step + 32, 0, full) == (full, 2 * MIN_BLOCKS, 1)
    lens += [full * step - 32, full * step, full * step + 32, 2 * full * step + 32]
    dev, host = text_buffer(max(lens) + 64, PRINTABLE, plants, every=4093)
    for n in lens:
        for off in (0, 13):
            c.check(dev, host, off, n, RUN_BEGIN | RUN_END, what="length")


def test_offsets_marks_and_straddling_plants(cuda_device):
    """Start offsets 0..31 with the four mark combinations, over a two-CTA grid whose pieces are 256 or 288 bytes: a
    plant every 256 bytes straddles the piece boundaries."""
    image, plants = glue10()
    c = Checker(image)
    n = 32 * BLOCK * MIN_BLOCKS + 32 * 7 + 5
    assert pieces(n, 0, full_grid(c.sc.info().hot_rows))[:2] == (2, 8)
    dev, host = text_buffer(n + 128, PRINTABLE, plants, every=256, seed=2)
    for off in range(32):
        for flags in MARKS:
            c.check(dev, host, off, n, flags, what="offset")


def image_cases():
    from pire_b200 import workloads as W
    g10 = glue10()
    cases = {"AppendixA": (next(x for x in GOLDEN if x.name == "AppendixA").image, PRINTABLE, [b"hello world", b"hello  wxd"]),
             "glue10": (g10[0], PRINTABLE, g10[1]),
             "headline_iu": (W.load_image("headline_iu"), PRINTABLE, [b"HeLLo \t WoRlD", b"hello wd"]),
             "parity": (STRING_IMAGES["parity"]["image"], b"a", []),
             "shift11": (STRING_IMAGES["shift11"]["image"], b"ab", [])}
    for name, e in EDGE.items():
        cases[name] = (e["image"], ALPHABETS[name], [b"foo", b"GET ", b"error"] if name in ("absorbing", "glued") else [])
    return cases


IMAGE_CASES = image_cases()


@pytest.mark.parametrize("name", sorted(IMAGE_CASES))
def test_images(cuda_device, name):
    image, alphabet, plants = IMAGE_CASES[name]
    c = Checker(image)
    dev, host = text_buffer(3_000_064, alphabet, plants, every=50_001, seed=3)
    for n in (3, 1000, 300_007, 3_000_011):
        for flags in (RUN_BEGIN | RUN_END, 0):
            c.check(dev, host, 5, n, flags, what=name)


def test_hot_sets_and_variants(cuda_device):
    """max_hot 255 / 6 / 2 / 1, static and tuned (on a fixed-length view), variants plain, exit filter and look-ahead."""
    import pire_b200 as P
    image, plants = glue10()
    dev, host = text_buffer(2_000_128, PRINTABLE, plants, every=3001, seed=4)
    for tuned in (False, True):
        c = Checker(image)
        if tuned:
            c.sc.Tune(P.Batch(dev[: len(host) // 4096 * 4096], fixed_len=4096))
        for max_hot in (255, 6, 2, 1):
            c.sc.set_max_hot(max_hot)
            for variant in (1, 2, 4):
                c.sc.set_variant(variant)
                for flags in (RUN_BEGIN | RUN_END, 0):
                    c.check(dev, host, 3, 2_000_003, flags, what=(tuned, max_hot, variant))


def test_resume_chained_in_place(cuda_device):
    """Random cuts (empty chunks and odd alignments included), chained through one device word updated in place: BEGIN on
    the first call, END on the last; the chain equals one call and the oracle."""
    import torch
    from pire_b200 import _native as N
    rng = np.random.default_rng(5)
    g10, g10_plants = glue10()
    for image, alphabet, plants in ((g10, PRINTABLE, g10_plants), (STRING_IMAGES["parity"]["image"], b"a", []),
                                    (STRING_IMAGES["shift11"]["image"], b"ab", [])):
        c = Checker(image)
        n = 3_000_017
        dev, host = text_buffer(n + 64, alphabet, plants, every=7919, seed=6)
        one = c.check(dev, host, 1, n, RUN_BEGIN | RUN_END, what="one call")
        for trial in range(4):
            cuts = np.sort(np.concatenate([[0, n], rng.integers(0, n, size=6), rng.integers(0, 40, size=2)]))
            cuts = np.concatenate([cuts[:3], cuts[2:3], cuts[3:]])          # an empty chunk
            out = torch.full((3, 64), SENTINEL, dtype=torch.int32, device="cuda:0")
            state = out[2].data_ptr()
            for k in range(len(cuts) - 1):
                flags = (RUN_BEGIN if k == 0 else 0) | (RUN_END if k == len(cuts) - 2 else 0)
                N.check(N.lib.pire_gpu_run_string(c.sc._h, dev.data_ptr() + 1 + int(cuts[k]), int(cuts[k + 1] - cuts[k]), flags,
                                                  None if k == 0 else state, out[0].data_ptr(), out[1].data_ptr(), state,
                                                  _stream()), "pire_gpu_run_string")
            o = out.cpu().numpy().view(np.uint32)
            assert (o[:, 1:] == SENTINEL).all()
            assert tuple(int(x) for x in o[:, 0]) == one, (trial, cuts)


def test_resume_from_every_state(cuda_device):
    """From every state of the AppendixA scanner, from cold states of glue10 with two hot rows, and from starts outside
    the scanner (also with d_start == d_state_idx)."""
    import torch
    from pire_b200 import _native as N
    case = next(x for x in GOLDEN if x.name == "AppendixA")
    c = Checker(case.image)
    dev, host = text_buffer(300_064, PRINTABLE, [b"hello world", b"world"], every=1001, seed=7)
    size = c.sc.Size()
    for st in range(size):
        for flags in MARKS:
            for n in (0, 7, 300_001):
                c.check(dev, host, 9, n, flags, start=st, what="AppendixA state")
    image, plants = glue10()
    c = Checker(image, max_hot=2)
    hot = set(static_hot_order(c.sc, 2))
    cold = [s for s in range(c.sc.Size()) if s not in hot][:: max(1, c.sc.Size() // 24)]
    assert len(cold) >= 12
    dev, host = text_buffer(700_064, PRINTABLE, plants, every=3001, seed=8)
    for st in cold:
        for flags in (0, RUN_BEGIN | RUN_END):
            c.check(dev, host, 3, 700_001, flags, start=st, what="cold start")
    for st in (c.sc.Size(), c.sc.Size() + 1, 0xFFFFFFFF):
        for flags in MARKS:
            assert c.string(dev, 0, 1000, flags, start=st) == (0, 0, 0xFFFFFFFF)
    # in place: the start word is the state word
    out = torch.full((3, 64), SENTINEL, dtype=torch.int32, device="cuda:0")
    out[2, 0] = -1
    N.check(N.lib.pire_gpu_run_string(c.sc._h, dev.data_ptr(), 700_000, RUN_END, out[2].data_ptr(), out[0].data_ptr(),
                                      out[1].data_ptr(), out[2].data_ptr(), _stream()), "pire_gpu_run_string")
    o = out.cpu().numpy().view(np.uint32)
    assert tuple(int(x) for x in o[:, 0]) == (0, 0, 0xFFFFFFFF) and (o[:, 1:] == SENTINEL).all()


def test_parity_worst_case(cuda_device):
    """Walks that never fall together: the stitch degrades to the serial walk and must still be exact.  Pieces are whole
    32-byte blocks, so the guess (the even state) is wrong in every piece only behind an odd head: offsets 1 and 3."""
    c = Checker(STRING_IMAGES["parity"]["image"])
    n = 16 * 2 ** 20 + 1
    dev, host = text_buffer(n + 64, b"a", seed=9)
    for off in (0, 1, 3):
        for flags in (RUN_BEGIN | RUN_END, 0):
            c.check(dev, host, off, n - off % 2, flags, what="parity")


def test_string_past_4_gib(cuda_device):
    """A string longer than 4 GiB, filled on the device; the oracle walks a host copy, one 256 MiB slice at a time.
    headline (hello\\s+w.+d$), with the one plant near the end: before it the walks fall together at once."""
    import torch
    from pire_b200 import workloads as W
    image = W.load_image("headline")
    c = Checker(image)
    n = 2 ** 32 + 4096 + 13
    dev = torch.empty((n + 1023) // 1024 * 1024, dtype=torch.uint8, device="cuda:0")
    try:
        W.SynthSpec(dev.numel() // 1024, 1024).fill_device(dev)
        plant = torch.frombuffer(bytearray(b"hello \t world d"), dtype=torch.uint8).to("cuda:0")
        dev[n - 5000:n - 5000 + plant.numel()] = plant
        for flags in (RUN_BEGIN | RUN_END, 0):
            got = c.string(dev, 0, n, flags)
            w = StringWalk(c.orc)
            if flags & RUN_BEGIN:
                w.Begin()
            for lo in range(0, n, 2 ** 28):
                w.Run(dev[lo:min(n, lo + 2 ** 28)].cpu().numpy())
            if flags & RUN_END:
                w.End()
            assert got == w.result(), flags
    finally:
        del dev
        torch.cuda.empty_cache()


def test_two_streams_one_handle(cuda_device):
    """Two strings on two streams at the same time, one handle: both exact."""
    import torch
    from pire_b200 import _native as N
    image, plants = glue10()
    c = Checker(image)
    n = 64 * 2 ** 20
    dev_a, host_a = text_buffer(n + 64, PRINTABLE, plants, every=100_003, seed=10)
    dev_b, host_b = text_buffer(n + 64, PRINTABLE, plants[::-1], every=77_777, seed=11)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [torch.full((3, 64), SENTINEL, dtype=torch.int32, device="cuda:0") for _ in range(2)]
    torch.cuda.synchronize()
    for rep in range(3):
        for s, dev, out in zip(streams, (dev_a, dev_b), outs):
            N.check(N.lib.pire_gpu_run_string(c.sc._h, dev.data_ptr() + rep, n - rep, RUN_BEGIN | RUN_END, None, out[0].data_ptr(),
                                              out[1].data_ptr(), out[2].data_ptr(), s.cuda_stream), "pire_gpu_run_string")
        torch.cuda.synchronize()
        for host, out in zip((host_a, host_b), outs):
            o = out.cpu().numpy().view(np.uint32)
            assert (o[:, 1:] == SENTINEL).all()
            assert tuple(int(x) for x in o[:, 0]) == run_from(c.orc, host[rep:n], None, True, True)


def test_arguments_and_empty_scanner(cuda_device):
    import torch
    from pire_b200 import _native as N
    image, _ = glue10()
    c = Checker(image)
    dev = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    for flags in (4, 8, 1 << 31, RUN_BEGIN | 4):
        assert N.lib.pire_gpu_run_string(c.sc._h, dev.data_ptr(), 10, flags, None, None, None, None, _stream()) == -1
    assert N.lib.pire_gpu_run_string(c.sc._h, None, 1, RUN_BEGIN, None, None, None, None, _stream()) == -1
    assert N.lib.pire_gpu_run_string(None, dev.data_ptr(), 1, 0, None, None, None, None, _stream()) == -1
    # zero-length strings, with and without a text pointer; all outputs NULL is legal
    for flags in MARKS:
        assert c.string(None, 0, 0, flags) == run_from(c.orc, np.zeros(0, np.uint8), None, bool(flags & 1), bool(flags & 2))
        assert c.string(dev, 0, 0, flags) == c.batch(dev, 0, 0, flags)
    N.check(N.lib.pire_gpu_run_string(c.sc._h, dev.data_ptr(), 64, 3, None, None, None, None, _stream()), "all outputs NULL")
    empty = next(x for x in GOLDEN if x.name == "EmptyScanner@784")
    e = Checker(empty.image)
    dev, host = text_buffer(100_064, PRINTABLE, seed=12)
    for flags in MARKS:
        for n in (0, 5, 100_000):
            e.check(dev, host, 0, n, flags, what="empty scanner")
        e.check(dev, host, 0, 1000, flags, start=0, what="empty scanner, from state 0")


def test_python_string_runner(cuda_device):
    import pire_b200 as P
    image, plants = glue10()
    c = Checker(image)
    n = 5_000_003
    dev, host = text_buffer(n + 64, PRINTABLE, plants, every=100_003, seed=13)
    want = run_from(c.orc, host[:n], None, True, True)
    cuts = [0, 0, 1, 33, 1_000_000, 1_000_000, 4_000_001, n]
    r = P.StringRunner(c.sc).Begin()
    for lo, hi in zip(cuts, cuts[1:]):
        r.Run(dev[lo:hi])
    r.End()
    ids = c.sc.AcceptedRegexps(want[2])
    assert (int(r.Final()), r.AcceptMask(), r.State()) == want and bool(r) == bool(want[0]) and r.AcceptedRegexps() == ids
    # Runner(sc, st): the first half without End(), the rest from the state reached
    half = P.StringRunner(c.sc).Begin().Run(dev[: n // 2])
    st = half.State()
    assert st == run_from(c.orc, host[: n // 2], None, True, False)[2]
    rest = P.StringRunner(c.sc, st).Run(dev[n // 2: n]).End()
    assert (int(rest.Final()), rest.AcceptMask(), rest.State()) == want
    assert P.StringRunner(c.sc, c.sc.Size()).Begin().Run(dev[:100]).End().State() == 0xFFFFFFFF
    assert P.StringRunner(c.sc).State() == run_from(c.orc, host[:0], None, False, False)[2]


def test_python_string_runner_reuses_one_buffer(cuda_device):
    """A text arriving in chunks through ONE staging buffer, refilled behind each Run() in stream order: every chunk
    must be scanned as it was when Run() was called."""
    import torch
    import pire_b200 as P
    image, plants = glue10()
    c = Checker(image)
    n = 3_000_017
    dev, host = text_buffer(n + 64, PRINTABLE, plants, every=50_021, seed=14)
    cuts = [0, 7, 1_000_003, 1_000_003, 1_500_000, 2_999_000, n]
    buf = torch.empty(max(b - a for a, b in zip(cuts, cuts[1:])) + 16, dtype=torch.uint8, device="cuda:0")
    for begin, end in ((True, True), (False, False), (True, False)):
        r = P.StringRunner(c.sc)
        if begin:
            r.Begin()
        for lo, hi in zip(cuts, cuts[1:]):
            buf[: hi - lo].copy_(dev[lo:hi])
            r.Run(buf[: hi - lo])
        if end:
            r.End()
        assert (int(r.Final()), r.AcceptMask(), r.State()) == run_from(c.orc, host[:n], None, begin, end), (begin, end)


def test_cpp_string_runner(tmp_path, cuda_device):
    """tests/cpp/string_check.cpp through include/pire_gpu.hpp's StringRunner: one call, a chain through one device word,
    pire_gpu_run_batch, and a resumed runner agree."""
    from pire_b200 import workloads as W
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "string_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "string_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    image = tmp_path / "glue10.pire"
    image.write_bytes(W.load_image("glue10"))
    for n, seed in ((50_000_017, 1), (1000, 2), (0, 3)):
        out = subprocess.run([exe, str(image), str(n), str(seed)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout + out.stderr
        assert ": 0 mismatches" in out.stdout
