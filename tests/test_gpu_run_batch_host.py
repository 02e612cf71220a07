"""pire_gpu_run_batch_host, called through ctypes so that any output may be NULL, against the reference and against
the same batch resident in HBM (pire_gpu_run_batch / pire_gpu_run_lines), whose results the call promises to equal.

The host call has machinery of its own: it cuts a batch into chunks of whole 32-string units, rebases each chunk's CSR
offsets, stages pageable input through pinned slots with a pool of copy threads (pinned input is DMA-ed from the
caller's buffer), packs the outputs it was asked for into one buffer per slot, and picks one of three device calls per
chunk (length-binned CSR, lines, plain).  Small chunks (PIRE_B200_HOST_CHUNK_MB, read on every call) put chunk and
tail edges, unbinned chunks of 32 strings and strings longer than a chunk into batches of a few MiB.

Every output array is padded with sentinel words past ceil(n / 32) or n, and they must survive every call, failed
ones included."""
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

from refpire import Oracle, csr
from test_edge_images import ALPHABETS, EDGE, static_hot_order

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
EINVAL = -1
BeginMark = 258
SENTINEL = 0xC3A5C3A5
PAD = 9                                    # sentinel words past every output
MARKS = ((True, True), (False, False), (True, False), (False, True))
OUTPUTS = [(b, m, s) for b in (True, False) for m in (True, False) for s in (True, False)]     # all 8 subsets
ALL = (True, True, True)
PRINTABLE = bytes(range(0x20, 0x7F))
LITERALS = [b"GET /index", b"timeout", b"error 42", b"(555) 123-4567", b"https://x", b"fatal", b"hello \t world",
            b"XABCDEFGHIJKLMNOPQRSTUVWXYZ", b"GET /", b"a timeout"]


def flags_of(begin, end, lines=False):
    return (RUN_BEGIN if begin else 0) | (RUN_END if end else 0) | (RUN_LINES if lines else 0)


def ptr(a):
    return None if a is None else a.ctypes.data


# ------------------------------------------------------------------------------------------------------------ calls

def host_call(sc, corpus, corpus_bytes, offsets, fixed_len, n, flags, want=ALL):
    """The C call with the outputs `want` (bits, masks, states) and NULL for the others: (rc, outputs)."""
    from pire_b200 import _native as N
    sizes = ((n + 31) // 32, n, n)
    outs = [np.full(k + PAD, SENTINEL, np.uint32) if w else None for k, w in zip(sizes, want)]
    rc = N.lib.pire_gpu_run_batch_host(sc._h, ptr(corpus), corpus_bytes, ptr(offsets), fixed_len, n, flags, *map(ptr, outs))
    for a, k in zip(outs, sizes):
        assert a is None or (a[k:] == SENTINEL).all(), "a word past the output was written"
    return rc, [None if a is None else a[:k] for a, k in zip(outs, sizes)]


def run_host(sc, corpus, corpus_bytes, offsets, fixed_len, n, flags, want=ALL):
    from pire_b200 import _native as N
    rc, outs = host_call(sc, corpus, corpus_bytes, offsets, fixed_len, n, flags, want)
    N.check(rc, "pire_gpu_run_batch_host")
    return outs


def device_run(sc, corpus, offsets, fixed_len, n, flags):
    """The same batch resident in HBM: pire_gpu_run_lines for LINES, else pire_gpu_run_batch; all three outputs."""
    import torch
    from pire_b200 import _native as N
    size = 0 if corpus is None else len(corpus)
    data = np.zeros(size + 64, np.uint8)
    data[:size] = corpus if size else 0
    d_corpus = torch.from_numpy(data).to("cuda:0")
    d_off = None if offsets is None else torch.from_numpy(np.asarray(offsets, np.uint64).view(np.int64)).to("cuda:0")
    sizes = ((n + 31) // 32, n, n)
    outs = [torch.from_numpy(np.full(k + PAD, SENTINEL, np.uint32).view(np.int32)).to("cuda:0") for k in sizes]
    stream = torch.cuda.current_stream().cuda_stream
    if flags & RUN_LINES:
        rc = N.lib.pire_gpu_run_lines(sc._h, d_corpus.data_ptr(), d_off.data_ptr(), None, n, flags,
                                      *[o.data_ptr() for o in outs], stream)
    else:
        rc = N.lib.pire_gpu_run_batch(sc._h, d_corpus.data_ptr(), None if d_off is None else d_off.data_ptr(), fixed_len, n,
                                      flags, *[o.data_ptr() for o in outs], stream)
    N.check(rc, "pire_gpu_run_lines" if flags & RUN_LINES else "pire_gpu_run_batch")
    torch.cuda.synchronize()
    got = [o.cpu().numpy().view(np.uint32) for o in outs]
    for a, k in zip(got, sizes):
        assert (a[k:] == SENTINEL).all()
    return [a[:k] for a, k in zip(got, sizes)]


def pack(final):
    n = len(final)
    b = np.zeros((n + 31) // 32 * 32, np.uint8)
    b[:n] = final
    return np.packbits(b, bitorder="little").view(np.uint32)


def reference(sc_ref, corpus, offsets, fixed_len, n, begin, end, lines=False):
    """(bits, masks, states) of Runner(sc).[Begin()].Run(s).[End()] per string; a line is its bytes without the '\\n'."""
    if lines:
        strings = [bytes(corpus[int(offsets[i]): int(offsets[i + 1]) - 1]) for i in range(n)]
        c, o = csr(strings)
        final, masks, states = sc_ref.run(c, o, begin=begin, end=end, threads=8)
    elif offsets is None and fixed_len == 0:
        c, o = csr([b""] * n)
        final, masks, states = sc_ref.run(c, o, begin=begin, end=end, threads=8)
    else:
        final, masks, states = sc_ref.run(corpus, offsets, fixed_len=fixed_len, n=n, begin=begin, end=end, threads=8)
    return [pack(final), masks, states]


def check(sc, sc_ref, corpus, corpus_bytes, offsets, fixed_len, n, begin, end, lines=False, outputs=(ALL,), want=None,
          label=""):
    """The host call equals the reference and the resident batch, for each output subset in `outputs`."""
    flags = flags_of(begin, end, lines)
    if want is None:
        want = reference(sc_ref, corpus, offsets, fixed_len, n, begin, end, lines)
    dev = device_run(sc, corpus, offsets, fixed_len, n, flags)
    for w, d, name in zip(want, dev, ("bits", "masks", "states")):
        assert (w == d).all(), ("resident", name, label)
    for subset in outputs:
        got = run_host(sc, corpus, corpus_bytes, offsets, fixed_len, n, flags, subset)
        for g, w, name in zip(got, want, ("bits", "masks", "states")):
            if g is not None:
                bad = np.flatnonzero(g != w)
                assert bad.size == 0, (label, name, subset, bad[:5], g[bad[:5]], w[bad[:5]])
    return want


# ----------------------------------------------------------------------------------------------------------- inputs

def random_bytes(rng, size, alphabet=PRINTABLE, literals=LITERALS, every=60):
    """`size` bytes of `alphabet` with a literal written about every `every` bytes."""
    buf = np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), size=size)]
    for at in rng.integers(0, max(1, size), size=size // every):
        lit = np.frombuffer(literals[int(rng.integers(0, len(literals)))], np.uint8)
        buf[int(at): int(at) + len(lit)] = lit[: size - int(at)]
    return buf


def ragged(rng, lens, lead=0, alphabet=PRINTABLE, literals=LITERALS):
    """A CSR batch of strings of lengths `lens` whose first string starts `lead` bytes into the corpus."""
    offs = np.zeros(len(lens) + 1, np.uint64)
    np.cumsum(np.asarray(lens, np.uint64), out=offs[1:])
    offs += lead
    corpus = random_bytes(rng, int(offs[-1]) + 13, alphabet, literals)
    for i in range(0, len(lens), 3):                  # whole strings that are literals, for the anchored patterns
        if lens[i] >= 5:
            lit = np.frombuffer(literals[int(rng.integers(0, len(literals)))], np.uint8)
            corpus[int(offs[i + 1]) - min(len(lit), lens[i]): int(offs[i + 1])] = lit[-min(len(lit), lens[i]):]
    return corpus, offs


def text_lines(rng, n_lines, ending, long_len, alphabet=PRINTABLE, literals=LITERALS):
    """A text of lines, as _text_of in test_gpu_parity: empty lines, a run of them, lines that are literals, one line
    of `long_len` bytes; ending b'\\n' or b''."""
    lines = []
    for _ in range(n_lines):
        r = rng.random()
        if r < 0.15:
            lines.append(b"")
        elif r < 0.35:
            lines.append(literals[int(rng.integers(0, len(literals)))])
        else:
            lines.append(bytes(random_bytes(rng, int(rng.integers(1, 90)), alphabet, literals)))
    lines = [ln.replace(b"\n", b" ") for ln in lines]
    for k in range(n_lines // 4, n_lines // 4 + 40):
        lines[k] = b""
    lines[n_lines // 2] = bytes(random_bytes(rng, long_len, alphabet, literals)).replace(b"\n", b" ")
    lines[-1] = lines[-1] or b"timeout"
    return b"\n".join(lines) + ending


def getline_offsets(text):
    """std::getline over `text`: line i is text[o[i] : o[i+1] - 1]; a last line without '\\n' ends at len(text)."""
    nl = np.flatnonzero(np.frombuffer(text, np.uint8) == 10).astype(np.uint64) + 1
    offs = np.concatenate([np.zeros(1, np.uint64), nl])
    if text and not text.endswith(b"\n"):
        offs = np.append(offs, np.uint64(len(text) + 1))
    return offs


def device_line_offsets(text):
    import torch
    import pire_b200 as P
    batch = P.Batch.from_text(torch.from_numpy(np.frombuffer(text, np.uint8).copy()).to("cuda:0"))
    return batch.offsets.cpu().numpy().view(np.uint64).copy()


def csr_chunks(offs, n, chunk_bytes):
    """The chunks pire_gpu_run_batch_host cuts a CSR batch into: [(first, last)]."""
    out, first = [], 0
    while first < n:
        lo, last = int(offs[first]), first
        while True:
            last = min(n, last + 32)
            if not (last < n and int(offs[min(n, last + 32)]) - lo <= chunk_bytes):
                break
        out.append((first, last))
        first = last
    return out


def pinned_copy(data):
    import torch
    t = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
    arr = t.numpy()
    arr[:] = data
    return t, arr


class OracleRef:
    """The in-repo oracle with the reference's run() signature, for images the reference did not compile."""

    def __init__(self, image):
        self.o = Oracle(image)

    def run(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, threads=1):
        return self.o.run(corpus, offsets, fixed_len=fixed_len, n=n, begin=begin, end=end)


@pytest.fixture(scope="module")
def scanners(ref, cuda_device):
    """name -> (reference, device scanner, alphabet, literals)."""
    import pire_b200 as P
    from pire_b200 import workloads as W
    out = {"glue10": (ref.glue_all(W.GLUE10), P.Scanner(W.load_image("glue10"), cuda_device), PRINTABLE, LITERALS)}
    anchored = ref.compile(rb"^GET /[a-z]*$|^timeout$", "")
    out["anchored"] = (anchored, P.Scanner(anchored.save(), cuda_device), PRINTABLE, LITERALS)
    every = ref.compile(rb".*", "")
    out["every"] = (every, P.Scanner(every.save(), cuda_device), PRINTABLE, LITERALS)
    # an edge image with one hot row, outside which a run without Begin() starts (the cold start)
    image = EDGE["anchored"]["image"]
    host = P.Scanner(image, -1)
    assert host.Initialize() not in set(static_hot_order(host, 1))
    edge = P.Scanner(image, cuda_device)
    edge.set_max_hot(1)
    out["edge_anchored"] = (OracleRef(image), edge, ALPHABETS["anchored"], [b"abcd", b"abcde", b"cdabe", b"ababe"])
    return out


# ------------------------------------------------------------------------------------------------------------ tests

def test_fixed_length_shapes(scanners, monkeypatch):
    """Lengths 0, 1, 31, 32, 100, 1024 and one longer than a chunk (chunks of 32 strings then), n around multiples of
    32 and around a chunk's string count; chunks whose string count is rounded down to a multiple of 32."""
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "1")
    sc_ref, sc, _, _ = scanners["glue10"]
    rng = np.random.default_rng(11)
    chunk = 1 << 20
    for length in (1, 31, 32, 100, 1024, chunk + 100):
        per = max(32, chunk // length // 32 * 32)
        ns = sorted({31, 33, per - 1, per + 1, 3 * per + 5} if length < chunk else {1, 33})
        for n in ns:
            corpus = random_bytes(rng, n * length + 5)
            check(sc, sc_ref, corpus, n * length, None, length, n, True, True, label=(length, n))
    # every mark combination and every output subset where chunks hold a rounded-down count (33824 strings of 31)
    per = chunk // 31 // 32 * 32
    n = 2 * per + 77
    corpus = random_bytes(rng, n * 31)
    for begin, end in MARKS:
        check(sc, sc_ref, corpus, len(corpus), None, 31, n, begin, end, outputs=OUTPUTS, label=("marks", begin, end))
    # fixed_len 0: n empty strings, with and without a corpus
    for n in (1, 31, 32, 33, 1000):
        want = check(sc, sc_ref, None, 0, None, 0, n, True, True, outputs=OUTPUTS, label=("empty", n))
        got = run_host(sc, np.zeros(7, np.uint8), 7, None, 0, n, flags_of(True, True))
        assert all((g == w).all() for g, w in zip(got, want))


def test_csr_shapes(scanners, monkeypatch):
    """CSR batches that start past the corpus's first byte, with empty strings, of fewer than 64 strings, with chunks of
    32 strings (not binned) and binned chunks holding a string of 8 KiB and more (the split kernel); n around multiples
    of 32."""
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "1")
    sc_ref, sc, _, _ = scanners["glue10"]
    rng = np.random.default_rng(12)
    chunk = 1 << 20
    for n in (1, 31, 32, 33, 63, 64, 65, 95, 97):
        lens = rng.integers(0, 300, size=n)
        lens[::7] = 0
        for lead in (0, 16, 4099):
            corpus, offs = ragged(rng, lens, lead)
            check(sc, sc_ref, corpus, len(corpus), offs, 0, n, True, True, outputs=OUTPUTS if lead == 16 else (ALL,),
                  label=("small", n, lead))
    # strings of about 20 KiB: chunks of 32 strings, each launched unbinned; then a tail of 5
    lens = rng.integers(18 << 10, 24 << 10, size=32 * 5 + 5)
    corpus, offs = ragged(rng, lens, 3)
    chunks = csr_chunks(offs, len(lens), chunk)
    assert len(chunks) >= 4 and all(b - a == 32 for a, b in chunks[:-1]) and chunks[-1][1] - chunks[-1][0] < 64
    check(sc, sc_ref, corpus, len(corpus), offs, 0, len(lens), True, True, label="unbinned chunks")
    # binned chunks of hundreds of strings, some of 8 KiB and more, empty ones, one longer than a chunk
    lens = np.concatenate([rng.integers(0, 3000, size=2500), [8192, 8193, 9000, 12345, 20000, 0, 0, 0, chunk + 5]])
    rng.shuffle(lens)
    for n in (len(lens), len(lens) - 38):
        corpus, offs = ragged(rng, lens[:n], 77)
        chunks = csr_chunks(offs, n, chunk)
        assert any(b - a >= 64 and (np.diff(offs[a:b + 1].astype(np.int64)) >= 8192).any() for a, b in chunks)
        check(sc, sc_ref, corpus, len(corpus), offs, 0, n, True, True, outputs=OUTPUTS[:4], label=("binned", n))


@pytest.mark.parametrize("name", ["glue10", "anchored", "every", "edge_anchored"])
def test_flags_lines_and_outputs(name, scanners, monkeypatch):
    """Every mark combination with and without RUN_LINES on the lines of texts with and without a final newline, with
    a line longer than a chunk and runs of empty lines: the line batch (offsets from getline on the host, equal to
    those pire_gpu_split_lines finds, corpus_bytes = the text's size) and the same lines as a plain CSR batch.  Every
    output subset for one mark combination."""
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "1")
    sc_ref, sc, alphabet, literals = scanners[name]
    rng = np.random.default_rng(len(name))
    for ending in (b"\n", b""):
        text = text_lines(rng, 80000, ending, (1 << 20) + 3000, alphabet, literals)
        offs = getline_offsets(text)
        assert (device_line_offsets(text) == offs).all()
        n = len(offs) - 1
        assert len(csr_chunks(offs, n, 1 << 20)) >= 4
        corpus = np.frombuffer(text, np.uint8).copy()
        lines = [text[int(offs[i]): int(offs[i + 1]) - 1] for i in range(n)]
        assert lines == (text.split(b"\n")[:-1] if ending else text.split(b"\n"))
        c, o = csr(lines)
        for begin, end in MARKS:
            outputs = OUTPUTS if (begin, end) == (True, False) else (ALL,)
            want = check(sc, sc_ref, corpus, len(text), offs, 0, n, begin, end, lines=True, outputs=outputs,
                         label=(name, ending, begin, end, "lines"))
            check(sc, sc_ref, c, len(c), o, 0, n, begin, end, outputs=outputs, want=want,
                  label=(name, ending, begin, end, "csr"))
            if name == "anchored" and begin and end:
                assert 0 < int(np.unpackbits(want[0].view(np.uint8)).sum()) < n


@pytest.mark.parametrize("kind", ["pageable_1", "pageable_6", "pinned", "registered", "pinned_staged"])
def test_input_memory(kind, scanners, monkeypatch):
    """Pageable input staged by a pool of one and of six threads with 5 MiB chunks (three pieces per chunk), pinned
    torch memory and cudaHostRegister-ed numpy memory DMA-ed from the caller's buffer, and pinned input staged anyway
    (PIRE_B200_HOST_FORCE_STAGING): a fixed-length batch, a CSR batch that starts past the buffer's first byte, and a
    text without a final newline in a buffer of exactly its size."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "5")
    monkeypatch.setenv("PIRE_B200_HOST_THREADS", kind.split("_")[1] if kind.startswith("pageable") else "4")
    if kind == "pinned_staged":
        monkeypatch.setenv("PIRE_B200_HOST_FORCE_STAGING", "1")
    sc_ref = scanners["glue10"][0]
    sc = P.Scanner(W.load_image("glue10"), 0)                     # a fresh handle: its pool takes the thread count
    rng = np.random.default_rng(13)
    n_fixed = 5 * 5120 + 37
    fixed = random_bytes(rng, n_fixed * 1024)
    corpus, offs = ragged(rng, rng.integers(0, 2500, size=9000), 1000)
    text = text_lines(rng, 60000, b"", 7 << 20)
    line_offs = getline_offsets(text)
    batches = [(fixed, None, 1024, n_fixed, False), (corpus, offs, 0, len(offs) - 1, False),
               (np.frombuffer(text, np.uint8), line_offs, 0, len(line_offs) - 1, True)]
    for data, o, fixed_len, n, lines in batches:
        want = reference(sc_ref, data, o, fixed_len, n, True, True, lines)
        keep, registered = None, None
        if kind in ("pinned", "pinned_staged"):
            keep, buf = pinned_copy(data)
        elif kind == "registered":
            raw = np.empty(len(data) + 4096, np.uint8)
            at = (-raw.ctypes.data) % 4096
            buf = raw[at: at + len(data)]
            buf[:] = data
        else:
            buf = np.array(data, np.uint8)
        try:
            if kind == "registered":
                rc = torch.cuda.cudart().cudaHostRegister(buf.ctypes.data, buf.nbytes, 0)
                assert int(rc) == 0, rc
                registered = buf.ctypes.data
            check(sc, sc_ref, buf, len(buf), o, fixed_len, n, True, True, lines, outputs=((True, True, False), ALL),
                  want=want, label=(kind, fixed_len, lines))
        finally:
            if registered is not None:
                torch.cuda.cudart().cudaHostUnregister(registered)
        del keep


@pytest.mark.parametrize("variant", [1, 2, 4, 7, "tuned"], ids=["plain", "pred", "look", "look_ring1", "autoselect"])
def test_variants_through_chunks(variant, scanners, monkeypatch):
    """The kernel variants on a uniform fixed-length corpus cut into chunks, and the handle after Tune and AutoSelect
    on that corpus resident in HBM."""
    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "1")
    sc_ref = scanners["glue10"][0]
    sc = P.Scanner(W.load_image("glue10"), 0)
    n = 3 * 1024 + 40
    corpus = W.SynthSpec(n, 1024, plants=W.GLUE10_PLANTS).host_sample(0, n)
    if variant == "tuned":
        batch = P.Batch(torch.from_numpy(corpus.copy()).to("cuda:0"), fixed_len=1024, n=n)
        sc.Tune(batch, 2048)
        sc.AutoSelect(batch)
    else:
        sc.set_variant(variant)
    want = reference(sc_ref, corpus, None, 1024, n, True, True)
    assert 0 < int(np.unpackbits(want[0].view(np.uint8)).sum()) < n
    for begin, end in MARKS:
        check(sc, sc_ref, corpus, len(corpus), None, 1024, n, begin, end, outputs=((True, False, True), ALL),
              want=want if begin and end else None, label=(variant, begin, end))


def test_workspace_reuse_threads_and_failure(scanners, monkeypatch):
    """One handle: calls that grow and then shrink the chunk shape and change their outputs; four threads at once, each
    with its own shape, flags and outputs; a call refused in its third chunk (offsets step back there) after two chunks
    were launched, then a good call on the same handle."""
    from pire_b200 import _native as N
    sc_ref, sc, _, _ = scanners["glue10"]
    rng = np.random.default_rng(14)
    small = random_bytes(rng, 3000 * 100)
    big = random_bytes(rng, 12000 * 1024)
    corpus, offs = ragged(rng, rng.integers(0, 3000, size=4000), 5)
    text = text_lines(rng, 20000, b"", 3000)
    line_offs = getline_offsets(text)
    tbuf = np.frombuffer(text, np.uint8).copy()
    calls = [  # (chunk MB, corpus, offsets, fixed_len, n, begin, end, lines, outputs)
        ("1", small, None, 100, 3000, True, True, False, ALL),
        ("5", big, None, 1024, 12000, False, True, False, (True, True, False)),
        ("1", corpus, offs, 0, 4000, True, False, False, (False, True, True)),
        ("2", tbuf, line_offs, 0, len(line_offs) - 1, True, True, True, (False, False, True)),
        ("1", small[:31 * 100], None, 100, 31, True, True, False, (True, False, False)),
        ("5", big, None, 1024, 12000, True, True, False, ALL),
    ]
    wants = [reference(sc_ref, c, o, fl, n, b, e, ln) for _, c, o, fl, n, b, e, ln, _ in calls]
    for (mb, c, o, fl, n, b, e, ln, out), want in zip(calls, wants):
        monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", mb)
        check(sc, sc_ref, c, len(c), o, fl, n, b, e, ln, outputs=(out,), want=want, label=("sequence", mb, fl, n))

    # threads: each repeats its call; the chunk size is the same for all of them
    monkeypatch.setenv("PIRE_B200_HOST_CHUNK_MB", "1")
    errors = []

    def work(k):
        _, c, o, fl, n, b, e, ln, out = calls[k]
        try:
            for _ in range(3):
                got = run_host(sc, c, len(c), o, fl, n, flags_of(b, e, ln), out)
                for g, w in zip(got, wants[k]):
                    assert g is None or (g == w).all(), k
        except Exception as ex:                                     # noqa: BLE001  (reported below)
            errors.append((k, repr(ex)))
    ts = [threading.Thread(target=work, args=(k,)) for k in (0, 1, 2, 3)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors, errors

    # refused in its third chunk: offsets step back inside it; the first two chunks were already launched
    chunks = csr_chunks(offs, 4000, 1 << 20)
    assert len(chunks) >= 4
    a, b = chunks[2]
    bad = offs.copy()
    k = (a + b) // 2
    bad[k] = bad[k + 1] + 1
    rc, _ = host_call(sc, corpus, len(corpus), bad, 0, 4000, flags_of(True, True))
    assert rc == EINVAL, rc
    assert b"ascending" in N.lib.pire_gpu_last_error()
    _, c, o, fl, n, b_, e, ln, _ = calls[2]
    got = run_host(sc, c, len(c), o, fl, n, flags_of(b_, e, ln))
    assert all((g == w).all() for g, w in zip(got, wants[2]))


def test_refusals(scanners):
    """A line batch whose text is shorter than offsets[n] - 1, offsets past the corpus, and unknown flag bits are
    refused; a line batch that needs exactly corpus_bytes is not."""
    sc_ref, sc, _, _ = scanners["anchored"]
    text = np.frombuffer(b"GET /a\ntimeout\nx", np.uint8).copy()
    offs = getline_offsets(bytes(text))
    assert int(offs[-1]) == len(text) + 1
    lines = flags_of(True, True, True)
    rc, _ = host_call(sc, text, len(text) - 1, offs, 0, 3, lines)
    assert rc == EINVAL
    got = run_host(sc, text, len(text), offs, 0, 3, lines)
    assert [int(got[0][0]) & 7] == [3]                              # "GET /a" and "timeout"; "x" does not match
    rc, _ = host_call(sc, text, len(text), offs, 0, 3, flags_of(True, True))   # without LINES the last string ends past it
    assert rc == EINVAL
    for flags in (8, 16, 1 << 31, RUN_BEGIN | 32):
        for n in (0, 3):
            rc, _ = host_call(sc, text, len(text), offs, 0, n, flags)
            assert rc == EINVAL, (flags, n)


def test_matches_host_from_cpp(tmp_path, scanners):
    """Pire::Gpu::MatchesHost (include/pire_gpu.hpp) from plain C++ on a device: a CSR batch, and the lines of a text
    without a final newline, read from a buffer of exactly the text's size."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not present")
    exe = str(tmp_path / "host_check")
    lib_dir = os.path.join(ROOT, "pire_b200")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(HERE, "cpp", "host_check.cpp"),
                    os.path.join(lib_dir, "libpire_b200.so"), "-o", exe, "-Xlinker", "-rpath=" + lib_dir], check=True)
    sc_ref, sc, _, _ = scanners["anchored"]
    (tmp_path / "sc.pire").write_bytes(sc_ref.save())
    rng = np.random.default_rng(15)
    corpus, offs = csr(text_lines(rng, 3000, b"\n", 200).split(b"\n"))
    text = text_lines(rng, 5000, b"", 200)
    line_offs = getline_offsets(text)
    cases = [("csr", corpus.tobytes(), offs, flags_of(True, True), False),
             ("lines", text, line_offs, flags_of(True, True, True), True)]
    for label, data, o, flags, lines in cases:
        n = len(o) - 1
        want = reference(sc_ref, np.frombuffer(data, np.uint8), o, 0, n, True, True, lines)
        final = np.unpackbits(want[0].view(np.uint8), bitorder="little")[:n]
        assert 0 < int(final.sum()) < n
        (tmp_path / "corpus").write_bytes(data)
        (tmp_path / "offsets").write_bytes(o.astype("<u8").tobytes())
        (tmp_path / "expected").write_bytes(final.astype(np.uint8).tobytes())
        out = subprocess.run([exe, str(tmp_path / "sc.pire"), str(tmp_path / "corpus"), str(tmp_path / "offsets"),
                              str(tmp_path / "expected"), str(flags)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, (label, out.stdout + out.stderr)
        assert "%d strings: 0 mismatches" % n in out.stdout, label
