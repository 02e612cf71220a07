"""A small pass through every kernel of the library, for compute-sanitizer:
    compute-sanitizer --tool memcheck  python tools/sanitize_run.py
    compute-sanitizer --tool racecheck python tools/sanitize_run.py
Checks results against the oracle on the way (bit-exact)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch
import pire_b200 as P
from pire_b200 import _native as N
from pire_b200 import workloads as W
from refpire import Oracle, csr

dev = "cuda:0"


def check(sc, orc, batch, corpus_host, offsets_host, fixed_len, n, tag):
    f, m, s = orc.run(corpus_host, offsets_host, fixed_len=fixed_len, n=n, shortcuts=True)
    for variant in (N.VARIANT_PLAIN, N.VARIANT_PRED, N.VARIANT_PRIV, N.VARIANT_LOOK, N.VARIANT_LOOK64, N.VARIANT_LOOK1):
        sc.set_variant(variant)
        r = P.Runner(sc).Begin().Run(batch).End()
        assert (r.Matches().astype(np.uint8) == f).all() and (r.AcceptMasks() == m).all() and (r.States() == s).all(), (tag, variant)
    print("ok", tag, "n=%d matches=%d" % (n, int(f.sum())), flush=True)


# glued 10-pattern scanner, fixed-length strings: uniform kernels incl. PRIV, tune, tiny hot sets (replay/cold paths)
img = W.load_image("glue10")
orc = Oracle(img)
sc = P.Scanner(img, 0)
n = 2048 + 3
spec = W.SynthSpec(n, 256, plants=W.GLUE10_PLANTS)
d = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
spec.fill_device(d)
host = spec.host_sample(0, n)
batch = P.Batch(d, fixed_len=256, n=n)
check(sc, orc, batch, host, None, 256, n, "glue10 static")
sc.Tune(batch, 512)
check(sc, orc, batch, host, None, 256, n, "glue10 tuned")
sc.set_max_hot(3)
check(sc, orc, batch, host, None, 256, n, "glue10 hot=3")
print(sc.AutoSelect(batch))
# the same batch through glue10 (hot=3) and a full glue10 handle at once (ScanPairKernel), against the oracle
full = P.Scanner(img, 0)
pr = P.Runner(P.ScannerPair(sc, full)).Begin().Run(batch).End()
f, m, s = orc.run(host, None, fixed_len=256, n=n, shortcuts=True)
for half in (pr.First(), pr.Second()):
    assert (half.Matches().astype(np.uint8) == f).all() and (half.AcceptMasks() == m).all() and (half.States() == s).all(), "pair"
print("ok pair n=%d" % n, flush=True)

# UTF-8 scanner, ragged CSR batch: generic kernels, ordered launch, host entry point
img = W.load_image("headline_iu")
orc = Oracle(img)
sc = P.Scanner(img, 0)
mspec = W.MixedSpec(1500)
mc, mo = mspec.device_batch(dev)
hc, ho = mspec.host_batch(0, 1500)
b = P.Batch(mc, mo, n=1500)
check(sc, orc, b, hc, ho, 0, 1500, "mixed unordered")
b.bin_by_length()
check(sc, orc, b, hc, ho, 0, 1500, "mixed binned")
bits, masks, states = sc.run_batch_host(hc, offsets=ho, want_masks=True, want_states=True)
f, m, s = orc.run(hc, ho)
assert (np.unpackbits(bits.view(np.uint8), bitorder="little")[:1500] == f).all() and (states == s).all()
# the lines of a text without a final newline, from a buffer of exactly its size: the last line's virtual separator
# lies one byte past the text, and nothing may be read there
text = b"\n".join(b"line %d hello  world" % i if i % 5 else b"" for i in range(3000)) + b"\nlast hello world"
htext = np.frombuffer(text, np.uint8).copy()
hl = np.concatenate([[0], np.flatnonzero(htext == 10) + 1, [len(text) + 1]]).astype(np.uint64)
bits, _, states = sc.run_batch_host(htext, offsets=hl, flags=N.RUN_BEGIN | N.RUN_END | N.RUN_LINES, want_states=True)
lines = text.split(b"\n")
c, o = csr(lines)
f, m, s = orc.run(c, o)
assert (np.unpackbits(bits.view(np.uint8), bitorder="little")[:len(lines)] == f).all() and (states == s).all()
assert int(f.sum()) > 100 and f[-1] == 1
print("ok host entry")
# odd shapes: empty strings, unaligned starts
strings = [b"", b"x", b"hello world", b"\xd0\xbf" * 7 + b"HeLLo  World", b"a" * 33, b""] * 20
bb = P.Batch.from_strings(strings)
r = P.Runner(sc).Begin().Run(bb).End()
from refpire import csr
c, o = csr(strings)
f, m, s = orc.run(c, o)
assert (r.Matches().astype(np.uint8) == f).all() and (r.States() == s).all()
print("ok ragged")
# tiny automaton (one private quad) over bytes >= 128, fixed length: the PRIV kernel's speculative steps
from conftest import GOLDEN
case = next(c for c in GOLDEN if c.name == "UTF8@181b")
sc = P.Scanner(case.image, 0)
orc = Oracle(case.image)
rng = np.random.default_rng(5)
fx = rng.choice(np.frombuffer("x\u0424y ab".encode() + bytes(range(120, 256)), np.uint8), size=(1024, 64)).reshape(-1)
fb = P.Batch(torch.from_numpy(fx).to(dev), fixed_len=64, n=1024)
check(sc, orc, fb, fx, None, 64, 1024, "tiny DFA, high bytes, PRIV")
# lines of text: split on the device, lines kernel (plain / pred) and the generic kernel on the same lines;
# the text starts and ends off a 16-byte boundary so that the clipped chunk loads are exercised
rng = np.random.default_rng(9)
words = [b"hello", b"world", b"GET /x", b"error", b"timeout", b"", b"fatal https://a", b"x" * 70, b"hello   wd"]
text_lines = [b" ".join(words[int(j)] for j in rng.integers(0, len(words), size=int(k))) for k in rng.integers(0, 9, size=3000)]
blob = b"\n".join(text_lines) + b"\n"
pad = torch.zeros(len(blob) + 64, dtype=torch.uint8, device=dev)
text_dev = pad[5:5 + len(blob)]
text_dev.copy_(torch.from_numpy(np.frombuffer(blob, np.uint8).copy()))
lb = P.Batch.from_text(text_dev)
assert lb.n == len(text_lines)
c, o = csr(text_lines)
for name in ("headline", "glue10"):
    image = W.load_image(name)
    orc = Oracle(image)
    f, m, s_ = orc.run(c, o)
    for max_hot in (255, 2):
        sc = P.Scanner(image, 0)
        sc.set_max_hot(max_hot)
        for variant in (N.VARIANT_PLAIN, N.VARIANT_PRED, N.VARIANT_LOOK):
            sc.set_variant(variant)
            r = P.Runner(sc).Begin().Run(lb).End()
            assert (r.Matches().astype(np.uint8) == f).all() and (r.AcceptMasks() == m).all() and (r.States() == s_).all(), (name, max_hot, variant)
print("ok lines", flush=True)
# prefix and suffix scans (all four kernels), ragged + fixed, tiny hot set
from refpire import oracle_prefix, oracle_suffix
for name in ("headline", "count_words5"):
    image = W.load_image(name)
    orc = Oracle(image)
    strings = [b"", b"x", b"hello  world", b"ab cd" * 40, b"a" * 33, b"zz hello\tworld", b"q" * 100] * 30
    c, o = csr(strings)
    bb = P.Batch.from_strings(strings)
    for max_hot in (255, 2):
        sc = P.Scanner(image, 0)
        sc.set_max_hot(max_hot)
        for shortest in (False, True):
            for m1 in (False, True):
                for m2 in (False, True):
                    got = (P.ShortestPrefix if shortest else P.LongestPrefix)(sc, bb, throughBeginMark=m1, throughEndMark=m2)
                    assert (got == oracle_prefix(orc, c, o, shortest=shortest, through_begin=m1, through_end=m2)).all()
                    got = (P.ShortestSuffix if shortest else P.LongestSuffix)(sc, bb, throughEndMark=m1, throughBeginMark=m2)
                    assert (got == oracle_suffix(orc, c, o, shortest=shortest, through_end=m1, through_begin=m2)).all()
    # fixed-length, 32-byte aligned batch: the uniform prefix kernel (no ring; chunks walked in final states only)
    rng_u = np.random.default_rng(7)
    nu, lu = 1024 + 5, 96
    hu = rng_u.choice(np.frombuffer(b"helo wrd\tab", np.uint8), size=(nu, lu))
    hu[::3, :12] = np.frombuffer(b"hello  world", np.uint8)
    hu = np.ascontiguousarray(hu).reshape(-1)
    bu = P.Batch(torch.from_numpy(hu).to(dev), fixed_len=lu, n=nu)
    scu = P.Scanner(image, 0)
    for shortest in (False, True):
        for m1 in (False, True):
            got = (P.ShortestPrefix if shortest else P.LongestPrefix)(scu, bu, throughBeginMark=m1, throughEndMark=True)
            assert (got == oracle_prefix(orc, hu, fixed_len=lu, n=nu, shortest=shortest, through_begin=m1, through_end=True)).all()
    print("ok prefix/suffix", name, flush=True)
# counting kernels (HalfFinalScanner): accept lists / packed / packed on every chunk, tiny hot sets, ragged + fixed
from refpire import oracle_count
for name in ("hf_glue10", "count_words5"):
    image = W.load_image(name)
    orc = Oracle(image)
    strings = [b"", b"x", b"GET /a error timeout", b"hello  world fatal https://x", b"ab cd" * 40, b"a" * 33, b"zz"] * 40
    c, o = csr(strings)
    want, wfin = oracle_count(orc, c, o)
    bb = P.Batch.from_strings(strings)
    for max_hot in (255, 2):
        sc = P.Scanner(image, 0)
        sc.set_max_hot(max_hot)
        for mode in (1, 2, 3):
            sc.set_count_mode(mode)
            res = P.HalfFinalCount(sc, bb)
            assert (res.counts == want).all() and (res.final == wfin.astype(bool)).all(), (name, max_hot, mode)
    spec = W.SynthSpec(1024 + 5, 256, plants=W.GLUE10_PLANTS)
    d = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
    spec.fill_device(d)
    host = spec.host_sample(0, 1024 + 5)
    want, wfin = oracle_count(orc, host, fixed_len=256, n=1024 + 5)
    sc = P.Scanner(image, 0)
    fbatch = P.Batch(d, fixed_len=256, n=1024 + 5)
    sc.Tune(fbatch, 512)
    res = P.HalfFinalCount(sc, fbatch)
    assert (res.counts == want).all() and (res.final == wfin.astype(bool)).all(), name
    print("ok counting", name, flush=True)
# round 2: register-streaming bodies of the prefix / counting kernels (fixed length, multiple of 32, partial last warp),
# accept sets, the streaming host entry point (1 MiB chunks, pageable input), the one-rank sharded call
image = W.load_image("headline")
orc = Oracle(image)
sc = P.Scanner(image, 0)
spec = W.SynthSpec(1024 + 7, 160, plants=W.HEADLINE_PLANTS)
d = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
spec.fill_device(d)
host = spec.host_sample(0, 1024 + 7)
fbatch = P.Batch(d, fixed_len=160, n=1024 + 7)
for shortest in (False, True):
    got = (P.ShortestPrefix if shortest else P.LongestPrefix)(sc, fbatch, throughBeginMark=True, throughEndMark=True)
    assert (got == oracle_prefix(orc, host, fixed_len=160, n=1024 + 7, shortest=shortest, through_begin=True, through_end=True)).all()
image = W.load_image("hf_glue10")
sc_hf = P.Scanner(image, 0)
want, wfin = oracle_count(Oracle(image), host, fixed_len=160, n=1024 + 7)
for mode in (1, 2, 3):
    sc_hf.set_count_mode(mode)
    res = P.HalfFinalCount(sc_hf, fbatch)
    assert (res.counts == want).all(), mode
print("ok uniform bodies", flush=True)
import ctypes as C
r = P.Runner(sc).Begin().Run(fbatch).End()
states = torch.from_numpy(r.States().astype(np.int32)).to(dev)
sets = torch.zeros(1024 + 7, dtype=torch.int32, device=dev)
N.check(N.lib.pire_gpu_accept_sets(sc._h, states.data_ptr(), 1024 + 7, sets.data_ptr(), None), "accept sets")
assert (sets.cpu().numpy().view(np.uint32) == r.AcceptMasks()).all()
os.environ["PIRE_B200_HOST_CHUNK_MB"] = "1"
big = W.SynthSpec(6000, 1024, plants=W.HEADLINE_PLANTS)
hbig = big.host_sample(0, 6000)
bits, masks, _ = sc.run_batch_host(hbig, fixed_len=1024, n=6000, want_masks=True)
f, m, _ = orc.run(hbig, fixed_len=1024, n=6000)
assert (np.unpackbits(bits.view(np.uint8), bitorder="little")[:6000] == f).all() and (masks == m).all()
from pire_b200.dist import Comm
comm = Comm(0, rank=0, world=1)
ball = torch.full((comm.words(1024 + 7),), -1, dtype=torch.int32, device=dev)
comm.run_sharded(sc, fbatch, 1024 + 7, N.RUN_BEGIN | N.RUN_END, ball)
torch.cuda.synchronize()
assert (np.unpackbits(ball.cpu().numpy().view(np.uint8), bitorder="little")[:1024 + 7] == r.Matches().astype(np.uint8)).all()
comm.close()
print("ok accept sets, host streaming, sharded(1)", flush=True)
# per-string starts (pire_gpu_run_batch_from), chained in place through the state buffer: a uniform batch (the two-string
# ring kernel and the one-string ring kernel, some starts outside the scanner) and an ordered CSR batch with strings long
# enough for the split kernel; the results against one run over the whole strings
from string_oracle import run_from
img = W.load_image("glue10")
orc = Oracle(img)
sc = P.Scanner(img, 0)
rng = np.random.default_rng(13)
n, half = 64 * 3 + 5, 128
whole = rng.choice(np.frombuffer(b"GET error timeout https:// ab(5)", np.uint8), size=(n, 2 * half))
for variant in (N.VARIANT_LOOK, N.VARIANT_LOOK_RING1):
    sc.set_variant(variant)
    st = torch.full((n,), sc.Initialize(), dtype=torch.int32, device=dev)
    st[7] = sc.Size()
    for k, flags in ((0, N.RUN_BEGIN), (1, N.RUN_END)):
        piece = torch.from_numpy(np.ascontiguousarray(whole[:, k * half:(k + 1) * half]).reshape(-1)).to(dev)
        sc.run_batch(P.Batch(piece, fixed_len=half, n=n), flags, None, None, st, start_idx=st)
    got = st.cpu().numpy().view(np.uint32)
    want = [run_from(orc, whole[i], sc.Size() if i == 7 else sc.Initialize(), True, True)[2] for i in range(n)]
    assert (got == np.array(want, np.uint32)).all(), variant
strings = [bytes(rng.choice(np.frombuffer(b"GET error timeout ab", np.uint8), size=int(k))) for k in [9000, 20000] + list(rng.integers(0, 600, size=100))]
bb = P.Batch.from_strings(strings).bin_by_length()
starts = rng.integers(0, sc.Size(), size=len(strings))
st = torch.from_numpy(starts.astype(np.int32)).to(dev)
sc.set_variant(N.VARIANT_PRED)
sc.run_batch(bb, N.RUN_BEGIN | N.RUN_END, None, None, st, start_idx=st)
want = [run_from(orc, np.frombuffer(s, np.uint8), int(x), True, True)[2] for s, x in zip(strings, starts)]
assert (st.cpu().numpy().view(np.uint32) == np.array(want, np.uint32)).all()
print("ok run_batch_from", flush=True)
# HalfFinalScanner counts of many streams (pire_gpu_count_batch_from): a ragged CSR batch cut into two rounds, chained in
# place through one state array and one counts array (some starts outside the scanner), in every count mode, against
# one count over the whole strings
from count_oracle import count_from
img = W.load_image("hf_glue10")
orc = Oracle(img)
sc = P.Scanner(img, 0)
strings = [bytes(rng.choice(np.frombuffer(b"GET error timeout https:// ab", np.uint8), size=int(k))) for k in rng.integers(0, 400, size=70)]
cuts = [int(rng.integers(0, len(s) + 1)) for s in strings]
starts = rng.integers(0, sc.Size(), size=len(strings))
starts[5] = sc.Size()
for mode in (1, 2, 3):
    sc.set_count_mode(mode)
    st = torch.from_numpy(starts.astype(np.int32)).to(dev)
    c = P.BatchCounter(sc, len(strings), st).Begin()
    for k in (0, 1):
        c.Run(P.Batch.from_strings([s[:x] if k == 0 else s[x:] for s, x in zip(strings, cuts)]))
    c.End()
    got = c.Counts().cpu().numpy()
    for i, s in enumerate(strings):
        assert got[i].tolist() == count_from(orc, np.frombuffer(s, np.uint8), int(starts[i]))[0], (mode, i)
print("ok count_batch_from", flush=True)
# where the matches end in one string (pire_gpu_match_ends_string): three chained pieces, one cut inside a 32-byte block,
# into a buffer too small for the answer, against count_string on the same bytes and a call with room for all of it
sc.set_count_mode(0)
text = torch.from_numpy(rng.choice(np.frombuffer(b"GET error timeout https:// ab", np.uint8), size=300_007)).to(dev)
cnt = P.StringCounter(sc).Begin().Run(text).End()
total = sum(cnt.Result(r) for r in range(max(1, sc.RegexpsCount())))
full = P.StringMatchEnds(sc, total).Begin().Run(text).End()
part = P.StringMatchEnds(sc, total // 2).Begin().Run(text[:5]).Run(text[5:100_003]).Run(text[100_003:]).End()
assert full.Found() == part.Found() == total
assert (part.Ends() == full.Ends()[: total // 2]).all() and (part.Ids() == full.Ids()[: total // 2]).all()
assert np.bincount(full.Ids(), minlength=max(1, sc.RegexpsCount())).tolist() == [cnt.Result(r) for r in range(max(1, sc.RegexpsCount()))]
print("ok match_ends_string", flush=True)
# where the matches end in many streams (pire_gpu_match_ends_batch_from): the ragged batch above in its two rounds, into
# a buffer too small for the answer, against BatchCounter on the same rounds and a call with room for all of it
regs = max(1, sc.RegexpsCount())
halves = [P.Batch.from_strings([s[:x] if k == 0 else s[x:] for s, x in zip(strings, cuts)]) for k in (0, 1)]
c = P.BatchCounter(sc, len(strings)).Begin().Run(halves[0]).Run(halves[1]).End()
total = int(c.Counts().sum().item())
full = P.BatchMatchEnds(sc, len(strings), total).Begin().Run(halves[0]).Run(halves[1]).End()
part = P.BatchMatchEnds(sc, len(strings), total // 2).Begin().Run(halves[0]).Run(halves[1]).End()
assert full.Found() == part.Found() == total
assert (part.Ends() == full.Ends()[: total // 2]).all() and (part.Strings() == full.Strings()[: total // 2]).all()
key = full.Strings().astype(np.int64) * regs + full.Ids()
assert (np.bincount(key, minlength=len(strings) * regs).reshape(-1, regs) == c.Counts().cpu().numpy()).all()
print("ok match_ends_batch_from", flush=True)
# where the matches end in every line of a text (pire_gpu_match_ends_lines): the ragged strings above joined into a text,
# into a buffer too small for the answer and one with room for all of it, against count_batch with LINES
text = torch.frombuffer(bytearray(b"\n".join(s.replace(b"\n", b" ") for s in strings)), dtype=torch.uint8).to("cuda:0")
lb = P.Batch.from_text(text)
lc = P.HalfFinalCount(sc, lb)
ltotal = int(lc.counts.sum())
lfull = P.LineMatchEnds(sc, ltotal).Begin().Run(lb).End()
lpart = P.LineMatchEnds(sc, ltotal // 2).Begin().Run(lb).End()
assert lfull.Found() == lpart.Found() == ltotal and (lpart.Ends() == lfull.Ends()[: ltotal // 2]).all()
key = lfull.Lines().astype(np.int64) * regs + lfull.Ids()
assert (np.bincount(key, minlength=lb.n * regs).reshape(-1, regs) == lc.counts).all()
print("ok match_ends_lines", flush=True)
# a text streamed from host memory (pire_gpu_line_stream): pageable and pinned pieces, a line longer than the slot
long_text = b"\n".join(s.replace(b"\n", b" ") for s in strings) + b"\n" + b"x" * 5000 + b"\nend"
pinned = torch.empty(len(long_text), dtype=torch.uint8, pin_memory=True)
pinned.copy_(torch.frombuffer(bytearray(long_text), dtype=torch.uint8))
whole = P.Batch.from_text(torch.frombuffer(bytearray(long_text), dtype=torch.uint8).to("cuda:0"))
want_bits = P.Runner(sc).Begin().Run(whole).End().Matches()
ls = P.LineStream(0, 1024)
got_bits = []
half = len(long_text) // 2
for k, piece in enumerate((np.frombuffer(long_text[:half], np.uint8), pinned[half:])):
    for f in ls.feed(piece, last=k == 1):
        got_bits += P.Runner(sc).Begin().Run(f).End().Matches().tolist()
assert got_bits == want_bits.tolist()
print("ok line_stream", flush=True)
# two scanners over the lines of that text in one walk (pire_gpu_run_pair_lines), against the two single calls
other = P.Scanner(W.load_image("headline"), 0)
both = P.Runner(P.ScannerPair(sc, other)).Begin().RunLines(whole).End()
for half_, one in ((both.First(), sc), (both.Second(), other)):
    ref = P.Runner(one).Begin().Run(whole).End()
    assert (half_.Matches() == ref.Matches()).all() and (half_.AcceptMasks() == ref.AcceptMasks()).all() \
        and (half_.States() == ref.States()).all()
print("ok pair_lines", flush=True)
# a SlowScanner on both paths (pire_gpu_slow_run_batch): the reference's recorded answers, a CSR batch and lines of a text
from slow_fixtures import SLOW
for name in ("heavy/a30", "heavy/error200"):
    e = next(x for x in SLOW if x.name == name)
    ssc = P.SlowScanner(e.image, 0)
    r = P.Runner(ssc).Begin().Run(P.Batch.from_strings(e.strings)).End()
    final, sets = e.runs[(True, True, False)]
    assert (r.Matches() == final).all() and (r.Sets() == sets).all(), name
    text = b"\n".join(e.strings) + b"\n"          # the strings hold newlines of their own: compare line by line
    lines = P.Batch.from_text(torch.tensor(list(text), dtype=torch.uint8, device=dev))
    want = P.Runner(ssc).Begin().Run(P.Batch.from_strings(text.split(b"\n")[:-1])).End()
    got = P.Runner(ssc).Begin().Run(lines).End()
    assert (got.Matches() == want.Matches()).all() and (got.Sets() == want.Sets()).all(), name + " lines"
print("ok slow_run_batch", flush=True)
torch.cuda.synchronize()
print("sanitize_run done, launches:", N.lib.pire_gpu_launch_count())
