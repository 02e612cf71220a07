"""The two-string look-ahead kernel fed from a cp.async ring (ScanUniformLookRingKernel) against the in-repo oracle.

Every case checks match bits, accept masks and StateIndex against the oracle, with sentinels past n.  One launch is
profiled first, to assert that the ring kernel is the one that runs."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from test_edge_images import ALPHABETS, EDGE, static_hot_order  # noqa: E402
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, MARKS, RUN_BEGIN, RUN_END, BeginMark, Checker, HostBatch, _filled,  # noqa: E402
                            _host, _stream, expect_equal, expect_untouched, fixed_batch, glue10_image, kernels_launched,
                            random_rows, random_strings, unpack_bits)

pytestmark = pytest.mark.gpu

RING_WARPS = 24                   # warps per CTA of ScanUniformLookRingKernel (kRingBlock / 32), one CTA per SM
HEADLINE_ALPHABET = b"abcdefghijklmnopqrstuvwxyz ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789.,:;-_/()[]{}@#"


def run_look(chk, hb, begin, end, label):
    """pire_gpu_run_batch with the look-ahead variant on a uniform batch; every output against the oracle."""
    from pire_b200 import _native as N
    assert hb.offsets is None and hb.fixed_len % 32 == 0 and hb.corpus_ptr() % 32 == 0, label      # a uniform batch
    chk.sc.set_variant(N.VARIANT_LOOK)
    n = hb.n
    bits, masks, states = _filled((n + 31) // 32 + 1), _filled(n + EXTRA), _filled(n + EXTRA)
    flags = (RUN_BEGIN if begin else 0) | (RUN_END if end else 0)
    N.check(N.lib.pire_gpu_run_batch(chk.sc._h, hb.corpus_ptr(), None, hb.fixed_len, n, flags, bits.data_ptr(), masks.data_ptr(),
                                     states.data_ptr(), _stream()), "run (%s)" % label)
    f, m, s = (x[:n] for x in chk.want(hb, "run", begin, end))
    hb_bits, hm, hs = _host(bits), _host(masks), _host(states)
    expect_untouched(label, "accept masks", hm, n)
    expect_untouched(label, "state indices", hs, n)
    expect_equal(label, "StateIndex", hs[:n], s)
    expect_equal(label, "accept masks", hm[:n], m)
    expect_equal(label, "match bits", unpack_bits(label, hb_bits, n), f)


def batch_at_allocation_end(rows):
    """A uniform batch whose last string ends on the last byte of its device allocation (a 16 MiB buffer, which the
    caching allocator takes from cudaMalloc at exactly that size)."""
    size = 16 << 20
    n, length = rows.shape
    base = size - n * length
    assert base >= 0 and base % 32 == 0
    buf = np.zeros(size, np.uint8)
    buf[base:] = np.ascontiguousarray(rows).reshape(-1)
    hb = HostBatch(buf, base=base, fixed_len=length, n=n)
    assert hb.corpus_ptr() + n * length == hb.device()[0].data_ptr() + hb.device()[0].numel()
    return hb


def noexit_byte(host, begin):
    """A byte that sends the start state to a state no byte leaves (an anchored pattern that failed), and that state."""
    start = host.Next(host.Initialize(), BeginMark) if begin else host.Initialize()
    for c in b"xz ":
        d = host.Next(start, c)
        if all(host.Next(d, b) == d for b in range(256)):
            return c, d
    raise AssertionError("no byte reaches a NoExit state")


def test_ring_kernel_matches_oracle(cuda_device):
    import torch
    import pire_b200 as P
    rng = np.random.default_rng(2024)
    # first of all, with the cache emptied, so that the caching allocator gives it a cudaMalloc of its own
    torch.cuda.empty_cache()
    end_rows = random_rows(rng, 32 * 501 + 7, 1024, GLUE10_ALPHABET, [b"GET ", b"error", b"timeout"])
    at_end = batch_at_allocation_end(end_rows)
    at_end.device()

    glue = Checker(glue10_image(), "glue10")
    launched = kernels_launched(lambda: run_look(glue, at_end, True, True, "probe"))
    assert "ScanUniformLookRingKernel" in launched, launched[:2000]

    from pire_b200 import workloads as W
    images = [("glue10", glue10_image(), GLUE10_ALPHABET, [b"GET ", b"error", b"timeout", b"(555) 123-4567"]),
              ("headline", W.load_image("headline"), HEADLINE_ALPHABET, [b"error", b"GET ", b"timeout"])]
    shapes = [(length, n) for length in (32, 64, 96, 1024) for n in (1, 31, 33, 63, 64, 65, 32 * 5 + 3)] + [(65536, 65)]
    batches = [(length, n, fixed_batch(random_rows(rng, n, length, alphabet, literals)))
               for length, n in shapes for alphabet, literals in [(GLUE10_ALPHABET, [b"GET ", b"error", b"timeout"])]]
    tune_sample = random_strings(rng, GLUE10_ALPHABET, [1024] * 64, [b"GET ", b"error"])
    for name, image, alphabet, literals in images:
        rows = random_rows(rng, 64 * 7 + 5, 1024, alphabet, literals)
        own = fixed_batch(rows)
        for tuned in (False, True):
            for max_hot in (255, 6, 2, 1):
                chk = Checker(image, name)
                chk.sc.set_max_hot(max_hot)
                if tuned:
                    chk.sc.Tune(P.Batch.from_strings(tune_sample), len(tune_sample), begin=True, end=True)
                    assert chk.sc.info().tuned == 1
                tag = "%s %s max_hot=%d" % (name, "tuned" if tuned else "static", max_hot)
                for begin, end in MARKS:
                    run_look(chk, own, begin, end, "%s own begin=%d end=%d" % (tag, begin, end))
                if max_hot in (255, 2) and name == "glue10":
                    for length, n, hb in batches:
                        for begin, end in MARKS:
                            run_look(chk, hb, begin, end, "%s len=%d n=%d begin=%d end=%d" % (tag, length, n, begin, end))
                    run_look(chk, at_end, True, True, tag + " ends at the allocation's end")

    # wide tables (32-bit cells): lanes leave the hot rows at once and are replayed block by block
    e = EDGE["wide"]
    rows = rng.choice(np.frombuffer(b"ab", np.uint8), size=(64 * 9 + 33, 256))
    rows[::17, 100] = ord("c")
    wide = fixed_batch(rows)
    for max_hot in (255, 2):
        chk = Checker(e["image"], "wide")
        chk.sc.set_max_hot(max_hot)
        assert chk.sc.info().table_bytes == chk.sc.info().states * chk.sc.info().letters * 4
        for begin, end in MARKS:
            run_look(chk, wide, begin, end, "wide max_hot=%d begin=%d end=%d" % (max_hot, begin, end))

    # NoExit early exit, then a further pair of units on the same warp: the strings of every warp's first pair fall into
    # a state no byte leaves within their first block (the warp leaves after 64 of 128 bytes with two blocks still in
    # flight), the later pairs (^(ab|cd)+e$ kept alive by tokens ab / cd, half of them ending in e) are walked to their end
    # from the same ring slots
    anchored = EDGE["anchored"]["image"]
    host = P.Scanner(anchored, -1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    first = 64 * RING_WARPS * sms
    for begin, end in ((True, True), (False, False)):
        c, dead = noexit_byte(host, begin)
        assert dead in set(static_hot_order(host, 255))                  # a hot row: the kernel's NoExit ballot sees it
        rows = random_rows(rng, 2 * first + 64 * 3 + 17, 128, ALPHABETS["anchored"])
        rows[:first, 0] = c
        tokens = np.frombuffer(b"abcd", np.uint8).reshape(2, 2)
        later = rows.shape[0] - first
        rows[first:, :] = tokens[rng.integers(0, 2, size=(later, 64))].reshape(later, 128)
        rows[first::2, 127] = ord("e")
        chk = Checker(anchored, "anchored")
        run_look(chk, fixed_batch(rows), begin, end, "NoExit exit, then another pair begin=%d end=%d" % (begin, end))
        _, _, states = chk.want(fixed_batch(rows[:64]), "run", begin, False)
        assert (states == dead).all()
