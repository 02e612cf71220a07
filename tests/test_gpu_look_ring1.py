"""The one-string look-ahead kernel fed from a cp.async ring (ScanUniformLookRing1Kernel, variant LOOK_RING1) against the
in-repo oracle and against the two-string ring kernel of the LOOK variant (ScanUniformLookRingKernel).

Each variant runs in a child process of its own, as in test_gpu_look_ring.py: the child checks match bits, accept masks
and StateIndex of every case against the oracle (with sentinels past n), saves the outputs, and the parent then asserts
that both variants wrote the same words.  Each child first profiles one launch and asserts that the kernel it means to
test is the one that ran.  The variant's other paths (CSR batches, AutoSelect) are checked in-process.

Run as a script (``python tests/test_gpu_look_ring1.py <ring1|look> <out.npz>``) the module is that child."""
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
from test_gpu_edges import (EXTRA, GLUE10_ALPHABET, MARKS, RUN_BEGIN, RUN_END, Checker, _filled, _host, _stream, csr_batch,  # noqa: E402
                            expect_equal, expect_untouched, fixed_batch, glue10_image, random_rows, random_strings, unpack_bits)
from test_gpu_look_ring import HEADLINE_ALPHABET, batch_at_allocation_end, kernels_launched, noexit_byte  # noqa: E402

pytestmark = pytest.mark.gpu

RING1_WARPS = 32                  # warps per CTA of ScanUniformLookRing1Kernel (kRing1Block / 32), one CTA per SM


def run_variant(chk, hb, variant, begin, end, label, out):
    """pire_gpu_run_batch with one variant on a uniform batch; every output against the oracle, kept in ``out`` under
    ``label`` for the comparison between the two variants."""
    from pire_b200 import _native as N
    assert hb.offsets is None and hb.fixed_len % 32 == 0 and hb.corpus_ptr() % 32 == 0, label      # a uniform batch
    chk.sc.set_variant(variant)
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
    assert label not in out, label
    out[label + " bits"], out[label + " masks"], out[label + " states"] = hb_bits, hm, hs


def child(key, path):
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    variant = {"ring1": N.VARIANT_LOOK_RING1, "look": N.VARIANT_LOOK}[key]
    rng = np.random.default_rng(2025)
    out = {}
    # first of all, so that the caching allocator gives it a cudaMalloc of its own
    end_rows = random_rows(rng, 32 * 501 + 7, 1024, GLUE10_ALPHABET, [b"GET ", b"error", b"timeout"])
    at_end = batch_at_allocation_end(end_rows)
    at_end.device()

    glue = Checker(glue10_image(), "glue10")
    launched = kernels_launched(lambda: run_variant(glue, at_end, variant, True, True, "probe", {}))
    want_kernel = "ScanUniformLookRing1Kernel" if key == "ring1" else "ScanUniformLookRingKernel"
    assert want_kernel in launched and ("ScanUniformLookRing1Kernel" in launched) == (key == "ring1"), launched[:2000]

    from pire_b200 import workloads as W
    images = [("glue10", glue10_image(), GLUE10_ALPHABET, [b"GET ", b"error", b"timeout", b"(555) 123-4567"]),
              ("headline", W.load_image("headline"), HEADLINE_ALPHABET, [b"error", b"GET ", b"timeout"])]
    shapes = [(length, n) for length in (32, 64, 96, 1024) for n in (1, 31, 33, 63, 64, 65, 32 * 5 + 3)] + [(65536, 65)]
    batches = [(length, n, fixed_batch(random_rows(rng, n, length, GLUE10_ALPHABET, [b"GET ", b"error", b"timeout"])))
               for length, n in shapes]
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
                    run_variant(chk, own, variant, begin, end, "%s own begin=%d end=%d" % (tag, begin, end), out)
                if max_hot in (255, 2) and name == "glue10":
                    for length, n, hb in batches:
                        for begin, end in MARKS:
                            run_variant(chk, hb, variant, begin, end, "%s len=%d n=%d begin=%d end=%d" % (tag, length, n, begin, end), out)
                    run_variant(chk, at_end, variant, True, True, tag + " ends at the allocation's end", out)

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
            run_variant(chk, wide, variant, begin, end, "wide max_hot=%d begin=%d end=%d" % (max_hot, begin, end), out)

    # NoExit early exit, then further units on the same warp: the strings of every warp's first unit of the one-string
    # kernel fall into a state no byte leaves within their first block (the warp leaves after 64 of 128 bytes with two
    # blocks still in flight), the later units (^(ab|cd)+e$ kept alive by tokens ab / cd, half of them ending in e) are
    # walked to their end from the same ring slots
    anchored = EDGE["anchored"]["image"]
    host = P.Scanner(anchored, -1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    first = 32 * RING1_WARPS * sms
    for begin, end in ((True, True), (False, False)):
        c, dead = noexit_byte(host, begin)
        assert dead in set(static_hot_order(host, 255))                  # a hot row: the kernel's NoExit ballot sees it
        rows = random_rows(rng, 2 * first + 32 * 3 + 17, 128, ALPHABETS["anchored"])
        rows[:first, 0] = c
        tokens = np.frombuffer(b"abcd", np.uint8).reshape(2, 2)
        later = rows.shape[0] - first
        rows[first:, :] = tokens[rng.integers(0, 2, size=(later, 64))].reshape(later, 128)
        rows[first::2, 127] = ord("e")
        chk = Checker(anchored, "anchored")
        run_variant(chk, fixed_batch(rows), variant, begin, end, "NoExit exit, then further units begin=%d end=%d" % (begin, end), out)
        _, _, states = chk.want(fixed_batch(rows[:32]), "run", begin, False)
        assert (states == dead).all()

    np.savez_compressed(path, **out)
    print("LOOK-RING1 %s ok %d" % (key, len(out)))
    return 0


def test_ring1_kernel_matches_oracle_and_ring_kernel(cuda_device, tmp_path):
    import subprocess
    outs = {}
    for key in ("ring1", "look"):
        path = str(tmp_path / ("%s.npz" % key))
        env = {k: v for k, v in os.environ.items() if not k.startswith("PIRE_B200_")}
        proc = subprocess.run([sys.executable, os.path.abspath(__file__), key, path], env=env, cwd=ROOT, capture_output=True,
                              text=True, timeout=900)
        assert proc.returncode == 0, "%s failed (%d):\n%s\n%s" % (key, proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
        assert "LOOK-RING1 %s ok" % key in proc.stdout, proc.stdout[-2000:]
        outs[key] = np.load(path)
    ring1, look = outs["ring1"], outs["look"]
    assert sorted(ring1.files) == sorted(look.files) and len(ring1.files) > 300
    for k in ring1.files:
        expect_equal(k, "output words", ring1[k], look[k])


def test_ring1_variant_on_csr_batches(cuda_device):
    """On CSR batches the variant runs the CSR look-ahead kernel: oracle-exact, in order and length-ordered."""
    from pire_b200 import _native as N
    rng = np.random.default_rng(7)
    lengths = [0, 1, 31, 32, 33, 1024, 4099] + [int(x) for x in rng.integers(0, 3000, size=300)]
    hb = csr_batch(random_strings(rng, GLUE10_ALPHABET, lengths, [b"GET ", b"error", b"timeout", b"(555) 123-4567"]))
    chk = Checker(glue10_image(), "glue10")
    chk.sc.set_variant(N.VARIANT_LOOK_RING1)
    assert chk.sc.info().variant == N.VARIANT_LOOK_RING1
    for begin, end in MARKS:
        label = "CSR variant=%d begin=%d end=%d" % (N.VARIANT_LOOK_RING1, begin, end)
        chk.run(hb, begin, end, label)
        chk.run(hb, begin, end, label + " ordered", ordered=True)


def test_autoselect_times_ring1_on_uniform_batches_only(cuda_device):
    """AutoSelect times the variant on a uniform batch and not on a CSR batch, and info() reports the fastest variant
    timed (7 when the one-string ring kernel wins, as it does on the glued benchmark's batch on an H100)."""
    import pire_b200 as P
    import torch
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    ids = {name: v for v, name in N.VARIANT_NAMES.items()}
    spec = W.SynthSpec(1 << 19, 1024, plants=W.GLUE10_PLANTS)              # 512 MiB of 1 KiB strings
    dev = torch.empty(spec.total_bytes(), dtype=torch.uint8, device="cuda:0")
    spec.fill_device(dev)
    batch = P.Batch(dev, fixed_len=1024, n=spec.n_strings)
    chk = Checker(glue10_image(), "glue10")
    chk.sc.Tune(batch, 1 << 16)
    ms = chk.sc.AutoSelect(batch)
    assert ms.get("look_ring1", 0) > 0, ms
    best = min(ms, key=ms.get)
    assert chk.sc.info().variant == ids[best], (ms, chk.sc.info().variant)
    if best == "look_ring1":
        assert chk.sc.info().variant == 7

    # AUTO now runs the choice on uniform batches: oracle-exact on a sample of the same corpus
    n = 32 * 97 + 5
    rows = spec.host_sample(0, n).reshape(n, 1024)
    hb = fixed_batch(rows)
    chk.sc.set_variant(N.VARIANT_AUTO)
    for begin, end in MARKS:
        chk.run(hb, begin, end, "AUTO (%s) begin=%d end=%d" % (best, begin, end))

    rng = np.random.default_rng(11)
    strings = random_strings(rng, GLUE10_ALPHABET, [int(x) for x in rng.integers(1, 4000, size=2048)], [b"GET ", b"error"])
    ms_csr = chk.sc.AutoSelect(P.Batch.from_strings(strings))
    assert ms_csr and "look_ring1" not in ms_csr and "look1" not in ms_csr, ms_csr
    assert chk.sc.info().variant == ids[best]                               # info() names the choice for uniform batches


if __name__ == "__main__":
    sys.exit(child(sys.argv[1], sys.argv[2]))
