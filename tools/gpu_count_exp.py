#!/usr/bin/env python
"""HalfFinalScanner counting on the device (pire_gpu_count_batch): throughput on the BASELINE configs[2]
corpus (1 KiB printable-ASCII strings, 1/8 planted) for
  hf_glue10     the ten patterns as glued HalfFinalScanners (211 states; finals are rare), and
  count_words5  the five HalfFinalFsm counters of [a-z]+ (3 states; almost every byte is final),
with a sample of every run checked against the real reference (oracle/_ref) or the oracle port.
Usage: python tools/gpu_count_exp.py [strings]   (run on a GPU host)
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import pire_b200 as P  # noqa: E402
from pire_b200 import _native as N  # noqa: E402
from pire_b200 import workloads as W  # noqa: E402
import refpire  # noqa: E402


def main():
    n = (int(sys.argv[1]) if len(sys.argv) > 1 else 4 * 1024 * 1024) // 32 * 32
    dev = torch.device("cuda:0")
    spec = W.SynthSpec(n, 1024, plants=W.GLUE10_PLANTS)
    corpus = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
    spec.fill_device(corpus)
    batch = P.Batch(corpus, fixed_len=1024, n=n)
    payload = n * 1024
    sample = min(n, 8192)
    host = corpus[: sample * 1024].cpu().numpy()
    ref = refpire.Ref() if refpire.have_ref() else None
    out = {"strings": n, "bytes": payload, "checker": "reference (oracle/_ref)" if ref else "oracle port"}

    # the ordinary glued Scanner on the same bytes: which regexps does it accept per string?
    sc10 = P.Scanner(W.load_image("glue10"), 0)
    sc10.Tune(batch, 16384)
    masks10 = P.Runner(sc10).Begin().Run(batch).End().AcceptMasks()

    for name in ("hf_glue10", "count_words5"):
        image = W.load_image(name)
        sc = P.Scanner(image, 0)
        regs = sc.RegexpsCount()
        counts = torch.empty((n, regs), dtype=torch.int32, device=dev)
        bits = torch.zeros(n // 32, dtype=torch.int32, device=dev)
        flags = N.RUN_BEGIN | N.RUN_END
        stream = torch.cuda.current_stream(dev).cuda_stream

        def run():
            N.check(N.lib.pire_gpu_count_batch(sc._h, corpus.data_ptr(), None, 1024, n, flags, counts.data_ptr(), bits.data_ptr(),
                                               stream), "pire_gpu_count_batch")
        res = {}
        for label, mode, tuned in (("lists", 1, False), ("packed", 2, False), ("every_chunk", 3, False), ("auto_tuned", 0, True)):
            sc.set_count_mode(mode)
            if tuned:
                sc.Tune(batch, 16384)
            for _ in range(2):
                run()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(5):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            res[label] = {"ms": ms, "GBps": payload / 1e9 / (ms / 1e3)}
            got = counts[:sample].cpu().numpy().view(np.uint32)
            if label == "lists":
                if ref:
                    want, wfin = ref.load_half_final(image).count(host, fixed_len=1024, n=sample, threads=8)
                else:
                    want, wfin = refpire.oracle_count(refpire.Oracle(image), host, fixed_len=1024, n=sample)
            assert (got == want).all(), (name, label, np.argwhere(got != want)[:5])
        words = bits[: sample // 32].cpu().numpy().view(np.uint32)
        fin = (words[np.arange(sample) // 32] >> (np.arange(sample) % 32).astype(np.uint32)) & 1
        assert (fin == wfin).all()
        res["sample_checked"] = sample
        res["regexps"] = regs
        res["states"] = sc.Size()
        res["mean_count_per_string"] = [float(x) for x in counts.float().mean(dim=0).cpu().numpy()]
        if name == "hf_glue10":
            # AcceptedRegexps of the HalfFinalScanner (regexps with a non-zero counter) vs the glued Scanner's accept mask
            nz = (counts != 0).to(torch.int64)
            m = (nz << torch.arange(regs, device=dev)).sum(dim=1).cpu().numpy().astype(np.uint32)
            res["agrees_with_glued_scanner_masks"] = bool((m == masks10).all())
            res["strings_with_any_match"] = int((m != 0).sum())
        out[name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
