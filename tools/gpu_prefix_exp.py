#!/usr/bin/env python
"""Throughput of pire_gpu_prefix_batch (LongestPrefix / ShortestPrefix) on the configs[2] corpus.
Usage: python tools/gpu_prefix_exp.py [strings]   (run on a GPU host)"""
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
    n = (int(sys.argv[1]) if len(sys.argv) > 1 else 2 * 1024 * 1024) // 32 * 32
    dev = torch.device("cuda:0")
    spec = W.SynthSpec(n, 1024, plants=W.GLUE10_PLANTS)
    corpus = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
    spec.fill_device(corpus)
    batch = P.Batch(corpus, fixed_len=1024, n=n)
    payload = n * 1024
    sample = min(n, 4096)
    host = corpus[: sample * 1024].cpu().numpy()
    out = {"strings": n, "bytes": payload}
    lens = torch.empty(n, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for name in ("headline", "glue10", "count_words5"):
        image = W.load_image(name)
        sc = P.Scanner(image, 0)
        sc.Tune(batch, 16384)
        orc = refpire.Oracle(image)
        res = {}
        for shortest in (0, 1):
            def run():
                N.check(N.lib.pire_gpu_prefix_batch(sc._h, corpus.data_ptr(), None, 1024, n, N.RUN_BEGIN, shortest, lens.data_ptr(), stream),
                        "pire_gpu_prefix_batch")
            run()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(3):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 3
            got = lens[:sample].cpu().numpy().view(np.uint32).astype(np.int64)
            got[got == 0xFFFFFFFF] = -1
            want = refpire.oracle_prefix(orc, host, fixed_len=1024, n=sample, shortest=bool(shortest), through_begin=True)
            assert (got == want).all(), (name, shortest)
            res["shortest" if shortest else "longest"] = {"ms": ms, "GBps": payload / 1e9 / (ms / 1e3),
                                                          "mean_len": float(np.where(got < 0, 0, got).mean()),
                                                          "found": int((got >= 0).sum())}
        out[name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
