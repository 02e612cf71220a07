#!/usr/bin/env python
"""Two scanners over one batch (pire_gpu_run_pair_batch) measured against the two single pire_gpu_run_batch calls.

    python tools/pair_bench.py [--gib 10] [--reps 10] [--mixed 200000] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); `gib` GiB of 1 KiB synthetic strings
generated on the device with the glue10 and headline plants; then for each pair (glue10 + headline, glue10 + hf_glue10,
headline + headline_iu), both handles tuned and auto-selected on the batch as bench.py does:
  1. the fused call and the two single calls back to back, alternated `reps` times after a warm-up of each, timed with
     CUDA events: medians, minimum and maximum, the ratio of the medians (single / fused) and the rate over the corpus;
  2. the six outputs of the fused call compared word for word with the single calls' on the whole timed corpus.
Then one CSR pair (headline_iu + glue10 on `mixed` strings of the utf8mixed corpus, 16 B .. 64 KiB), which takes the
unfused path, timed the same way.  Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/pair_bench.json."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

STRING_LEN = 1024
PAIRS = [("glue10", "headline"), ("glue10", "hf_glue10"), ("headline", "headline_iu")]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--mixed", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W

    dev = torch.device("cuda:0")
    flags = N.RUN_BEGIN | N.RUN_END

    def outputs(n):
        return (torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev),
                torch.zeros(n, dtype=torch.int32, device=dev))

    def event_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def compare(fn_fused, fn_single, batch, nbytes):
        """Alternated timings and the word-for-word parity of the six outputs."""
        fn_fused()
        fn_single()
        torch.cuda.synchronize()
        fused, single = [], []
        for _ in range(args.reps):
            fused.append(event_ms(fn_fused))
            single.append(event_ms(fn_single))
        stat = lambda v: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)),
                          "median_gbps": nbytes / float(np.median(v)) / 1e6}
        return {"fused": stat(fused), "single_pair": stat(single), "single_over_fused": float(np.median(single) / np.median(fused))}

    def pair_case(sc1, sc2, batch, nbytes):
        n = batch.n
        got, want = outputs(n) + outputs(n), outputs(n) + outputs(n)
        pair = P.ScannerPair(sc1, sc2)
        fused = lambda: pair.run_pair_batch(batch, flags, got[:3], got[3:])

        def single():
            sc1.run_batch(batch, flags, *want[:3])
            sc2.run_batch(batch, flags, *want[3:])
        res = compare(fused, single, batch, nbytes)
        fused()
        single()
        torch.cuda.synchronize()
        res["mismatched_words"] = sum(int((a != b).sum().item()) for a, b in zip(got, want))
        res["matches"] = [int(np.unpackbits(t.cpu().numpy().view(np.uint8)).sum()) for t in (got[0], got[3])]
        return res

    n = int(args.gib * 2 ** 30) // STRING_LEN // 32 * 32
    spec = W.SynthSpec(n, STRING_LEN, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS)
    corpus = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
    spec.fill_device(corpus)
    batch = P.Batch(corpus, fixed_len=STRING_LEN, n=n)
    handles = {}
    for name in sorted({x for p in PAIRS for x in p}):
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(batch, min(n, 16384))
        sc.AutoSelect(batch)
        handles[name] = sc
    res = {"card": card(), "n_strings": n, "string_len": STRING_LEN, "gib": n * STRING_LEN / 2 ** 30, "reps": args.reps,
           "variants": {k: N.VARIANT_NAMES.get(v.info().variant, str(v.info().variant)) for k, v in handles.items()},
           "hot_rows": {k: int(v.info().hot_rows) for k, v in handles.items()}, "pairs": {}}
    for a, b in PAIRS:
        res["pairs"]["%s+%s" % (a, b)] = pair_case(handles[a], handles[b], batch, n * STRING_LEN)
    del corpus, batch
    torch.cuda.empty_cache()

    # the unfused path: a CSR batch of mixed lengths
    mc, mo = W.MixedSpec(args.mixed).device_batch(dev)
    mixed = P.Batch(mc, offsets=mo)
    iu, g = P.Scanner(W.load_image("headline_iu"), 0), P.Scanner(W.load_image("glue10"), 0)
    for sc in (iu, g):
        sc.Tune(mixed, min(args.mixed, 16384))
        sc.AutoSelect(mixed)
    res["csr"] = {"pair": "headline_iu+glue10", "n_strings": args.mixed, "bytes": int(mo[-1].item())}
    res["csr"].update(pair_case(iu, g, mixed, int(mo[-1].item())))
    res["card_after"] = card()
    bad = sum(p["mismatched_words"] for p in res["pairs"].values()) + res["csr"]["mismatched_words"]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pair_bench.json"), "w") as f:
            f.write(line + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
