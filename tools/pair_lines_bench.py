#!/usr/bin/env python
"""Two scanners over the lines of a text (pire_gpu_run_pair_lines) measured against the two single pire_gpu_run_lines
calls.

    python tools/pair_lines_bench.py [--gib 4] [--reps 10] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); `gib` GiB of 80-120-byte planted
lines (tools/match_ends_lines_bench.py's make_text), split once; then for each pair (glue10 + headline, glue10 +
hf_glue10 -- 255 + 211 hot rows, the largest shared-memory footprint -- and headline + headline_iu), every handle tuned
on a sample of 65 536 lines of the batch:
  1. the fused call and the two single calls back to back, alternated `reps` times after a warm-up of each, timed with
     CUDA events: medians, minimum and maximum, the ratio of the medians (single / fused) and the rate over the text;
  2. the six outputs of the fused call compared word for word with the single calls' over the whole text.
Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/pair_lines_bench.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from match_ends_lines_bench import make_text  # noqa: E402
from pair_bench import card  # noqa: E402

PAIRS = [("glue10", "headline"), ("glue10", "hf_glue10"), ("headline", "headline_iu")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    if not torch.cuda.is_available():
        sys.exit("pair_lines_bench needs a CUDA device")

    dev = torch.device("cuda:0")
    flags = N.RUN_BEGIN | N.RUN_END
    text = make_text(torch, W, args.gib)
    lines = P.Batch.from_text(text)
    n, nbytes = lines.n, text.numel()

    def outputs():
        return (torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev),
                torch.zeros(n, dtype=torch.int32, device=dev))

    def event_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    handles = {}
    for name in sorted({x for p in PAIRS for x in p}):
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(lines, 1 << 16)
        handles[name] = sc
    res = {"card": card(), "n_lines": n, "bytes": nbytes, "gib": nbytes / 2 ** 30, "reps": args.reps,
           "hot_rows": {k: int(v.info().hot_rows) for k, v in handles.items()}, "pairs": {}}
    bad = 0
    for a, b in PAIRS:
        sc1, sc2 = handles[a], handles[b]
        got, want = outputs() + outputs(), outputs() + outputs()
        pair = P.ScannerPair(sc1, sc2)
        fused = lambda: pair.run_pair_lines(lines, flags, got[:3], got[3:])       # noqa: E731

        def single():
            sc1.run_batch(lines, flags, *want[:3])
            sc2.run_batch(lines, flags, *want[3:])
        fused()
        single()
        torch.cuda.synchronize()
        f_ms, s_ms = [], []
        for _ in range(args.reps):
            f_ms.append(event_ms(fused))
            s_ms.append(event_ms(single))
        stat = lambda v: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)),   # noqa: E731
                          "median_gbps": nbytes / float(np.median(v)) / 1e6}
        r = {"fused": stat(f_ms), "single_pair": stat(s_ms), "single_over_fused": float(np.median(s_ms) / np.median(f_ms))}
        r["mismatched_words"] = sum(int((x != y).sum().item()) for x, y in zip(got, want))
        r["matches"] = [int(np.unpackbits(t.cpu().numpy().view(np.uint8)).sum()) for t in (got[0], got[3])]
        bad += r["mismatched_words"]
        res["pairs"]["%s+%s" % (a, b)] = r
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pair_lines_bench.json"), "w") as f:
            f.write(line + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
