#!/usr/bin/env python
"""pire_gpu_slow_run_batch (Pire::SlowScanner, patterns that cannot be determinised) measured on synthetic text.

    python tools/slow_bench.py [--gib 4] [--reps 5] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); `gib` GiB of 1 KiB printable-ASCII
strings (workloads.SynthSpec, GLUE10 plants), then for each SlowScanner of tests/golden/slow_images.json.xz below --
a.{30}$, foo.{64}bar, a.{100}$ (lane path), ^.{0,80}error.{200}$ and internationalization at distance 1 (warp path) --
the batch with Begin and End, timed with CUDA events after one warm-up: medians, minimum and maximum over `reps`, and the
rate over the batch.  One line-text run (the same bytes cut into 80-120-byte lines, PIRE_GPU_RUN_LINES) per scanner, and
pire_gpu_run_batch of the glued 10-pattern DFA (glue10) on the same strings as context.  One JSON line goes to stdout
and to DIR/slow_bench.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from match_ends_lines_bench import make_text  # noqa: E402
from pair_bench import card  # noqa: E402

SCANNERS = ["heavy/a30", "heavy/foo64bar", "heavy/a100", "heavy/error200", "approx1"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    from slow_fixtures import SLOW
    if not torch.cuda.is_available():
        sys.exit("slow_bench needs a CUDA device")

    dev = torch.device("cuda:0")
    flags = N.RUN_BEGIN | N.RUN_END
    gpu = card()                  # name, power limit and SM clock; read again right after the timed runs
    n = int(args.gib * 2 ** 30) // 1024
    corpus = torch.empty(n * 1024, dtype=torch.uint8, device=dev)
    W.SynthSpec(n, 1024, plants=W.GLUE10_PLANTS).fill_device(corpus)
    batch = P.Batch(corpus, fixed_len=1024, n=n)
    bits = torch.empty((n + 31) // 32, dtype=torch.int32, device=dev)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ms)), "min_ms": min(ms), "max_ms": max(ms),
                "gbps": corpus.numel() / (float(np.median(ms)) * 1e6)}

    rows = {}
    for name in SCANNERS:
        e = next(x for x in SLOW if x.name == name)
        sc = P.SlowScanner(e.image, 0)
        info = sc.info()
        row = {"states": info.states, "letters": info.letters, "path": "lane" if info.states <= 256 else "warp",
               "table_bytes": info.table_bytes, "shared_bytes": info.shared_bytes}
        row["batch"] = timed(lambda: sc.run_batch(batch, flags, bits, None))
        row["matches"] = int(np.unpackbits(bits.cpu().numpy().view(np.uint8))[:n].sum())
        rows[name] = row
        print(name, json.dumps(row), flush=True)
    del batch

    # the same bytes as lines of text
    text = make_text(torch, W, args.gib)
    lines = P.Batch.from_text(text)
    lbits = torch.empty((lines.n + 31) // 32, dtype=torch.int32, device=dev)
    for name in SCANNERS:
        e = next(x for x in SLOW if x.name == name)
        sc = P.SlowScanner(e.image, 0)
        rows[name]["lines"] = timed(lambda: sc.run_batch(lines, flags, lbits, None))
        print(name, "lines", json.dumps(rows[name]["lines"]), flush=True)
    del lines, text

    batch = P.Batch(corpus, fixed_len=1024, n=n)
    dfa = P.Scanner(W.load_image("glue10"), 0)
    context = timed(lambda: dfa.run_batch(batch, flags, bits, None, None))

    result = {"bench": "slow_bench", "card": gpu, "card_after": card(), "gib": args.gib, "strings": n, "string_bytes": 1024, "reps": args.reps,
              "scanners": rows, "dfa_glue10_run_batch": context}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "slow_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
