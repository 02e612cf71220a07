#!/usr/bin/env python
"""A batch of streams resumed from per-string states (pire_gpu_run_batch_from), measured against pire_gpu_run_batch.

    python tools/batch_resume_bench.py [--gib 4] [--reps 5] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); the glued workload of bench.py (1 KiB
synthetic strings with the glue10 plants, resident in HBM, the scanner tuned and auto-selected on the batch as bench.py
does); then
  1. run_batch against run_batch_from with every start = Initialize() and BEGIN|END: the words (match bits, accept masks,
     StateIndex) compared one for one, and the two timed with CUDA events in three alternating pairs (median of `reps`
     launches each);
  2. the same strings cut into 4 rounds of 256 bytes, each round a fixed-length batch laid out round-major, chained in
     place through one state buffer (BEGIN on the first round, END on the last): the final words compared with
     run_batch over the whole strings, every round timed.
Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/batch_resume_bench.json."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

STRING_LEN = 1024
ROUNDS = 4


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


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

    dev = torch.device("cuda:0")
    n = int(args.gib * 2 ** 30) // STRING_LEN
    spec = W.SynthSpec(n, STRING_LEN, plants=W.GLUE10_PLANTS)
    corpus = torch.empty(spec.total_bytes(), dtype=torch.uint8, device=dev)
    spec.fill_device(corpus)
    batch = P.Batch(corpus, fixed_len=STRING_LEN, n=n)
    sc = P.Scanner(W.load_image("glue10"), 0)
    sc.Tune(batch, min(n, 16384))
    variant_ms = sc.AutoSelect(batch)
    chosen = N.VARIANT_NAMES.get(sc.info().variant, str(sc.info().variant))
    flags = N.RUN_BEGIN | N.RUN_END
    words = (n + 31) // 32

    def outputs():
        return (torch.zeros(words, dtype=torch.int32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev),
                torch.zeros(n, dtype=torch.int32, device=dev))

    def timed(fn):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    # 1. run_batch against run_batch_from from Initialize()
    base, resumed = outputs(), outputs()
    init = torch.full((n,), sc.Initialize(), dtype=torch.int32, device=dev)
    run = lambda: sc.run_batch(batch, flags, *base)
    run_from = lambda: sc.run_batch(batch, flags, *resumed, start_idx=init)
    pairs = []
    for _ in range(3):
        pairs.append((timed(run), timed(run_from)))
    torch.cuda.synchronize()
    mismatch_identity = sum(int((a != b).sum().item()) for a, b in zip(base, resumed))
    gbps = lambda ms: n * STRING_LEN / ms / 1e6

    # 2. four rounds of 256 bytes, round-major, chained in place
    piece = STRING_LEN // ROUNDS
    rows = corpus[: n * STRING_LEN].view(n, STRING_LEN)
    round_batches = [P.Batch(rows[:, r * piece:(r + 1) * piece].contiguous(), fixed_len=piece, n=n) for r in range(ROUNDS)]
    chained = outputs()
    state = chained[2]

    def chain(times=None):
        state.fill_(sc.Initialize())
        for r, b in enumerate(round_batches):
            f = (N.RUN_BEGIN if r == 0 else 0) | (N.RUN_END if r == ROUNDS - 1 else 0)
            last = r == ROUNDS - 1
            if times is not None:
                times[r][0].record()
            sc.run_batch(b, f, chained[0] if last else None, chained[1] if last else None, state, start_idx=state)
            if times is not None:
                times[r][1].record()

    chain()
    round_ms = []
    for _ in range(args.reps):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(ROUNDS)]
        torch.cuda.synchronize()
        chain(ev)
        torch.cuda.synchronize()
        round_ms.append([a.elapsed_time(b) for a, b in ev])
    round_ms = np.median(np.array(round_ms), axis=0)
    run()
    torch.cuda.synchronize()
    mismatch_chain = sum(int((a != b).sum().item()) for a, b in zip(base, chained))

    res = {
        "card": card(),
        "n_strings": n, "string_len": STRING_LEN, "gib": n * STRING_LEN / 2 ** 30,
        "variant": chosen, "variant_ms": variant_ms,
        "run_batch_ms": [p[0] for p in pairs], "run_batch_from_ms": [p[1] for p in pairs],
        "run_batch_gbps": [gbps(p[0]) for p in pairs], "run_batch_from_gbps": [gbps(p[1]) for p in pairs],
        "from_over_batch_median": float(np.median([p[1] for p in pairs]) / np.median([p[0] for p in pairs])),
        "identity_mismatched_words": mismatch_identity,
        "chained_round_ms": [float(x) for x in round_ms], "chained_total_ms": float(round_ms.sum()),
        "chained_gbps": gbps(float(round_ms.sum())),
        "chained_mismatched_words": mismatch_chain,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_resume_bench.json"), "w") as f:
            f.write(line + "\n")
    return 1 if mismatch_identity or mismatch_chain else 0


if __name__ == "__main__":
    sys.exit(main())
