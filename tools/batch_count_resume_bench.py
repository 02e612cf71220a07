#!/usr/bin/env python
"""HalfFinalScanner counts of many streams resumed from their own states (pire_gpu_count_batch_from), against
pire_gpu_count_batch on the same bytes.

    python tools/batch_count_resume_bench.py [--reps 10] [--gib 4] [--out DIR]

In one process: synthetic 1 KiB strings with the glue10 and headline plants, --gib GiB of them
in one resident buffer, for the hf_glue10 and count_words5 images, each tuned on a sample.  Median CUDA-event times of
    batch        pire_gpu_count_batch: zeroes its u32 rows, then writes them
    from_null    pire_gpu_count_batch_from with d_start == NULL: adds into u64 rows (zeroed once, before the first call)
    chain4       the same strings cut into four rounds of 256 B (four fixed-length batches), chained in place through one
                 state array and one counts array: BEGIN on the first round, END on the last
Before any timing, the counts of from_null and chain4 are checked against batch's, counter by counter, and their match
bits and states against each other.  The arms are warmed up, then timed in turns (batch, from_null, chain4, batch, ...).
Each row carries the card's name, power limit and SM clock (nvidia-smi, read-only) as read just after it was timed.
Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/batch_count_resume_bench.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from string_bench import card  # noqa: E402

RUN_BEGIN, RUN_END = 1, 2
IMAGES = ("hf_glue10", "count_words5")
ROUNDS = 4


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--out", default=None, help="directory for batch_count_resume_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    if not torch.cuda.is_available():
        sys.exit("batch_count_resume_bench needs a CUDA device")
    stream = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731

    length = 1024
    n = int(args.gib * 2 ** 30) // length
    dev = torch.empty(n * length, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(n, length, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    piece_len = length // ROUNDS
    pieces = [dev.view(n, ROUNDS, piece_len)[:, r].contiguous().view(-1) for r in range(ROUNDS)]
    result = {"card_before": card(), "reps": args.reps, "strings": n, "string_bytes": length, "rounds": ROUNDS}
    print(result["card_before"], flush=True)
    mismatches = 0

    for name in IMAGES:
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(P.Batch(dev, fixed_len=length, n=n), 1 << 16)
        regs = max(1, sc.RegexpsCount())
        rows32 = torch.empty((n, regs), dtype=torch.int32, device="cuda:0")
        rows64 = torch.zeros((n, regs), dtype=torch.int64, device="cuda:0")
        chain64 = torch.zeros((n, regs), dtype=torch.int64, device="cuda:0")
        words = (n + 31) // 32
        bits = torch.zeros((3, words), dtype=torch.int32, device="cuda:0")
        states = torch.zeros((2, n), dtype=torch.int32, device="cuda:0")

        def batch():
            N.check(N.lib.pire_gpu_count_batch(sc._h, dev.data_ptr(), None, length, n, RUN_BEGIN | RUN_END, rows32.data_ptr(),
                                               bits[0].data_ptr(), stream()), "count_batch")

        def from_null():
            N.check(N.lib.pire_gpu_count_batch_from(sc._h, dev.data_ptr(), None, length, n, RUN_BEGIN | RUN_END, None,
                                                    rows64.data_ptr(), bits[1].data_ptr(), states[0].data_ptr(), stream()),
                    "count_batch_from")

        def chain4():
            st = states[1].data_ptr()
            for r, p in enumerate(pieces):
                flags = (RUN_BEGIN if r == 0 else 0) | (RUN_END if r == ROUNDS - 1 else 0)
                N.check(N.lib.pire_gpu_count_batch_from(sc._h, p.data_ptr(), None, piece_len, n, flags, st if r else None,
                                                        chain64.data_ptr(), bits[2].data_ptr() if r == ROUNDS - 1 else None, st,
                                                        stream()), "count_batch_from round %d" % r)

        # equal answers first, on counters zeroed once
        batch()
        from_null()
        chain4()
        want = rows32.cpu().numpy().view(np.uint32).astype(np.int64)
        row = {"bytes": n * length, "matches": int(want.sum())}
        for what, got in (("from_null", rows64), ("chain4", chain64)):
            ok = bool((got.cpu().numpy() == want).all())
            row[what + "_equal_counts"] = ok
            if not ok:
                mismatches += 1
                print("MISMATCH %s %s: counts differ from count_batch" % (name, what), file=sys.stderr)
        hb = bits.cpu().numpy()
        hs = states.cpu().numpy()
        row["equal_bits_and_states"] = bool((hb[0] == hb[1]).all() and (hb[0] == hb[2]).all() and (hs[0] == hs[1]).all())
        if not row["equal_bits_and_states"]:
            mismatches += 1
            print("MISMATCH %s: match bits or states differ" % name, file=sys.stderr)

        arms = {"batch": batch, "from_null": from_null, "chain4": chain4}
        for fn in arms.values():                     # warm-up
            fn()
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():               # the arms in turns
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
        for k, v in times.items():
            row[k + "_ms"] = float(np.median(v))
            row[k + "_ms_range"] = [float(min(v)), float(max(v))]
            row[k + "_gbs"] = n * length / row[k + "_ms"] / 1e6
        row["from_null_over_batch"] = row["from_null_ms"] / row["batch_ms"]
        row["chain4_over_batch"] = row["chain4_ms"] / row["batch_ms"]
        row["card"] = card()
        result[name] = row
        print(name, json.dumps(row), flush=True)
        del rows32, rows64, chain64

    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_count_resume_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
