#!/usr/bin/env python
"""Where the HalfFinalScanner matches of many streams end (pire_gpu_match_ends_batch_from), against counting them
(pire_gpu_count_batch_from) on the same bytes.

    python tools/match_ends_batch_bench.py [--reps 10] [--gib 4] [--out DIR]

In one process: synthetic 1 KiB strings with the glue10 and headline plants, --gib GiB of them in one resident buffer,
for the hf_glue10 and count_words5 images, each tuned on a sample.  Median CUDA-event times of
    count        pire_gpu_count_batch_from with d_start == NULL (u64 rows zeroed once, before the first call)
    ends         pire_gpu_match_ends_batch_from with d_start == NULL, one call (*d_found zeroed in the window)
    ends_chain4  the same strings cut into four rounds of 256 B (four fixed-length batches), chained in place through
                 one state array and one position array (both reset in the window): BEGIN on the first round, END on the
                 last
The capacity is the whole answer where its 16 bytes per entry (u32 string, u64 end, u32 id) fit in the free HBM, else
as many entries as fit (the call then still counts every entry but writes only the first ones).  Before any timing the
per-string histograms of the entries are checked against count's rows (where the whole answer fits), *d_found against
their sum, and match bits and states against count's.  The arms are warmed up, then timed in turns.  Each row carries
the card's name, power limit and SM clock (nvidia-smi, read-only) as read just after it was timed.  Exit 1 on any
mismatch.  One JSON line goes to stdout and to DIR/match_ends_batch_bench.json."""
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
ENTRY_BYTES = 16


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--out", default=None, help="directory for match_ends_batch_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    if not torch.cuda.is_available():
        sys.exit("match_ends_batch_bench needs a CUDA device")
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
        rows = torch.zeros((n, regs), dtype=torch.int64, device="cuda:0")
        words = (n + 31) // 32
        bits = torch.zeros((3, words), dtype=torch.int32, device="cuda:0")
        states = torch.zeros((3, n), dtype=torch.int32, device="cuda:0")
        pos = torch.zeros((2, n), dtype=torch.int64, device="cuda:0")
        found = torch.zeros(2, dtype=torch.int64, device="cuda:0")

        def count():
            N.check(N.lib.pire_gpu_count_batch_from(sc._h, dev.data_ptr(), None, length, n, RUN_BEGIN | RUN_END, None,
                                                    rows.data_ptr(), bits[0].data_ptr(), states[0].data_ptr(), stream()),
                    "count_batch_from")

        count()
        entries = int(rows.sum().item())
        free, _ = torch.cuda.mem_get_info()
        capacity = max(1, min(entries, (free - 2 * 2 ** 30) // ENTRY_BYTES))
        out_s = torch.empty(capacity, dtype=torch.int32, device="cuda:0")
        out_e = torch.empty(capacity, dtype=torch.int64, device="cuda:0")
        out_i = torch.empty(capacity, dtype=torch.int32, device="cuda:0")

        def call(corpus, fixed_len, flags, start, k):
            N.check(N.lib.pire_gpu_match_ends_batch_from(sc._h, corpus, None, fixed_len, n, flags, start, pos[k - 1].data_ptr(),
                                                         out_s.data_ptr(), out_e.data_ptr(), out_i.data_ptr(), capacity,
                                                         found[k - 1].data_ptr(), bits[k].data_ptr(), states[k].data_ptr(), stream()),
                    "match_ends_batch_from")

        def ends():
            found[0].zero_()
            pos[0].zero_()
            call(dev.data_ptr(), length, RUN_BEGIN | RUN_END, None, 1)

        def ends_chain4():
            found[1].zero_()
            pos[1].zero_()
            for r, p in enumerate(pieces):
                flags = (RUN_BEGIN if r == 0 else 0) | (RUN_END if r == ROUNDS - 1 else 0)
                call(p.data_ptr(), piece_len, flags, states[2].data_ptr() if r else None, 2)

        # equal answers first
        row = {"bytes": n * length, "entries": entries, "capacity": capacity, "entry_bytes_written": min(entries, capacity) * ENTRY_BYTES}
        for what, fn, k in (("ends", ends, 1), ("ends_chain4", ends_chain4, 2)):
            fn()
            ok = int(found[k - 1].item()) == entries and bool((bits[k] == bits[0]).all()) and bool((states[k] == states[0]).all())
            ok = ok and bool((pos[k - 1] == length).all())
            if capacity == entries:
                key = out_s.long() * regs + out_i.long()
                ok = ok and bool((torch.bincount(key, minlength=n * regs).view(n, regs) == rows).all())
            row[what + "_equal"] = ok
            if not ok:
                mismatches += 1
                print("MISMATCH %s %s: entries, bits, states or positions differ from count_batch_from" % (name, what), file=sys.stderr)

        arms = {"count": count, "ends": ends, "ends_chain4": ends_chain4}
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
        row["ends_over_count"] = row["ends_ms"] / row["count_ms"]
        row["ends_chain4_over_count"] = row["ends_chain4_ms"] / row["count_ms"]
        row["card"] = card()
        result[name] = row
        print(name, json.dumps(row), flush=True)
        del rows, out_s, out_e, out_i
        torch.cuda.empty_cache()

    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "match_ends_batch_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
