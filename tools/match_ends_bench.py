#!/usr/bin/env python
"""Where the HalfFinalScanner matches of one long string end, with the whole GPU (pire_gpu_match_ends_string), against
counting them and scanning the same bytes.

    python tools/match_ends_bench.py [--reps 10] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only) before and after; tools/string_bench.py's
planted 1 KiB synthetic text at 64 MiB and at 4 GiB (one resident buffer); for the hf_glue10, headline and count_words5
images (tuned on a fixed-length view), median CUDA-event times of
    ends         pire_gpu_match_ends_string over the text as ONE string (*d_found zeroed in the window)
    count        pire_gpu_count_string over the same bytes (counters zeroed in the window)
    run          pire_gpu_run_string over the same bytes (the locate walk alone)
The capacity is the whole answer where its 12 bytes per entry fit in the free HBM, else 2^20 entries (the call then
still walks every byte twice but writes only the first entries).  The arms are warmed up, then timed in turns.  Every
call's *d_found must equal the sum of count_string's counters, and its match and state run_string's.  Exit 1 on any
mismatch.  One JSON line goes to stdout and to DIR/match_ends_bench.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from string_bench import card  # noqa: E402

RUN_BEGIN, RUN_END = 1, 2
MIB = 2 ** 20
IMAGES = ("hf_glue10", "headline", "count_words5")
ENTRY_BYTES = 12                    # u64 end + u32 id
SMALL_CAPACITY = 2 ** 20


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--gib", type=float, default=4.0, help="size of the large text (GiB)")
    ap.add_argument("--out", default=None, help="directory for match_ends_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    if not torch.cuda.is_available():
        sys.exit("match_ends_bench needs a CUDA device")
    stream = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731

    total = int(args.gib * 2 ** 30) // 1024 * 1024
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(total // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    texts = [("64MiB", dev[: 64 * MIB]), ("%gGiB" % args.gib, dev)]
    result = {"card_before": card(), "reps": args.reps}
    print(result["card_before"], flush=True)
    mismatches = 0

    for name in IMAGES:
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(P.Batch(dev[: 256 * MIB], fixed_len=4096))
        regs = max(1, sc.RegexpsCount())
        counts = torch.zeros(regs, dtype=torch.int64, device="cuda:0")
        words = torch.zeros(6, dtype=torch.int32, device="cuda:0")
        found = torch.zeros(1, dtype=torch.int64, device="cuda:0")

        def count(t):
            counts.zero_()
            N.check(N.lib.pire_gpu_count_string(sc._h, t.data_ptr(), t.numel(), RUN_BEGIN | RUN_END, None, counts.data_ptr(),
                                                words.data_ptr(), words.data_ptr() + 4, stream()), "count_string")

        def run(t):
            w = words.data_ptr() + 8
            N.check(N.lib.pire_gpu_run_string(sc._h, t.data_ptr(), t.numel(), RUN_BEGIN | RUN_END, None, w, None, w + 4, stream()),
                    "run_string")

        for label, t in texts:
            n = t.numel()
            count(t)
            entries = int(counts.sum().item())
            free, _ = torch.cuda.mem_get_info()
            capacity = entries if entries * ENTRY_BYTES + 2 * 2 ** 30 <= free else SMALL_CAPACITY
            ends = torch.empty(max(1, capacity), dtype=torch.int64, device="cuda:0")
            ids = torch.empty(max(1, capacity), dtype=torch.int32, device="cuda:0")

            def locate(t=t, ends=ends, ids=ids, capacity=capacity):
                found.zero_()
                w = words.data_ptr() + 16
                N.check(N.lib.pire_gpu_match_ends_string(sc._h, t.data_ptr(), t.numel(), RUN_BEGIN | RUN_END, None, 0, ends.data_ptr(),
                                                         ids.data_ptr(), capacity, found.data_ptr(), w, w + 4, stream()),
                        "match_ends_string")

            arms = {"ends": locate, "count": lambda: count(t), "run": lambda: run(t)}
            for fn in arms.values():                 # warm-up
                fn()
                fn()
            times = {k: [] for k in arms}
            for _ in range(args.reps):
                for k, fn in arms.items():           # the arms in turns
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1))
            row = {"bytes": n, "entries": entries, "capacity": capacity,
                   "entry_bytes_written": min(entries, capacity) * ENTRY_BYTES}
            for k, v in times.items():
                row[k + "_ms"] = float(np.median(v))
                row[k + "_gbs"] = n / row[k + "_ms"] / 1e6
            row["ends_over_count"] = row["ends_ms"] / row["count_ms"]
            row["ends_over_run"] = row["ends_ms"] / row["run_ms"]
            locate()
            run(t)
            w = words.cpu().numpy().view(np.uint32)
            got = int(found.item())
            if got != entries or (w[4], w[5]) != (w[2], w[3]):
                mismatches += 1
                print("MISMATCH %s %s: %d entries against %d counted; (final, state) %s, run_string %s"
                      % (name, label, got, entries, w[4:6], w[2:4]), file=sys.stderr)
            if capacity == entries and entries > 1:
                ok, hist = True, torch.zeros(regs, dtype=torch.int64, device="cuda:0")
                for lo in range(0, entries, 2 ** 28):             # in slices: the answer may fill most of HBM
                    hi = min(entries, lo + 2 ** 28 + 1)
                    ok = ok and bool((ends[lo + 1:hi] >= ends[lo:hi - 1]).all())
                    hist += torch.bincount(ids[lo:min(entries, lo + 2 ** 28)].long(), minlength=regs)
                ok = ok and hist.tolist() == counts.tolist()
                row["ascending_and_histogram_equal"] = ok
                if not ok:
                    mismatches += 1
                    print("MISMATCH %s %s: ends out of order or histogram differs from count_string" % (name, label), file=sys.stderr)
            result["%s_%s" % (name, label)] = row
            print(name, label, json.dumps(row), flush=True)
            del ends, ids
            torch.cuda.empty_cache()

    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "match_ends_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
