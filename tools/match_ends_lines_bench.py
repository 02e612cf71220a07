#!/usr/bin/env python
"""Where the HalfFinalScanner matches end in every line of a text (pire_gpu_match_ends_lines), against scanning and
counting the same lines and against walking them one line per lane.

    python tools/match_ends_lines_bench.py [--reps 10] [--gib 4] [--out DIR]

In one process: --gib GiB of synthetic text (1 KiB strings with the glue10 and headline plants) cut into lines of 80
to 120 bytes by writing a '\\n' at seeded random distances and at the end, resident on the device and split once
(pire_gpu_split_lines), for the hf_glue10 and count_words5 images, each tuned on the line batch.  Median CUDA-event
times, BEGIN and END, of
    run_lines        pire_gpu_run_lines (match bits and states)
    count_lines      pire_gpu_count_batch with PIRE_GPU_RUN_LINES (u32 rows)
    ends_lines       pire_gpu_match_ends_lines (*d_found zeroed in the window)
    ends_starts      ends_lines, then pire_gpu_match_starts_lines with the reversed GLUE10 patterns (hf_glue10 only)
    ends_per_lane    pire_gpu_match_ends_batch_from over the same offsets as a plain CSR batch: one line per lane, each
                     line with its '\\n' (one byte more per line) -- the walk the in-stream kernel replaces
The capacity is the whole answer where its 16 bytes per entry fit in the free HBM, else as many entries as fit.  Before
any timing, *d_found is checked against the sum of count_lines's rows, the entries' per-line histograms against those
rows (where the whole answer fits) and the match bits and states against run_lines's.  The arms are warmed up, then
timed in turns.  Each row carries the card's name, power limit and SM clock (nvidia-smi, read-only) as read just after
it was timed.  Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/match_ends_lines_bench.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from string_bench import card  # noqa: E402

RUN_BEGIN, RUN_END, RUN_LINES = 1, 2, 4
IMAGES = ("hf_glue10", "count_words5")
ENTRY_BYTES = 16
CHUNK = 1 << 27                 # entries per bincount in the histogram check


def make_text(torch, W, gib):
    size = int(gib * 2 ** 30) // 1024 * 1024
    dev = torch.empty(size, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(size // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    dev[dev == 10] = 32
    g = torch.Generator(device="cuda:0")
    g.manual_seed(7)
    steps = torch.randint(80, 121, (size // 80 + 1,), generator=g, device="cuda:0", dtype=torch.int64)
    at = torch.cumsum(steps, 0)
    dev[at[at < size]] = 10
    dev[-1] = 10            # the last line ends with a newline too, so the plain CSR batch of ends_per_lane lies in the text
    return dev


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--out", default=None, help="directory for match_ends_lines_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    from start_images import START_IMAGES
    if not torch.cuda.is_available():
        sys.exit("match_ends_lines_bench needs a CUDA device")
    stream = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731

    text = make_text(torch, W, args.gib)
    batch = P.Batch.from_text(text)
    n, offs, size = batch.n, batch.offsets.data_ptr(), text.numel()
    flags = RUN_BEGIN | RUN_END
    result = {"card_before": card(), "reps": args.reps, "bytes": size, "lines": n}
    print(result["card_before"], flush=True)
    mismatches = 0
    rev = P.Scanner(START_IMAGES["glue10"]["reversed"], 0)

    for name in IMAGES:
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(batch, 1 << 16)
        regs = max(1, sc.RegexpsCount())
        words = (n + 31) // 32
        bits = torch.zeros((3, words), dtype=torch.int32, device="cuda:0")
        states = torch.zeros((3, n), dtype=torch.int32, device="cuda:0")
        rows = torch.empty((n, regs), dtype=torch.int32, device="cuda:0")
        found = torch.zeros(2, dtype=torch.int64, device="cuda:0")
        pos = torch.zeros(n, dtype=torch.int64, device="cuda:0")

        def run_lines():
            N.check(N.lib.pire_gpu_run_lines(sc._h, text.data_ptr(), offs, None, n, flags, bits[0].data_ptr(), None,
                                             states[0].data_ptr(), stream()), "run_lines")

        def count_lines():
            N.check(N.lib.pire_gpu_count_batch(sc._h, text.data_ptr(), offs, 0, n, flags | RUN_LINES, rows.data_ptr(), None,
                                               stream()), "count_batch")

        count_lines()
        run_lines()
        entries = int(rows.sum(dtype=torch.int64).item())
        free, _ = torch.cuda.mem_get_info()
        capacity = max(1, min(entries, (free - 4 * 2 ** 30) // ENTRY_BYTES))
        out_l = torch.empty(capacity, dtype=torch.int32, device="cuda:0")
        out_e = torch.empty(capacity, dtype=torch.int64, device="cuda:0")
        out_i = torch.empty(capacity, dtype=torch.int32, device="cuda:0")
        starts = torch.empty(capacity, dtype=torch.int64, device="cuda:0") if name == "hf_glue10" else None

        def ends_lines():
            found[0].zero_()
            N.check(N.lib.pire_gpu_match_ends_lines(sc._h, text.data_ptr(), offs, n, flags, out_l.data_ptr(), out_e.data_ptr(),
                                                    out_i.data_ptr(), capacity, found[0].data_ptr(), bits[1].data_ptr(),
                                                    states[1].data_ptr(), stream()), "match_ends_lines")

        def ends_starts():
            ends_lines()
            N.check(N.lib.pire_gpu_match_starts_lines(rev._h, text.data_ptr(), offs, n, flags, 0, out_l.data_ptr(),
                                                      out_e.data_ptr(), out_i.data_ptr(), None, found[0].data_ptr(), capacity,
                                                      starts.data_ptr(), None, stream()), "match_starts_lines")

        def ends_per_lane():
            found[1].zero_()
            pos.zero_()
            N.check(N.lib.pire_gpu_match_ends_batch_from(sc._h, text.data_ptr(), offs, 0, n, flags, None, pos.data_ptr(),
                                                         out_l.data_ptr(), out_e.data_ptr(), out_i.data_ptr(), capacity,
                                                         found[1].data_ptr(), bits[2].data_ptr(), states[2].data_ptr(), stream()),
                    "match_ends_batch_from")

        # equal answers first
        row = {"entries": entries, "capacity": capacity, "entry_bytes_written": min(entries, capacity) * ENTRY_BYTES}
        ends_lines()
        ok = int(found[0].item()) == entries and bool((bits[1] == bits[0]).all()) and bool((states[1] == states[0]).all())
        if capacity == entries:
            hist = torch.zeros(n * regs, dtype=torch.int64, device="cuda:0")
            for k in range(0, entries, CHUNK):
                key = out_l[k:k + CHUNK].long() * regs + out_i[k:k + CHUNK].long()
                hist += torch.bincount(key, minlength=n * regs)
                del key
            ok = ok and bool((hist.view(n, regs) == rows.long()).all())
            del hist
        row["ends_lines_equal"] = ok
        if not ok:
            mismatches += 1
            print("MISMATCH %s: entries, bits or states differ from count_lines / run_lines" % name, file=sys.stderr)
        ends_per_lane()
        row["ends_per_lane_entries"] = int(found[1].item())

        arms = {"run_lines": run_lines, "count_lines": count_lines, "ends_lines": ends_lines, "ends_per_lane": ends_per_lane}
        if starts is not None:
            arms["ends_starts"] = ends_starts
        else:
            row["ends_starts_ms"] = "not measured (no reversed image of these patterns)"
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
            row[k + "_gbs"] = size / row[k + "_ms"] / 1e6
        row["ends_lines_over_count_lines"] = row["ends_lines_ms"] / row["count_lines_ms"]
        row["ends_per_lane_over_ends_lines"] = row["ends_per_lane_ms"] / row["ends_lines_ms"]
        row["card"] = card()
        result[name] = row
        print(name, json.dumps(row), flush=True)
        del rows, out_l, out_e, out_i, starts
        torch.cuda.empty_cache()

    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "match_ends_lines_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
