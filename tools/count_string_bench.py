#!/usr/bin/env python
"""HalfFinalScanner counts of one long string with the whole GPU (pire_gpu_count_string), against what it costs and
what the library offered before it.

    python tools/count_string_bench.py [--reps 10] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); tools/string_bench.py's planted
1 KiB synthetic text at 64 MiB and at 4 GiB (one resident buffer); for the hf_glue10, headline and count_words5
images (tuned on a fixed-length view), median CUDA-event times of
    count        pire_gpu_count_string over the text as ONE string
    run          pire_gpu_run_string over the same bytes (the locate walk alone: the difference is the cost of counting)
    batch        pire_gpu_count_batch over the same bytes as 1 KiB strings (a rate reference only: other answers)
    one_lane     pire_gpu_count_batch with n = 1 at 64 MiB, the only exact route before (fewer repetitions: it is slow)
The arms are warmed up, then timed in turns (count, run, batch, count, run, batch, ...).  At 64 MiB count_string is
checked against the n = 1 result, counter by counter.  With oracle/_ref/test_file present it is also counted doubled to
>= 300 MB.  Exit 1 on any mismatch.  One JSON line goes to stdout and to DIR/count_string_bench.json."""
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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--one-lane-reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for count_string_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    if not torch.cuda.is_available():
        sys.exit("count_string_bench needs a CUDA device")
    stream = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731
    gbs = lambda nbytes, ms: nbytes / ms / 1e6                        # noqa: E731

    total = 4 * 2 ** 30
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(total // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    texts = [("64MiB", dev[: 64 * MIB]), ("4GiB", dev)]
    tf = os.path.join(ROOT, "oracle", "_ref", "test_file")
    if os.path.exists(tf):
        data = open(tf, "rb").read()
        while len(data) < 300_000_000:
            data += data
        texts.append(("test_file", torch.from_numpy(np.frombuffer(data, np.uint8).copy()).to("cuda:0")))
    result = {"card_before": card(), "reps": args.reps}
    print(result["card_before"], flush=True)
    mismatches = 0

    for name in IMAGES:
        sc = P.Scanner(W.load_image(name), 0)
        sc.Tune(P.Batch(dev[: 256 * MIB], fixed_len=4096))
        regs = max(1, sc.RegexpsCount())
        counts = torch.zeros(regs, dtype=torch.int64, device="cuda:0")
        words = torch.zeros(4, dtype=torch.int32, device="cuda:0")

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
            batch = P.Batch(t, fixed_len=1024, n=n // 1024) if n % 1024 == 0 else None
            rows = torch.empty((n // 1024, regs), dtype=torch.int32, device="cuda:0") if batch else None
            arms = {"count": lambda: count(t), "run": lambda: run(t)}
            if batch:
                arms["batch"] = lambda: N.check(N.lib.pire_gpu_count_batch(sc._h, t.data_ptr(), None, 1024, n // 1024, RUN_BEGIN | RUN_END,
                                                                           rows.data_ptr(), None, stream()), "count_batch")
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
            row = {"bytes": n}
            for k, v in times.items():
                row[k + "_ms"] = float(np.median(v))
                row[k + "_gbs"] = gbs(n, row[k + "_ms"])
            row["count_over_run"] = row["count_ms"] / row["run_ms"]
            count(t)
            got = [int(x) for x in counts.cpu().numpy()]
            row["matches"] = int(sum(got))
            run(t)
            w = words.cpu().numpy().view(np.uint32)
            if (w[0], w[1]) != (w[2], w[3]):
                mismatches += 1
                print("MISMATCH %s %s: count_string (final, state) %s, run_string %s" % (name, label, w[:2], w[2:]), file=sys.stderr)
            if label == "64MiB":
                # the only exact route before: one lane of count_batch walks the whole string
                one = torch.zeros(regs, dtype=torch.int32, device="cuda:0")
                offs = torch.tensor([0, n], dtype=torch.int64, device="cuda:0")
                ms = []
                for _ in range(args.one_lane_reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    N.check(N.lib.pire_gpu_count_batch(sc._h, t.data_ptr(), offs.data_ptr(), 0, 1, RUN_BEGIN | RUN_END, one.data_ptr(),
                                                       None, stream()), "count_batch n = 1")
                    e1.record()
                    e1.synchronize()
                    ms.append(e0.elapsed_time(e1))
                row["one_lane_ms"] = float(np.median(ms))
                row["one_lane_gbs"] = gbs(n, row["one_lane_ms"])
                want = [int(x) for x in one.cpu().numpy().view(np.uint32)]
                row["equals_one_lane"] = got == want
                if got != want:
                    mismatches += 1
                    print("MISMATCH %s: count_string %s, count_batch n = 1 %s" % (name, got, want), file=sys.stderr)
            result["%s_%s" % (name, label)] = row
            print(name, label, json.dumps(row), flush=True)
            del rows

    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "count_string_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
