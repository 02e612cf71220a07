#!/usr/bin/env python
r"""Where the HalfFinalScanner matches start (pire_gpu_match_starts_string / _batch), against finding where they end.

    python tools/match_starts_bench.py [--reps 5] [--gib 4] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only) before and after; tools/string_bench.py's
planted 1 KiB synthetic text of --gib GiB, as ONE string and as a batch of 1 KiB strings; median CUDA-event times of
    ends        match ends alone (pire_gpu_match_ends_string / _batch_from, *d_found and d_pos zeroed in the window)
    starts      match starts alone, over the entries of that call
    chained     both on one stream, the starts reading *d_found on the device
for the workloads
The scanners are the glue10 and words sets of tests/golden/start_images.json.xz: the forward HalfFinalScanner (glue10's
is hf_glue10) and the same patterns reversed (Fsm::Reverse(), no Surround()), glued in the same order.
    glue10_string       hf_glue10 / reversed GLUE10 on the one string, max_back = 4096
    glue10_string_mb0   the same with max_back = 0: the text ends with "hello world", and the walk of the never-dying
                        reversed hello\s+w.+d$ goes back to the text's start, at the speed of one lane; timed once, reported
    glue10_batch        hf_glue10 / reversed GLUE10 on the batch
    words_batch         [a-z]+ forward / reversed on the batch: nearly every lowercase byte ends a match; the capacity
                        is what the free HBM allows
Every starts result is spot-checked on a sample of entries against the in-repo oracle (a reversed walk of the reversed image from the
entry's end, testing its regexp id after every byte); the max_back = 0 answers must equal the max_back = 4096 ones
wherever those are not open.  Exit 1 on a mismatch.  One JSON line goes to stdout and to DIR/match_starts_bench.json."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from string_bench import card  # noqa: E402

RUN_BEGIN, RUN_END = 1, 2
NO_START = 0xFFFFFFFFFFFFFFFF
SAMPLE = 300


def oracle_start(lib, sc, text, lo, e, rid, begin, with_end):
    """The leftmost s in [lo, e] whose reversed walk from e accepts regexp rid (BeginMark at s == 0 when begin)."""
    buf = (C.c_uint64 * 64)()

    def acc(st):
        return lib.pire_oracle_final(sc, st) and rid in [buf[j] for j in range(lib.pire_oracle_accepted(sc, st, buf, 64))]

    best = NO_START
    for te in (False, True) if with_end else (False,):
        st = lib.pire_oracle_initial(sc)
        if te:
            st = lib.pire_oracle_step(sc, st, 259)
        here = NO_START
        if acc(st):
            here = e
        for p in range(e - 1, lo - 1, -1):
            st = lib.pire_oracle_step(sc, st, int(text[p]))
            if acc(st):
                here = p
        if begin and lo == 0 and acc(lib.pire_oracle_step(sc, st, 258)):
            here = 0
        if here != NO_START and (best == NO_START or here < best):
            best = here
    return best


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    from refpire import Oracle
    from string_oracle import _lib
    if not torch.cuda.is_available():
        sys.exit("match_starts_bench needs a CUDA device")
    stream = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731

    total = int(args.gib * 2 ** 30) // 1024 * 1024
    n = total // 1024
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(n, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    # the one string ends with a match of hello\s+w.+d$: its reversed .+ never dies on this text (it has no newline), so
    # without max_back that entry walks back to the text's start (twice: it sits at the text's end under END)
    tail = np.frombuffer(b"hello world", np.uint8)
    dev[total - tail.size:] = torch.from_numpy(tail.copy()).to("cuda:0")
    text = dev.cpu().numpy()
    result = {"card_before": card(), "reps": args.reps, "bytes": total, "strings": n}
    print(result["card_before"], flush=True)
    mismatches = 0
    rng = np.random.default_rng(7)

    def timed(arms, reps):
        for fn in arms.values():
            fn()
        times = {k: [] for k in arms}
        for _ in range(reps):
            for k, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
        return {k + "_ms": float(np.median(v)) for k, v in times.items()}

    from start_images import START_IMAGES
    for label in ("glue10", "words"):
        fwd_image, rev_image = START_IMAGES[label]["forward"], START_IMAGES[label]["reversed"]
        fwd, rev = P.Scanner(fwd_image, 0), P.Scanner(rev_image, 0)
        orc, lib = Oracle(rev_image), _lib()
        sc = C.byref(orc._sc)
        found = torch.zeros(1, dtype=torch.int64, device="cuda:0")
        pos = torch.zeros(n, dtype=torch.int64, device="cuda:0")
        flags = RUN_BEGIN | RUN_END
        shapes = (("string", 4096), ("string_mb0", 0), ("batch", 0)) if label == "glue10" else (("batch", 0),)
        for shape, max_back in shapes:
            one = shape.startswith("string")
            # how many entries, then buffers for as many as the free HBM holds (25 bytes each with strings and starts)
            found.zero_()
            pos.zero_()
            if one:
                N.check(N.lib.pire_gpu_match_ends_string(fwd._h, dev.data_ptr(), total, flags, None, 0, None, None, 0,
                                                         found.data_ptr(), None, None, stream()), "ends")
            else:
                N.check(N.lib.pire_gpu_match_ends_batch_from(fwd._h, dev.data_ptr(), None, 1024, n, flags, None, pos.data_ptr(),
                                                             None, None, None, 0, found.data_ptr(), None, None, stream()), "ends")
            entries = int(found.item())
            free, _ = torch.cuda.mem_get_info()
            cap = max(1, min(entries, (free - 4 * 2 ** 30) // 25))
            strings = torch.empty(cap, dtype=torch.int32, device="cuda:0")
            ends = torch.empty(cap, dtype=torch.int64, device="cuda:0")
            ids = torch.empty(cap, dtype=torch.int32, device="cuda:0")
            starts = torch.empty(cap, dtype=torch.int64, device="cuda:0")
            opened = torch.empty(cap, dtype=torch.uint8, device="cuda:0")

            def do_ends():
                found.zero_()
                if one:
                    N.check(N.lib.pire_gpu_match_ends_string(fwd._h, dev.data_ptr(), total, flags, None, 0, ends.data_ptr(),
                                                             ids.data_ptr(), cap, found.data_ptr(), None, None, stream()), "ends")
                else:
                    pos.zero_()
                    N.check(N.lib.pire_gpu_match_ends_batch_from(fwd._h, dev.data_ptr(), None, 1024, n, flags, None,
                                                                 pos.data_ptr(), strings.data_ptr(), ends.data_ptr(),
                                                                 ids.data_ptr(), cap, found.data_ptr(), None, None, stream()),
                            "ends")

            def do_starts():
                if one:
                    N.check(N.lib.pire_gpu_match_starts_string(rev._h, dev.data_ptr(), total, 0, flags, max_back, ends.data_ptr(),
                                                               ids.data_ptr(), None, found.data_ptr(), cap, starts.data_ptr(),
                                                               opened.data_ptr(), stream()), "starts")
                else:
                    N.check(N.lib.pire_gpu_match_starts_batch(rev._h, dev.data_ptr(), None, 1024, n, pos.data_ptr(), flags,
                                                              max_back, strings.data_ptr(), ends.data_ptr(), ids.data_ptr(), None,
                                                              found.data_ptr(), cap, starts.data_ptr(), opened.data_ptr(),
                                                              stream()), "starts")

            def chained():
                do_ends()
                do_starts()

            do_ends()
            row = {"entries": entries, "capacity": cap, "max_back": max_back}
            if shape == "string_mb0":
                # the worst case: timed once, with no warm-up run of its own
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                do_starts()
                e1.record()
                e1.synchronize()
                row["starts_ms"] = e0.elapsed_time(e1)
            else:
                row.update(timed({"ends": do_ends, "starts": do_starts, "chained": chained}, args.reps))
                chained()
            k = min(entries, cap)
            row["open_entries"] = int(opened[:k].sum().item())
            bad = 0
            if shape == "string_mb0":
                ref = result["%s_string" % label]["_starts"]
                s_h = starts[:k].cpu().numpy().view(np.uint64)
                same = ~ref[1]
                bad = int((s_h[same] != ref[0][same]).sum())
            else:
                pick = torch.from_numpy(np.sort(rng.choice(k, size=min(SAMPLE, k), replace=False))).to("cuda:0") if k else None
                sample = [] if pick is None else list(zip(*(t[pick].cpu().numpy().tolist() for t in (ends, ids, strings if not one else ids, starts))))
                for e, rid, si, got in sample:
                    got &= NO_START
                    rid &= 0xFFFFFFFF
                    if one:
                        lo = max(0, e - max_back) if max_back else 0
                        want = oracle_start(lib, sc, text, lo, e, rid, True, e == total)
                    else:
                        base = (si & 0xFFFFFFFF) * 1024
                        want = oracle_start(lib, sc, text[base:base + 1024], 0, e, rid, True, e == 1024)
                    if got != want:
                        bad += 1
                        print("MISMATCH %s %s end %d id %d: start %d, oracle %d" % (label, shape, e, rid, got, want), file=sys.stderr)
            row["spot_check_mismatches"] = bad
            mismatches += bad
            if shape == "string":
                row["_starts"] = (starts[:k].cpu().numpy().view(np.uint64), opened[:k].cpu().numpy().astype(bool))
            result["%s_%s" % (label, shape)] = row
            print(label, shape, json.dumps({k2: v for k2, v in row.items() if not k2.startswith("_")}), flush=True)
            del strings, ends, ids, starts, opened
            torch.cuda.empty_cache()

    for v in result.values():
        if isinstance(v, dict):
            v.pop("_starts", None)
    result["card_after"] = card()
    result["mismatches"] = mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "match_starts_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
