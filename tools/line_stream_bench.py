#!/usr/bin/env python
"""Cost of streaming a text from host memory to the line kernels (pire_gpu_line_stream), against the link alone.

The text is tools/string_bench.py's planted corpus cut into lines of 80 to 120 bytes, as large as the host's RAM
allows (--gib caps it; it must be held twice, pinned and pageable).  Timed end to end, from the first feed to the
last result on the host, medians of --reps with min and max:
  stream      LineStream frames from the pinned text, every frame scanned by pire_gpu_run_lines (glue10), or by
              pire_gpu_match_ends_lines + pire_gpu_match_starts_lines (hf_glue10 and its reversed scanner)
  copy        (a) the same bytes copied host to device alone, in the same slot sizes through a ring of three slots
  resident    (b) pire_gpu_split_lines + the same scan on a resident 4 GiB part of the text (no copy)
  pageable    (c) the stream from a pageable copy of the text
and the stream for several slot sizes (the default is chosen from them), and tools/pigrep.py -c on a file.
Writes line_stream_bench.json under --out."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
GIB, MIB = 1 << 30, 1 << 20


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def fill_text(host, chunk=4 * GIB):
    """The planted corpus cut into 80..120-byte lines, generated on the device chunk by chunk into `host`."""
    import numpy as np
    import torch
    from pire_b200 import workloads as W
    rng = np.random.default_rng(2024)
    total = host.numel()
    dev = torch.empty(chunk, dtype=torch.uint8, device="cuda:0")
    pos = 0
    carry = 0
    while pos < total:
        n = min(chunk, total - pos)
        W.SynthSpec(n // 1024, 1024, first_string=pos // 1024,
                    plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev[: n // 1024 * 1024])
        ends = carry + np.cumsum(rng.integers(80, 121, size=n // 80 + 2))
        carry = int(ends[ends >= n][0] - n)
        ends = ends[ends < n]
        dev[torch.from_numpy(ends).to("cuda:0")] = 10
        host[pos:pos + n].copy_(dev[:n])
        pos += n
    del dev
    torch.cuda.empty_cache()


def timed(fn, reps):
    import torch
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return {"median_s": statistics.median(times), "min_s": min(times), "max_s": max(times)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gib", type=float, default=16.0, help="largest text to stream (GiB)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pigrep-gib", type=float, default=8.0, help="size of the file pigrep -c reads (GiB)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import pire_b200 as P
    from pire_b200 import _native as N
    from pire_b200 import workloads as W
    from start_images import START_IMAGES
    if not torch.cuda.is_available():
        sys.exit("line_stream_bench needs a CUDA device")
    result = {"card": card(), "mem_available_gib": mem_available() / GIB, "reps": args.reps}
    print(result["card"], flush=True)
    size = int(min(args.gib * GIB, 0.3 * mem_available())) // GIB * GIB
    result["text_gib"] = size / GIB
    host = torch.empty(size, dtype=torch.uint8, pin_memory=True)
    fill_text(host)
    pageable = np.empty(size, np.uint8)
    pageable[:] = host.numpy()
    print("text: %.0f GiB pinned + the same pageable" % (size / GIB), flush=True)
    sc = P.Scanner(W.load_image("glue10"), 0)
    hf, rev = P.Scanner(W.load_image("hf_glue10"), 0), P.Scanner(START_IMAGES["glue10"]["reversed"], 0)
    flags = N.RUN_BEGIN | N.RUN_END

    def scan_run(frame, out):
        bits = torch.empty((frame.n + 31) // 32, dtype=torch.int32, device="cuda:0")
        sc.run_batch(frame, flags, bits)
        out.append(bits)

    def scan_spans(frame, out):
        ends = P.LineMatchEnds(hf, 4 * MIB).Begin().Run(frame).End()
        st = P.MatchStarts(rev, ends, frame).StartsTensor()
        out.append((ends.FoundTensor(), st))

    def stream(src, slot_bytes, scan):
        def go():
            ls = P.LineStream(0, slot_bytes)
            out = []
            for f in ls.feed(src, last=True):
                scan(f, out)
            torch.cuda.synchronize()
            return [x.cpu() if torch.is_tensor(x) else x[0].cpu() for x in out]
        return go

    def copy_alone(slot_bytes):
        ring = [torch.empty(slot_bytes, dtype=torch.uint8, device="cuda:0") for _ in range(3)]

        def go():
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for k, lo in enumerate(range(0, size, slot_bytes)):
                    hi = min(size, lo + slot_bytes)
                    ring[k % 3][: hi - lo].copy_(host[lo:hi], non_blocking=True)
            s.synchronize()
        return go

    part = min(size, 4 * GIB)
    resident = host[:part].to("cuda:0")

    def resident_scan(scan):
        def go():
            b = P.Batch.from_text(resident)
            scan(b, [])
        return go

    rows = {}
    for slot_mib in (16, 64, 256):
        rows["copy_%d" % slot_mib] = copy_alone(slot_mib * MIB)
        rows["stream_run_%d" % slot_mib] = stream(host, slot_mib * MIB, scan_run)
    rows["stream_run_default"] = stream(host, 0, scan_run)
    rows["pageable_run_64"] = stream(pageable, 64 * MIB, scan_run)
    rows["stream_spans_64"] = stream(host, 64 * MIB, scan_spans)
    rows["pageable_spans_64"] = stream(pageable, 64 * MIB, scan_spans)
    rows["resident_run_4gib"] = resident_scan(scan_run)
    rows["resident_spans_4gib"] = resident_scan(scan_spans)
    for fn in rows.values():                              # warm every shape once
        fn()
    timing = {}
    for name, fn in rows.items():
        t = timed(fn, args.reps)
        nbytes = part if name.startswith("resident") else size
        t["gb_per_s"] = nbytes / t["median_s"] / 1e9
        timing[name] = t
        print("%-22s %8.3f s  (%.3f .. %.3f)  %7.2f GB/s" % (name, t["median_s"], t["min_s"], t["max_s"], t["gb_per_s"]), flush=True)
    result["timing"] = timing
    for slot_mib in (16, 64, 256):
        result["stream_over_copy_%d" % slot_mib] = timing["stream_run_%d" % slot_mib]["gb_per_s"] / timing["copy_%d" % slot_mib]["gb_per_s"]
    result["spans_over_copy_64"] = timing["stream_spans_64"]["gb_per_s"] / timing["copy_64"]["gb_per_s"]
    # the streamed answer is the resident one
    # (bits past a frame's lines are 0, so the streamed matches add up to the resident count)
    got = sum(int(unpack(b).sum()) for b in stream(host[:part], 64 * MIB, scan_run)())
    wb = []
    scan_run(P.Batch.from_text(resident), wb)
    assert got == int(unpack(wb[0].cpu()).sum()), "streamed matches differ from the resident ones"
    result["matches_4gib"] = got
    del resident
    torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in result.items() if k != "timing"}), flush=True)

    # pigrep -c on a file
    tmp = tempfile.mkdtemp()
    try:
        free_disk = shutil.disk_usage(tmp).free
        free_hbm = torch.cuda.mem_get_info()[0]
        result["disk_free_gib"], result["hbm_free_gib"] = free_disk / GIB, free_hbm / GIB
        fsize = int(min(args.pigrep_gib * GIB, size, 0.5 * free_disk)) // MIB * MIB
        path = os.path.join(tmp, "text.log")
        with open(path, "wb") as f:
            f.write(memoryview(host.numpy()[:fsize]))
        sc_path = os.path.join(tmp, "glue10.pire")
        with open(sc_path, "wb") as f:
            f.write(W.load_image("glue10"))
        t0 = time.perf_counter()
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pigrep.py"), "--scanner", sc_path, "-c", path],
                             capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT))
        dt = time.perf_counter() - t0
        result["pigrep_c"] = {"file_gib": fsize / GIB, "s": dt, "gb_per_s": fsize / dt / 1e9, "count": out.stdout.strip(),
                              "rc": out.returncode, "stderr": out.stderr[-500:]}
        print("pigrep -c %.1f GiB: %.2f s (%.2f GB/s, process start included) -> %s" % (fsize / GIB, dt, fsize / dt / 1e9,
                                                                                     out.stdout.strip()), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "line_stream_bench.json"), "w") as f:
            json.dump(result, f, indent=1)


def unpack(words):
    import numpy as np
    return np.unpackbits(words.numpy().view(np.uint8), bitorder="little")


if __name__ == "__main__":
    main()
