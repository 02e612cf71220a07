#!/usr/bin/env python
"""One long string with the whole GPU (pire_gpu_run_string), measured against what the library reached before it.

    python tools/string_bench.py [--gib 4] [--reps 10] [--out DIR]

In one process: the card's name, power limit and SM clock (nvidia-smi, read-only); a resident buffer of 1 KiB synthetic
strings with plants, back to back; then, for the glue10 and headline images (tuned on a fixed-length view), CUDA-event
times of
    string        pire_gpu_run_string over the whole buffer as ONE string
    batch         pire_gpu_run_batch over the same bytes as 1 KiB strings (the rate the library reaches on them)
    warp64        pire_gpu_run_batch_ordered with n = 1 over a 64 MiB prefix: one warp, the best route before
    string64      pire_gpu_run_string over the same prefix
and the parity fixture (tests/golden/string_images.json.xz, a run of a's) at 64 MiB: the stitch's worst case.
Every run_string result is checked against run_batch_ordered with n = 1 on the same bytes, and against the oracle
(oracle/libpire_oracle.so) where the string is at most 1 GiB.  With oracle/_ref/test_file present it is also scanned
doubled to >= 300 MB, the shape of tools/ref_bench_continuity.sh.  Exit 1 on any mismatch.  One JSON line goes to
stdout and to DIR/string_bench.json."""
import argparse
import base64
import json
import lzma
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

RUN_BEGIN, RUN_END = 1, 2
MIB = 2 ** 20


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def parity_image():
    with open(os.path.join(ROOT, "tests", "golden", "string_images.json.xz"), "rb") as f:
        d = json.loads(lzma.decompress(f.read()))["images"]
    return lzma.decompress(base64.b64decode(d["parity"]["image_xz"]))


class Bench:
    def __init__(self, reps):
        import torch
        self.torch = torch
        self.reps = reps
        self.out = torch.zeros(3, dtype=torch.int32, device="cuda:0")
        self.mismatches = 0

    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def time(self, fn):
        """Median milliseconds of `reps` launches after two warm-up ones."""
        torch = self.torch
        for _ in range(2):
            fn()
        times = []
        for _ in range(self.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        return float(np.median(times))

    def string(self, sc, ptr, n):
        from pire_b200 import _native as N
        o = self.out.data_ptr()
        N.check(N.lib.pire_gpu_run_string(sc._h, ptr, n, RUN_BEGIN | RUN_END, None, o, o + 4, o + 8, self.stream()), "run_string")

    def warp(self, sc, ptr, n, order, offs, out):
        from pire_b200 import _native as N
        o = out.data_ptr()
        N.check(N.lib.pire_gpu_run_batch_ordered(sc._h, ptr, offs.data_ptr(), order.data_ptr(), 1, RUN_BEGIN | RUN_END, o, o + 4,
                                                 o + 8, self.stream()), "run_batch_ordered")

    def check(self, what, sc, dev, n, orc=None, host=None):
        """run_string's (match, mask, state) against the one-warp route, and against the oracle when given."""
        torch = self.torch
        offs = torch.tensor([0, n], dtype=torch.int64, device="cuda:0")
        order = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        ref = torch.zeros(3, dtype=torch.int32, device="cuda:0")
        self.string(sc, dev.data_ptr(), n)
        self.warp(sc, dev.data_ptr(), n, order, offs, ref)
        got = tuple(int(x) for x in self.out.cpu().numpy().view(np.uint32))
        want = tuple(int(x) for x in ref.cpu().numpy().view(np.uint32))
        ok = got == want
        if orc is not None:
            from string_oracle import run_from
            ok = ok and got == run_from(orc, host[:n], None, True, True)
        if not ok:
            self.mismatches += 1
            print("MISMATCH %s: run_string %s, one warp %s" % (what, got, want), file=sys.stderr)
        return got


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gib", type=float, default=4.0, help="size of the resident buffer (GiB)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for string_bench.json")
    args = ap.parse_args()

    import torch
    import pire_b200 as P
    from pire_b200 import workloads as W
    from refpire import Oracle
    if not torch.cuda.is_available():
        sys.exit("string_bench needs a CUDA device")
    b = Bench(args.reps)
    result = {"card": card(), "gib": args.gib, "reps": args.reps}
    print(result["card"], flush=True)

    total = int(args.gib * 2 ** 30) // 1024 * 1024
    prefix = min(64 * MIB, total)
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    W.SynthSpec(total // 1024, 1024, plants=W.GLUE10_PLANTS + W.HEADLINE_PLANTS).fill_device(dev)
    host_prefix = dev[:prefix].cpu().numpy()
    offs = torch.tensor([0, prefix], dtype=torch.int64, device="cuda:0")
    order = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    nstr = total // 1024
    bits = torch.zeros((nstr + 31) // 32, dtype=torch.int32, device="cuda:0")
    masks = torch.zeros(nstr, dtype=torch.int32, device="cuda:0")
    spare = torch.zeros(3, dtype=torch.int32, device="cuda:0")
    whole = P.Batch(dev, fixed_len=1024, n=nstr)
    gbs = lambda nbytes, ms: nbytes / ms / 1e6          # noqa: E731

    for name in ("glue10", "headline"):
        image = W.load_image(name)
        sc = P.Scanner(image, 0)
        sc.Tune(P.Batch(dev[: min(total, 256 * MIB) // 4096 * 4096], fixed_len=4096))
        orc = Oracle(image)
        row = {}
        row["string_ms"] = b.time(lambda: b.string(sc, dev.data_ptr(), total))
        row["batch_ms"] = b.time(lambda: sc.run_batch(whole, RUN_BEGIN | RUN_END, bits, masks))
        row["warp64_ms"] = b.time(lambda: b.warp(sc, dev.data_ptr(), prefix, order, offs, spare))
        row["string64_ms"] = b.time(lambda: b.string(sc, dev.data_ptr(), prefix))
        row["string_gbs"] = gbs(total, row["string_ms"])
        row["batch_gbs"] = gbs(total, row["batch_ms"])
        row["warp64_gbs"] = gbs(prefix, row["warp64_ms"])
        row["string64_gbs"] = gbs(prefix, row["string64_ms"])
        row["string_over_warp"] = row["string_gbs"] / row["warp64_gbs"]
        row["string64_over_warp"] = row["string64_gbs"] / row["warp64_gbs"]
        row["result"] = b.check(name + " whole buffer", sc, dev, total, orc if total <= 2 ** 30 else None,
                                dev.cpu().numpy() if total <= 2 ** 30 else None)
        b.check(name + " 64 MiB prefix", sc, dev, prefix, orc, host_prefix)
        result[name] = row
        print(name, json.dumps(row), flush=True)

    # the worst case: walks from different states never fall together
    image = parity_image()
    sc = P.Scanner(image, 0)
    # an odd head: pieces are whole 32-byte blocks, so behind an even one the guess (the even state) is right everywhere
    a = torch.full((prefix + 2,), ord("a"), dtype=torch.uint8, device="cuda:0")
    odd = a[1:]
    row = {"string64_ms": b.time(lambda: b.string(sc, odd.data_ptr(), prefix + 1))}
    row["string64_gbs"] = gbs(prefix + 1, row["string64_ms"])
    row["result"] = b.check("parity 64 MiB", sc, odd, prefix + 1, Oracle(image), odd.cpu().numpy())
    result["parity"] = row
    print("parity", json.dumps(row), flush=True)
    del a

    # the reference harness's shape: oracle/_ref/test_file doubled to >= 300 MB, one string
    tf = os.path.join(ROOT, "oracle", "_ref", "test_file")
    if os.path.exists(tf):
        data = open(tf, "rb").read()
        while len(data) < 300_000_000:
            data += data
        host = np.frombuffer(data, np.uint8)
        t = torch.from_numpy(host.copy()).to("cuda:0")
        for name in ("headline", "glue10"):
            image = W.load_image(name)
            sc = P.Scanner(image, 0)
            ms = b.time(lambda: b.string(sc, t.data_ptr(), len(data)))
            res = b.check("test_file " + name, sc, t, len(data), Oracle(image), host)
            result["test_file_" + name] = {"bytes": len(data), "ms": ms, "gbs": gbs(len(data), ms), "result": res}
            print("test_file", name, json.dumps(result["test_file_" + name]), flush=True)

    result["mismatches"] = b.mismatches
    line = json.dumps(result, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "string_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(1 if b.mismatches else 0)


if __name__ == "__main__":
    main()
