#!/usr/bin/env python
"""What the stitch of pire_gpu_run_string costs, by the shape of the text and the choice of the guess.

    python tools/string_stitch_probe.py

One string of 1, 4 and 16 MiB from a buffer of 1 KiB synthetic strings, back to back, with plants (every 8th string,
the glue10 and headline literals) and without; the headline and glue10 scanners, untuned and tuned on that buffer (a
4 KiB fixed-length view).  Each line: the case, the length, the wall time of one synchronised call, and (match word,
mask, StateIndex).  With plants, the scanners remember a match until the string ends; untuned glue10's guess (hot id 0,
the resting state of text without matches) then never falls together with the true walk.  Needs a CUDA device.
"""
import sys
import os
import time

sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import torch  # noqa: E402
import pire_b200 as P  # noqa: E402
from pire_b200 import _native as N, workloads as W  # noqa: E402


MIB = 2 ** 20


def main():
    if not torch.cuda.is_available():
        sys.exit("string_stitch_probe needs a CUDA device")
    dev = torch.empty(256 * MIB, dtype=torch.uint8, device="cuda:0")
    out = torch.zeros(3, dtype=torch.int32, device="cuda:0")

    def run(sc, n, tag):
        o = out.data_ptr()
        t = time.time()
        N.check(N.lib.pire_gpu_run_string(sc._h, dev.data_ptr(), n, N.RUN_BEGIN | N.RUN_END, None, o, o + 4, o + 8,
                                          torch.cuda.current_stream().cuda_stream), "pire_gpu_run_string")
        torch.cuda.synchronize()
        print(tag, n // MIB, "MiB", round((time.time() - t) * 1e3, 2), "ms", out.cpu().tolist(), flush=True)

    for planted in (True, False):
        W.SynthSpec(256 * 1024, 1024, plants=(W.GLUE10_PLANTS + W.HEADLINE_PLANTS) if planted else ()).fill_device(dev)
        for name in ("headline", "glue10"):
            for tuned in (False, True):
                sc = P.Scanner(W.load_image(name), 0)
                if tuned:
                    sc.Tune(P.Batch(dev, fixed_len=4096))
                for n in (1 * MIB, 4 * MIB, 16 * MIB):
                    run(sc, n, "planted=%d %s tuned=%d" % (planted, name, tuned))


if __name__ == "__main__":
    main()
