#!/usr/bin/env python
"""pigrep on the GPU: the reference's samples/pigrep/pigrep.cpp with the per-line loop
(std::getline + Runner(sc).Begin().Run(line).End()) moved to the device.

    python tools/pigrep.py --scanner patterns.pire file [file ...]     # precompiled Scanner::Save() image
    python tools/pigrep.py [-i] [-u] -e PATTERN file [file ...]        # compile with the reference front end
                                                                       # (needs oracle/_ref; developer convenience)
Prints matching lines like pigrep (with a "file: " prefix when several files are given); -c prints counts only.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser(add_help=True)
    ap.add_argument("--scanner")
    ap.add_argument("-e", dest="pattern")
    ap.add_argument("-i", action="store_true")
    ap.add_argument("-u", action="store_true")
    ap.add_argument("-c", action="store_true", help="print only the number of matching lines per file")
    ap.add_argument("files", nargs="+")
    args = ap.parse_args()
    import numpy as np
    import torch
    import pire_b200 as P
    if args.scanner:
        image = open(args.scanner, "rb").read()
    elif args.pattern:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from refpire import Ref           # the reference's own Lexer/Fsm/Compile, unchanged host code
        image = Ref().compile(args.pattern.encode(), ("i" if args.i else "") + ("u" if args.u else "")).save()
    else:
        ap.error("give --scanner FILE or -e PATTERN")
    sc = P.Scanner(image, 0)
    for name in args.files:
        data = np.fromfile(name, dtype=np.uint8)
        text = torch.from_numpy(data).to("cuda:0")
        batch = P.Batch.from_text(text)
        hit = P.Runner(sc).Begin().Run(batch).End().Matches()
        prefix = (name + ": ") if len(args.files) > 1 else ""
        if args.c:
            print("%s%d" % (prefix, int(hit.sum())))
            continue
        offs = batch.offsets.cpu().numpy()
        out = sys.stdout.buffer
        for i in np.nonzero(hit)[0]:
            out.write(prefix.encode() + data[offs[i]: offs[i + 1] - 1].tobytes() + b"\n")


if __name__ == "__main__":
    main()
