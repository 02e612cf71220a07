#!/usr/bin/env python
"""pigrep on the GPU: the reference's samples/pigrep/pigrep.cpp with the per-line loop
(std::getline + Runner(sc).Begin().Run(line).End()) moved to the device.

    python tools/pigrep.py --scanner patterns.pire file [file ...]     # precompiled Scanner::Save() image
    python tools/pigrep.py [-i] [-u] -e PATTERN file [file ...]        # compile with the reference front end
                                                                       # (needs oracle/_ref; developer convenience)
    python tools/pigrep.py --half-final hf.pire --reverse rev.pire -o file [file ...]

Prints matching lines like pigrep (with a "file: " prefix when several files are given); -c prints counts only,
-n puts the line number (from 1) in front, -b the byte offset in the file of the line (or, with -o, of the match).

-o prints every match on a line of its own.  Where the matches end comes from a HalfFinalScanner image (--half-final:
pire_gpu_match_ends_lines, every line its own run with BeginMark and EndMark), where they start from the same patterns
compiled with Fsm::Reverse() (--reverse: pire_gpu_match_starts_lines, the leftmost start of each match).  From the
(start, end) pairs of a line, non-empty spans are taken leftmost-longest and without overlap: sorted by start
ascending, then end descending, a span is taken when it starts at or after the end of the span taken before it.  That
is close to what grep -o prints, but it is this selection over Pire's spans, not GNU grep's matcher, and the two can
differ.  With -o, -c counts the lines that have at least one span.  With -e all three scanners are compiled from the
pattern.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def select_spans(spans):
    """Leftmost-longest non-overlapping spans of one line (see the module docstring)."""
    out, last = [], -1
    for s, e in sorted(set(spans), key=lambda x: (x[0], -x[1])):
        if s >= last:
            out.append((s, e))
            last = e
    return out


def line_spans(P, hf, rev, batch):
    """{line: [(start, end), ...]} of the selected spans, text positions."""
    import numpy as np
    probe = P.LineMatchEnds(hf, 0).Begin().Run(batch).End()
    ends = P.LineMatchEnds(hf, probe.Found()).Begin().Run(batch).End()
    starts = P.MatchStarts(rev, ends, batch, begin=True, end=True).Starts()
    lines, stops = ends.Lines(), ends.Ends()
    ok = (starts != np.uint64(P.NO_START)) & (stops > starts)
    per = {}
    for l, s, e in zip(lines[ok].tolist(), starts[ok].tolist(), stops[ok].tolist()):
        per.setdefault(l, []).append((s, e))
    return {l: select_spans(v) for l, v in per.items()}


def main():
    ap = argparse.ArgumentParser(add_help=True)
    ap.add_argument("--scanner")
    ap.add_argument("--half-final", dest="half_final", help="HalfFinalScanner image of the patterns (-o)")
    ap.add_argument("--reverse", help="Scanner image of the patterns built with Fsm::Reverse() (-o)")
    ap.add_argument("-e", dest="pattern")
    ap.add_argument("-i", action="store_true")
    ap.add_argument("-u", action="store_true")
    ap.add_argument("-c", action="store_true", help="print only the number of matching lines per file")
    ap.add_argument("-o", action="store_true", help="print every match on a line of its own")
    ap.add_argument("-n", action="store_true", help="prefix the line number")
    ap.add_argument("-b", action="store_true", help="prefix the byte offset of the line (with -o: of the match)")
    ap.add_argument("files", nargs="+")
    args = ap.parse_args()
    import numpy as np
    import torch
    import pire_b200 as P
    image = hf_image = rev_image = None
    if args.pattern:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from refpire import Ref           # the reference's own Lexer/Fsm/Compile, unchanged host code
        ref, opts = Ref(), ("i" if args.i else "") + ("u" if args.u else "")
        image = ref.compile(args.pattern.encode(), opts).save()
        hf_image = ref.compile_half_final(args.pattern.encode(), opts).save()
        rev_image = ref.compile(args.pattern.encode(), opts + "nr").save()
    else:
        image = open(args.scanner, "rb").read() if args.scanner else None
        hf_image = open(args.half_final, "rb").read() if args.half_final else None
        rev_image = open(args.reverse, "rb").read() if args.reverse else None
    if args.o and not (hf_image and rev_image):
        ap.error("-o needs --half-final FILE and --reverse FILE, or -e PATTERN")
    if not args.o and not image:
        ap.error("give --scanner FILE or -e PATTERN")
    sc = P.Scanner(image, 0) if image and not args.o else None
    hf = P.Scanner(hf_image, 0) if args.o else None
    rev = P.Scanner(rev_image, 0) if args.o else None
    out = sys.stdout.buffer
    for name in args.files:
        data = np.fromfile(name, dtype=np.uint8)
        text = torch.from_numpy(data).to("cuda:0")
        batch = P.Batch.from_text(text)
        prefix = (name + ": ") if len(args.files) > 1 else ""
        offs = batch.offsets.cpu().numpy()

        def head(line, at):
            return (prefix + ("%d:" % (line + 1) if args.n else "") + ("%d:" % at if args.b else "")).encode()

        if args.o:
            spans = line_spans(P, hf, rev, batch) if batch.n else {}
            if args.c:
                print("%s%d" % (prefix, len(spans)))
                continue
            for line in sorted(spans):
                for s, e in spans[line]:
                    out.write(head(line, s) + data[s:e].tobytes() + b"\n")
            continue
        hit = P.Runner(sc).Begin().Run(batch).End().Matches()
        if args.c:
            print("%s%d" % (prefix, int(hit.sum())))
            continue
        for i in np.nonzero(hit)[0]:
            out.write(head(int(i), int(offs[i])) + data[offs[i]: offs[i + 1] - 1].tobytes() + b"\n")


if __name__ == "__main__":
    main()
