#!/usr/bin/env python
"""pigrep on the GPU: the reference's samples/pigrep/pigrep.cpp with the per-line loop
(std::getline + Runner(sc).Begin().Run(line).End()) moved to the device.

    python tools/pigrep.py --scanner patterns.pire file [file ...]     # precompiled Scanner::Save() image
    python tools/pigrep.py --scanner a.pire --scanner b.pire file ...  # a pattern set glued into two scanners
    python tools/pigrep.py --scanner slow.pire file [file ...]          # a SlowScanner::Save() image (header type 3)
    python tools/pigrep.py [-i] [-u] -e PATTERN file [file ...]        # compile with the reference front end
                                                                       # (needs oracle/_ref and the reference tree;
                                                                       # developer convenience)
    python tools/pigrep.py --half-final hf.pire --reverse rev.pire -o file [file ...]
    zcat x.gz | python tools/pigrep.py --scanner patterns.pire            # no file, or "-": standard input

Prints matching lines like pigrep (with a "file: " prefix when several files are given, "(stdin): " for "-"); -c
prints counts only, -n puts the line number (from 1) in front, -b the byte offset in the file of the line (or, with -o,
of the match).

--scanner may be given twice, for a pattern set that Scanner::Glue could not put into one scanner: a line is printed
when either scanner accepts it (ScannerPair's Final()), and each frame is scanned once for both
(pire_gpu_run_pair_lines).  -c, -n and -b keep their meaning.

Every input, file or pipe, is read in blocks of --block-mb MiB (default 256) and streamed to the GPU through a
LineStream (pire_gpu_line_stream): frames of whole lines, each scanned as it arrives, so an input of any size works and
the GPU never holds more than three slots of it.  Line numbers and byte offsets are those of the whole input.  The
bytes of a block are kept on the host until every frame that holds them has been printed.

-o prints every match on a line of its own.  Where the matches end comes from a HalfFinalScanner image (--half-final:
pire_gpu_match_ends_lines, every line its own run with BeginMark and EndMark), where they start from the same patterns
compiled with Fsm::Reverse() (--reverse: pire_gpu_match_starts_lines, the leftmost start of each match).  From the
(start, end) pairs of a line, non-empty spans are taken leftmost-longest and without overlap: sorted by start
ascending, then end descending, a span is taken when it starts at or after the end of the span taken before it.  That
is close to what grep -o prints, but it is this selection over Pire's spans, not GNU grep's matcher, and the two can
differ.  With -o, -c counts the lines that have at least one span, and --scanner is not used.  With -e all three
scanners are compiled from the pattern.

Patterns that cannot be determinised (x.{40}$, foo.{64}bar): --scanner reads the image's header type, and a
Pire::SlowScanner image (type 3) runs pire_gpu_slow_run_batch over each frame's lines; -c, -n and -b keep their meaning.
-e compiles the way Pire::Regexp does (easy.h:211-214): when Fsm::Determine() fails, the pattern becomes a SlowScanner
built from the same Fsm (this needs the reference tree, $PIRE_REF, to build tests/golden/slow_ref.cpp; without it -e
compiles a Scanner as before).  Match spans (-o) and pairs of scanners are DFA-only: with a SlowScanner, -o or a second
--scanner exits with a message.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


SLOW_SCANNER = 3          # ScannerIOTypes::SlowScanner, pire/scanners/common.h:38


def image_type(image):
    """The scanner type in an image's stream header (common.h:44-63), or 0 for a buffer too short to hold one."""
    return int.from_bytes(image[16:20], "little") if len(image) >= 24 else 0


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
    ap.add_argument("--scanner", action="append", default=[],
                    help="Scanner::Save() image; give it twice for a pattern set split over two scanners")
    ap.add_argument("--half-final", dest="half_final", help="HalfFinalScanner image of the patterns (-o)")
    ap.add_argument("--reverse", help="Scanner image of the patterns built with Fsm::Reverse() (-o)")
    ap.add_argument("-e", dest="pattern")
    ap.add_argument("-i", action="store_true")
    ap.add_argument("-u", action="store_true")
    ap.add_argument("-c", action="store_true", help="print only the number of matching lines per file")
    ap.add_argument("-o", action="store_true", help="print every match on a line of its own")
    ap.add_argument("-n", action="store_true", help="prefix the line number")
    ap.add_argument("-b", action="store_true", help="prefix the byte offset of the line (with -o: of the match)")
    ap.add_argument("--block-mb", dest="block_mb", type=float, default=256.0,
                    help="bytes read from an input at a time, in MiB (default 256)")
    ap.add_argument("files", nargs="*", help="input files; none, or -, reads standard input")
    args = ap.parse_args()
    import pire_b200 as P
    images, hf_image, rev_image = [], None, None
    if args.pattern:
        sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
        import tempfile
        from make_slow_images import REF, build_helper, compile_slow
        opts = ("i" if args.i else "") + ("u" if args.u else "")
        slow_image, determinable = None, True
        if os.path.isdir(os.path.join(REF, "pire")):
            # Pire::SlowScanner's C face is built against the reference tree; without the tree the pattern is compiled
            # as a Scanner, as before
            with tempfile.TemporaryDirectory() as tmp:
                slow_image, determinable = compile_slow(build_helper(tmp), args.pattern.encode(), opts, max_size=0)
        if not determinable:
            images = [slow_image]
        else:
            from refpire import Ref           # the reference's own Lexer/Fsm/Compile, unchanged host code
            ref = Ref()
            images = [ref.compile(args.pattern.encode(), opts).save()]
            hf_image = ref.compile_half_final(args.pattern.encode(), opts).save()
            rev_image = ref.compile(args.pattern.encode(), opts + "nr").save()
    else:
        images = [open(name, "rb").read() for name in args.scanner]
        hf_image = open(args.half_final, "rb").read() if args.half_final else None
        rev_image = open(args.reverse, "rb").read() if args.reverse else None
    slow = [image_type(image) == SLOW_SCANNER for image in images]
    if any(slow) and args.o:
        ap.error("-o prints match spans, which need DFA images: a SlowScanner (a pattern that cannot be determinised) "
                 "gives matching lines only")
    if any(slow) and len(images) > 1:
        ap.error("a SlowScanner image runs alone: two scanners at once are DFA-only")
    if args.o and not (hf_image and rev_image):
        ap.error("-o needs --half-final FILE and --reverse FILE, or -e PATTERN")
    if not args.o and not images:
        ap.error("give --scanner FILE or -e PATTERN")
    if len(images) > 2:
        ap.error("--scanner may be given at most twice")
    block = max(1, int(args.block_mb * (1 << 20)))
    scanners = [P.SlowScanner(image, 0) if k else P.Scanner(image, 0) for image, k in zip(images, slow)] if not args.o else []
    sc = scanners[0] if len(scanners) == 1 else P.ScannerPair(*scanners) if scanners else None
    hf = P.Scanner(hf_image, 0) if args.o else None
    rev = P.Scanner(rev_image, 0) if args.o else None
    out = sys.stdout.buffer
    # samples/pigrep/pigrep.cpp: no file is stdin without a prefix; "-" is stdin, named "(stdin)" among several
    names = args.files or [None]
    for name in names:
        prefix = ((name if name not in (None, "-") else "(stdin)") + ": ") if len(names) > 1 else ""
        if name in (None, "-"):
            count = grep_stream(P, args, sc, hf, rev, sys.stdin.buffer, block, prefix, out)
        else:
            with open(name, "rb") as f:
                count = grep_stream(P, args, sc, hf, rev, f, block, prefix, out)
        if args.c:
            print("%s%d" % (prefix, count))


def read_block(f, block):
    """Up to `block` bytes of f (fewer only at the end of the input), read straight into a fresh numpy array."""
    import numpy as np
    buf = np.empty(block, dtype=np.uint8)
    view, got = memoryview(buf), 0
    while got < block:
        k = f.readinto(view[got:])
        if not k:
            break
        got += k
    return buf[:got]


class HeldText:
    """The host bytes of the input from the first frame not yet printed on: the blocks read so far, by position."""

    def __init__(self):
        self.blocks = []            # (position of the block's first byte, numpy block)

    def add(self, at, data):
        self.blocks.append((at, data))

    def bytes(self, lo, hi):
        parts = [data[max(lo, at) - at: min(hi, at + len(data)) - at] for at, data in self.blocks
                 if at < hi and at + len(data) > lo]
        return b"".join(p.tobytes() for p in parts)

    def drop_before(self, pos):
        self.blocks = [(at, data) for at, data in self.blocks if at + len(data) > pos]


def grep_stream(P, args, sc, hf, rev, f, block, prefix, out):
    """Greps one input; prints the matches and returns the -c count.  `sc` is a Scanner, a SlowScanner or a
    ScannerPair."""
    import numpy as np
    ls = P.LineStream(0)
    held = HeldText()
    count, at = 0, 0

    def head(line, pos):
        return (prefix + ("%d:" % (line + 1) if args.n else "") + ("%d:" % pos if args.b else "")).encode()

    last = False
    while not last:
        data = read_block(f, block)
        last = len(data) < block
        held.add(at, data)
        at += len(data)
        for frame in ls.feed(data, last=last):
            line0, byte0 = frame.first_line, frame.first_byte
            if args.o:
                spans = line_spans(P, hf, rev, frame)
                count += len(spans)
                if args.c:
                    continue
                for line in sorted(spans):
                    for s, e in spans[line]:
                        out.write(head(line0 + line, byte0 + s) + held.bytes(byte0 + s, byte0 + e) + b"\n")
            else:
                if isinstance(sc, P.ScannerPair):
                    hit = P.Runner(sc).Begin().RunLines(frame).End().Matches()
                else:
                    hit = P.Runner(sc).Begin().Run(frame).End().Matches()
                count += int(hit.sum())
                if args.c:
                    continue
                offs = frame.offsets.cpu().numpy()
                for i in np.nonzero(hit)[0]:
                    lo, hi = byte0 + int(offs[i]), byte0 + int(offs[i + 1]) - 1
                    out.write(head(line0 + int(i), lo) + held.bytes(lo, hi) + b"\n")
            held.drop_before(byte0 + frame.n_bytes)
    out.flush()
    return count

if __name__ == "__main__":
    main()
