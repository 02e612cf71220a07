#!/usr/bin/env python
"""Writes tests/golden/string_images.json.xz: scanner images, compiled by the reference, that put the stitch of one
string over the grid (pire_gpu_run_string) on its slow paths (tests/test_gpu_string.py, tests/test_string_images.py).

    parity    ^(aa)*$: the state after an even and after an odd number of a's; no run of a's brings the two together,
              so walks of a piece from different states never fall together and the stitch degrades to the serial walk
    shift11   (a|b)*a(a|b){10}: the state is the last eleven bytes, so walks from different states fall together only
              after eleven bytes (and not after ten)

Both are compiled the way tests/test_gpu_parity.py's test_long_strings_split_over_a_warp compiles them (option "n").
Each entry holds the Scanner::Save() image (xz, base64) and its state, letter and regexp counts.  The generator asserts
the property each image stands for.  It needs oracle/_ref (oracle/build_ref.sh) and is deterministic: a second run
writes a byte-identical file.
"""
import base64
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from refpire import Ref  # noqa: E402

OUT = os.path.join(HERE, "string_images.json.xz")
BEGIN_MARK = 258

PATTERNS = [
    ("parity", (rb"^(aa)*$", "n")),
    ("shift11", (rb"(a|b)*a(a|b)(a|b)(a|b)(a|b)(a|b)(a|b)(a|b)(a|b)(a|b)(a|b)", "n")),
]


def walk(sc, st, text):
    for b in text:
        st = sc.next(st, b)
    return st


def reachable(sc, alphabet, start):
    todo, seen = [start], {start}
    while todo:
        s = todo.pop()
        for c in alphabet:
            t = sc.next(s, c)
            if t not in seen:
                seen.add(t)
                todo.append(t)
    return sorted(seen)


def check(name, sc):
    """The property each image stands for; the same check runs on the stored images in tests/test_string_images.py."""
    if name == "parity":
        even = sc.next(sc.initial, BEGIN_MARK)
        odd = sc.next(even, ord("a"))
        a, b = even, odd
        for _ in range(2 * sc.size + 2):          # every pair the walk can reach has come round by then
            assert a != b
            a, b = sc.next(a, ord("a")), sc.next(b, ord("a"))
    if name == "shift11":
        # not surrounded and not anchored: BeginMark leads to a dead state, the walk starts from Initialize()
        states = reachable(sc, b"ab", sc.initial)
        assert len(states) >= 2048
        for k in range(32):                          # eleven bytes bring every state to one, whatever they are
            text = bytes(b"ab"[(k >> j) & 1 if j < 5 else (k * 7 >> (j - 5)) & 1] for j in range(11))
            assert len({walk(sc, s, text) for s in states}) == 1, text
        # ten do not: ten b's behind an "a" end in a match, behind nothing they do not
        s = sc.initial
        assert walk(sc, sc.next(s, ord("a")), b"b" * 10) != walk(sc, s, b"b" * 10)


def main():
    ref = Ref()
    entries = {}
    for name, (pat, opts) in PATTERNS:
        sc = ref.compile(pat, opts)
        assert not sc.empty
        check(name, sc)
        image = sc.save()
        entries[name] = {
            "patterns": [[pat.decode("latin-1"), opts]],
            "states": int(sc.size), "letters": int(sc.letters), "regexps": int(sc.regexps),
            "image_xz": base64.b64encode(lzma.compress(image, preset=9 | lzma.PRESET_EXTREME)).decode(),
        }
        print("%-8s %6d states x %3d letters, %d regexps, image %d bytes" % (name, sc.size, sc.letters, sc.regexps, len(image)))
    blob = json.dumps({"images": entries}, sort_keys=True, indent=1).encode()
    with open(OUT, "wb") as f:
        f.write(lzma.compress(blob, preset=9 | lzma.PRESET_EXTREME))
    print("%s: %d bytes" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
