#!/usr/bin/env python
"""Writes tests/golden/count_images.json.xz: glued scanners of many regexps, compiled by the reference, that put the
counting kernels on the paths sized by the number of regexps (tests/test_gpu_count_edges.py, tests/test_count_images.py).

    w256   [a-z]*w000 .. [a-z]*w255, not surrounded: 256 regexps, the most whose per-warp rows of counters still fit
           CountStringKernel's shared memory (kCountRowsMax)
    w257   [a-z]*w000 .. [a-z]*w256: the fewest that flush straight to the caller's u64 counters
    w300   [a-z]*w000 .. [a-z]*w299: well past the boundary, and accept sets of 10 words

A final state is reached by lowercase text ending in wNNN and lists exactly regexp NNN, so a text's counts are the
number of times each wNNN occurs in it.  Each entry holds the Scanner::Save() image (xz, base64) and its state,
letter and regexp counts.  The generator asserts every property it promises.  It needs oracle/_ref
(oracle/build_ref.sh) and is deterministic: a second run writes a byte-identical file.
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

OUT = os.path.join(HERE, "count_images.json.xz")
BEGIN_MARK, END_MARK = 258, 259
SIZES = {"w256": 256, "w257": 257, "w300": 300}
MAX_STATES = 4096


def patterns(k):
    return [(("[a-z]*w%03d" % i).encode(), "n") for i in range(k)]


def reachable(sc):
    todo, seen = [sc.initial], {sc.initial}
    while todo:
        s = todo.pop()
        for c in list(range(256)) + [BEGIN_MARK, END_MARK]:
            t = sc.next(s, c)
            if t not in seen:
                seen.add(t)
                todo.append(t)
    return seen


def walk(sc, text):
    s = sc.initial
    for b in text:
        s = sc.next(s, b)
    return s


def check(sc, k):
    assert sc.regexps == k, (sc.regexps, k)
    assert sc.size <= MAX_STATES, sc.size
    listed = []
    for s in reachable(sc):
        if sc.final(s):
            ids = sc.accepted(s)
            assert len(ids) == 1, (s, ids)
            listed += ids
    assert sorted(set(listed)) == list(range(k))           # every regexp has a final state of its own
    for i in (0, k // 2, k - 1):
        s = walk(sc, b"xyzw%03d" % i)
        assert sc.final(s) and sc.accepted(s) == [i], (i, sc.accepted(s))
    assert not sc.final(walk(sc, b"w%03d" % k))


def main():
    ref = Ref()
    entries = {}
    for name, k in sorted(SIZES.items()):
        pats = patterns(k)
        sc = ref.glue_all(pats)
        assert not sc.empty
        check(sc, k)
        image = sc.save()
        entries[name] = {
            "pattern": "[a-z]*w%03d", "options": "n", "ids": k,
            "states": int(sc.size), "letters": int(sc.letters), "regexps": int(sc.regexps),
            "image_xz": base64.b64encode(lzma.compress(image, preset=9 | lzma.PRESET_EXTREME)).decode(),
        }
        print("%-5s %5d states x %3d letters, %d regexps, image %d bytes" % (name, sc.size, sc.letters, sc.regexps, len(image)))
    blob = json.dumps({"images": entries}, sort_keys=True, indent=1).encode()
    with open(OUT, "wb") as f:
        f.write(lzma.compress(blob, preset=9 | lzma.PRESET_EXTREME))
    print("%s: %d bytes" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
