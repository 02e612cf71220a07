#!/usr/bin/env python
"""Writes tests/golden/edge_images.json.xz: scanner images, compiled by the reference, that put the device kernels on
the paths the default shapes never reach (tests/test_gpu_edges.py, tests/test_edge_images.py).

    wide       (a|b)*a(a|b){16}, not surrounded: more than 65 536 states, so the complete transition table has 32-bit
               cells (ScanTables::wide)
    anchored   ^(ab|cd)+e$: Next(Initialize(), BeginMark) != Initialize(), a string run without Begin() starts in a
               state that is not the first hot row
    glued      ^GET |error|x[0-9]+y glued: the same for a glued scanner
    all_final  .* surrounded: every state reachable by bytes and marks is final (first_final_hot == 0)
    none_hot   (ab|cd){140}, not surrounded: more states than hot rows, and none of the first 255 rows of the static
               hot order is final (first_final_hot == hot rows)
    absorbing  foo surrounded: an accepting state no byte leaves (the NoExit early stop)

Each entry holds the Scanner::Save() image (xz, base64) and its state, letter and regexp counts.  The generator
asserts every property it promises.  It needs oracle/_ref (oracle/build_ref.sh) and is deterministic: a second run
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

OUT = os.path.join(HERE, "edge_images.json.xz")
BEGIN_MARK, END_MARK = 258, 259
MAX_HOT = 255                       # pire_b200/csrc/dfa_tables.hpp kMaxHot

PATTERNS = [
    ("wide", [(rb"(a|b)*a(a|b){16}", "n")]),
    ("anchored", [(rb"^(ab|cd)+e$", "")]),
    ("glued", [(rb"^GET ", ""), (rb"error", ""), (rb"x[0-9]+y", "")]),
    ("all_final", [(rb".*", "")]),
    ("none_hot", [(rb"(ab|cd){140}", "n")]),
    ("absorbing", [(rb"foo", "")]),
]


def static_hot_order(sc, limit):
    """pire_b200/csrc/dfa_tables.cpp StaticHotOrder, its first `limit` entries."""
    order, seen = [], set()

    def push(s):
        if s not in seen:
            seen.add(s)
            order.append(s)
    push(sc.next(sc.initial, BEGIN_MARK))
    push(sc.initial)
    head = 0
    while head < len(order) and len(order) < limit:
        for b in range(256):
            push(sc.next(order[head], b))
        head += 1
    return order[:limit]


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


def check(name, sc):
    init = sc.initial
    if name == "wide":
        assert 65536 < sc.size <= 200000, sc.size
    if name in ("anchored", "glued"):
        assert sc.next(init, BEGIN_MARK) != init
    if name == "all_final":
        assert all(sc.final(s) for s in reachable(sc))
    if name == "none_hot":
        assert sc.size > MAX_HOT
        assert not any(sc.final(s) for s in static_hot_order(sc, MAX_HOT))
    if name == "absorbing":
        assert any(sc.final(s) and all(sc.next(s, b) == s for b in range(256)) for s in reachable(sc))


def main():
    ref = Ref()
    entries = {}
    for name, pats in PATTERNS:
        sc = ref.glue_all(pats)
        assert not sc.empty
        check(name, sc)
        image = sc.save()
        entries[name] = {
            "patterns": [[p.decode("latin-1"), o] for p, o in pats],
            "states": int(sc.size), "letters": int(sc.letters), "regexps": int(sc.regexps),
            "image_xz": base64.b64encode(lzma.compress(image, preset=9 | lzma.PRESET_EXTREME)).decode(),
        }
        print("%-10s %7d states x %3d letters, %d regexps, image %d bytes" % (name, sc.size, sc.letters, sc.regexps, len(image)))
    blob = json.dumps({"images": entries}, sort_keys=True, indent=1).encode()
    with open(OUT, "wb") as f:
        f.write(lzma.compress(blob, preset=9 | lzma.PRESET_EXTREME))
    print("%s: %d bytes" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
