#!/usr/bin/env python
"""Writes tests/golden/start_images.json.xz: the scanners the match-starts tests run (tests/test_gpu_match_starts.py).

Each pattern set holds
    forward     the regexps as surrounded HalfFinalScanners, glued in order: what match-ends runs
    reversed    the same regexps compiled with Fsm::Reverse() and no Surround() (options "nr"), glued in the same order:
                what match-starts runs
    per_regexp  each regexp's reversed scanner alone: the tests' independent answer for that regexp's starts
The sets:
    glue10      the GLUE10 benchmark patterns
    edges       ^GET , timeout$ and error: matches pinned to the text's start and end
    never       a.*b: a reversed walk that never dies before the text's start
    empty       x*: empty matches (start == end), at every position
    utf8_ci     a UTF-8 pattern ("u") and a case-insensitive one ("i")
    lit40       40 glued literals: regexp ids past 32
    words       [a-z]+: every lowercase byte of a text ends a match (the dense workload of tools/match_starts_bench.py)

The glue10 and words sets are also what smoke() and tools/match_starts_bench.py run (glue10's forward image is
pire_b200/data/hf_glue10's).  Images are Scanner::Save() streams (xz, base64).  The generator asserts that the glued reversed scanner accepts regexp
id r exactly where the per-regexp scanner r is final, on every suffix of sample texts, so that ids agree between the
forward and the reversed images.  It needs oracle/_ref (oracle/build_ref.sh) and is deterministic.
"""
import base64
import json
import lzma
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from refpire import Ref  # noqa: E402

OUT = os.path.join(HERE, "start_images.json.xz")


def glue10():
    import importlib.util
    spec = importlib.util.spec_from_file_location("workloads_data", os.path.join(ROOT, "pire_b200", "workloads.py"))
    src = open(spec.origin).read().replace("from . import _native as N", "N = None")
    ns = {}
    exec(compile(src, spec.origin, "exec"), ns)
    return [(p, o) for p, o in ns["GLUE10"]]


SETS = {
    "glue10": glue10(),
    "edges": [(b"^GET ", ""), (b"timeout$", ""), (b"error", "")],
    "never": [(b"a.*b", "")],
    "empty": [(b"x*", "")],
    "utf8_ci": [("привет".encode("utf-8"), "u"), (b"Error", "i")],
    "lit40": [(("k%02dz" % i).encode(), "") for i in range(40)],
    "words": [(b"[a-z]+", "")],
}


def samples(pats, rng):
    texts = [b"x error", b"GET timeout", b"xx error", b"a.b..ab", b"xxyx"]
    plants = [p.replace(b"^", b"").replace(b"$", b"").replace(b".*", b"q").replace(b"x*", b"xx") for p, _ in pats]
    alphabet = b"abxyzEeGTrorkz0123456789 \t-\xd0\xbf\xd1\x80"
    for _ in range(40):
        t = bytes(rng.choice(alphabet) for _ in range(rng.randrange(0, 40)))
        k = rng.randrange(len(plants))
        at = rng.randrange(len(t) + 1)
        texts.append(t[:at] + plants[k] + t[at:])
    return texts


def check_ids(rev, singles, texts):
    for text in texts:
        for e in range(len(text) + 1):
            for with_end in (0, 1):
                g = rev.initial
                s = [sc.initial for sc in singles]
                if with_end:
                    g = rev.next(g, 259)
                    s = [sc.next(x, 259) for sc, x in zip(singles, s)]
                for k in range(e - 1, -2, -1):
                    got = set(rev.accepted(g)) if rev.final(g) else set()
                    want = {r for r, (sc, x) in enumerate(zip(singles, s)) if sc.final(x)}
                    assert got == want, (text, e, k, got, want)
                    if k < 0:
                        break
                    g = rev.next(g, text[k])
                    s = [sc.next(x, text[k]) for sc, x in zip(singles, s)]


def pack(img):
    return base64.b64encode(lzma.compress(img, preset=9)).decode()


def main():
    ref = Ref()
    rng = random.Random(20261017)
    out = {}
    for name, pats in SETS.items():
        fwd = None
        for pat, opts in pats:
            one = ref.compile_half_final(pat, opts, 0)
            fwd = one if fwd is None else ref.glue_half_final(fwd, one)
        singles = [ref.compile(pat, opts + "nr") for pat, opts in pats]
        rev = ref.glue_all([(pat, opts + "nr") for pat, opts in pats])
        assert rev.regexps == len(pats) and fwd.regexps == len(pats)
        check_ids(rev, singles, samples(pats, rng))
        out[name] = {
            "patterns": [[pat.decode("latin-1"), opts] for pat, opts in pats],
            "forward": pack(fwd.save()),
            "reversed": pack(rev.save()),
            "per_regexp": [pack(sc.save()) for sc in singles],
        }
        print("%s: %d regexps, forward %d states, reversed %d states" % (name, len(pats), fwd.size, rev.size))
    with open(OUT, "wb") as f:
        f.write(lzma.compress(json.dumps(out, sort_keys=True).encode(), preset=9))


if __name__ == "__main__":
    main()
