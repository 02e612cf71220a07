"""The scanner images of tests/golden/count_images.json.xz (written by tests/golden/make_count_images.py), without a GPU:
they load as host-only scanners, the host Scanner concept agrees with the oracle on them, the oracle's counts are the
occurrences of wNNN the patterns describe, and the fixture still has an image on each side of kCountRowsMax, the
number of regexps up to which CountStringKernel keeps its counters in shared rows."""
import base64
import json
import lzma
import os
import re

import numpy as np
import pytest

from conftest import HERE, ROOT
from refpire import Oracle, csr, oracle_count

BeginMark, EndMark = 258, 259
LETTERS = b"abcdefghijklmnopqrstuvwxyz"


def load_count_images():
    """name -> {"image": bytes, "states", "letters", "regexps", "ids"}"""
    with open(os.path.join(HERE, "golden", "count_images.json.xz"), "rb") as f:
        d = json.loads(lzma.decompress(f.read()))["images"]
    out = {}
    for name, e in d.items():
        e = dict(e)
        e["image"] = lzma.decompress(base64.b64decode(e.pop("image_xz")))
        out[name] = e
    return out


COUNT_IMAGES = load_count_images()


def count_rows_max():
    """kCountRowsMax of pire_b200/csrc/scan_kernels.cuh."""
    with open(os.path.join(ROOT, "pire_b200", "csrc", "scan_kernels.cuh")) as f:
        m = re.search(r"constexpr\s+uint32_t\s+kCountRowsMax\s*=\s*(\d+)\s*;", f.read())
    assert m, "kCountRowsMax not found in scan_kernels.cuh"
    return int(m.group(1))


def w_text(rng, length, ids, plant_at=()):
    """Lowercase text of `length` bytes with 'w' + a 3-digit id of `ids` written at each offset of `plant_at`."""
    host = rng.choice(np.frombuffer(LETTERS, np.uint8), size=length)
    for k, at in enumerate(plant_at):
        lit = np.frombuffer(b"w%03d" % ids[k % len(ids)], np.uint8)
        host[at:at + 4] = lit[: max(0, min(4, length - at))]
    return host


def w_strings(rng, k, count, max_len):
    """Strings that end a match of some regexp (its id below k, ids past 255 among them), strings with a wNNN whose id
    has no regexp, strings with a digit before any w, and plain lowercase ones."""
    out = []
    for j in range(count):
        s = bytearray(rng.choice(np.frombuffer(LETTERS, np.uint8), size=int(rng.integers(0, max_len))).tobytes())
        kind = j % 5
        if kind in (0, 1, 2):
            i = (k - 1 - j % 7) if kind == 0 else j % 4 if kind == 1 else int(rng.integers(0, k))
            at = int(rng.integers(0, len(s) + 1))
            s[at:at] = b"w%03d" % i
        elif kind == 3:
            s[len(s) // 2:len(s) // 2] = b"w%03d" % (k + j % 50) if j % 2 else b"7"
        out.append(bytes(s))
    return out


def want_counts(strings, k):
    """What the patterns say: a string's prefix matches [a-z]*wNNN (not surrounded) at most once, where its first
    non-letter is the first digit after a 'w'."""
    counts = np.zeros((len(strings), k), np.uint32)
    for i, s in enumerate(strings):
        m = re.match(rb"[a-z]*w(\d{3})", s)
        if m and int(m.group(1)) < k:
            counts[i, int(m.group(1))] = 1
    return counts


def host_scanner(image):
    from pire_b200 import Scanner
    return Scanner(image, device=-1)


@pytest.mark.parametrize("name", sorted(COUNT_IMAGES))
def test_count_image_loads_and_host_concept_matches_oracle(name):
    e = COUNT_IMAGES[name]
    sc = host_scanner(e["image"])
    info = sc.info()
    assert (info.states, info.letters, info.regexps) == (e["states"], e["letters"], e["regexps"]) and e["regexps"] == e["ids"]
    orc = Oracle(e["image"])
    assert (orc.states, orc.letters, orc.regexps) == (e["states"], e["letters"], e["regexps"])
    k = e["regexps"]
    rng = np.random.default_rng(k)
    strings = w_strings(rng, k, 400, 40) + [b""]
    corpus, offs = csr(strings)
    for begin, end in ((True, True), (False, False), (True, False), (False, True)):
        final, mask, state = orc.run(corpus, offs, begin=begin, end=end, shortcuts=False)
        for j, s in enumerate(strings):
            st = sc.Initialize()
            if begin:
                st = sc.Next(st, BeginMark)
            for b in s:
                st = sc.Next(st, b)
            if end:
                st = sc.Next(st, EndMark)
            assert sc.StateIndex(st) == state[j], (name, begin, end, s)
            assert sc.Final(st) == bool(final[j]), (name, begin, end, s)
            ids = sc.AcceptedRegexps(st)
            assert sum(1 << r for r in ids if r < 32) == mask[j], (name, begin, end, s)
            assert len(ids) == (1 if final[j] else 0), (name, begin, end, s, ids)
    counts, fin = oracle_count(orc, corpus, offs, begin=False, end=False)
    want = want_counts(strings, k)
    assert (counts == want).all(), np.argwhere(counts != want)[:5]
    assert want[:, 256:].any() == (k > 256)                 # ids past 255 are counted where there are any
    ends = [bool(m) and int(m.group(1)) < k for m in (re.fullmatch(rb"[a-z]*w(\d{3})", s) for s in strings)]
    assert fin.astype(bool).tolist() == ends                # Final(): the string ends where its match ends


def test_count_images_straddle_count_rows_max():
    """One image at kCountRowsMax regexps (shared rows) and one just past it (flushes to the u64 counters): if the
    constant moves, the fixture has to be written again or the GPU tests leave the paths they are named after."""
    limit = count_rows_max()
    sizes = sorted(e["regexps"] for e in COUNT_IMAGES.values())
    assert limit in sizes and limit + 1 in sizes, (limit, sizes)
    assert max(sizes) > limit + 32                          # accept sets of more words than the boundary's
    for name, e in COUNT_IMAGES.items():
        sc = host_scanner(e["image"])
        assert sc.info().regexps == e["regexps"]
        assert sc.Size() <= 4096, name                      # the counts stay a table walk, not a state explosion
        for s in range(sc.Size()):
            if sc.Final(s):
                assert len(sc.AcceptedRegexps(s)) == 1, (name, s)
