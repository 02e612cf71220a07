"""The scanner images of tests/golden/edge_images.json.xz (written by tests/golden/make_edge_images.py), without a GPU:
they load as host-only scanners, the host Scanner concept agrees with the oracle on them, and each still has the
property that puts tests/test_gpu_edges.py on its kernel path."""
import base64
import json
import lzma
import os

import numpy as np
import pytest

from conftest import HERE
from refpire import Oracle, csr

BeginMark, EndMark = 258, 259
MAX_HOT = 255                       # pire_b200/csrc/dfa_tables.hpp kMaxHot


def load_edge_images():
    """name -> {"image": bytes, "states", "letters", "regexps", "patterns"}"""
    with open(os.path.join(HERE, "golden", "edge_images.json.xz"), "rb") as f:
        d = json.loads(lzma.decompress(f.read()))["images"]
    out = {}
    for name, e in d.items():
        e = dict(e)
        e["image"] = lzma.decompress(base64.b64decode(e.pop("image_xz")))
        e["patterns"] = [(p.encode("latin-1"), o) for p, o in e["patterns"]]
        out[name] = e
    return out


EDGE = load_edge_images()

# bytes the strings of each image are drawn from: the letters its patterns are made of, plus a few others
ALPHABETS = {
    "wide": b"ab" * 40 + b"c",
    "anchored": b"abcde x",
    "glued": b"GET error x0123456789y",
    "all_final": b"abc \x00\xff",
    "none_hot": b"abcd" * 20 + b"e",
    "absorbing": b"fo x",
}


def host_scanner(image):
    from pire_b200 import Scanner
    return Scanner(image, device=-1)


def static_hot_order(sc, limit):
    """pire_b200/csrc/dfa_tables.cpp StaticHotOrder, its first `limit` entries, through the host Scanner concept."""
    order, seen = [], set()

    def push(s):
        if s not in seen:
            seen.add(s)
            order.append(s)
    push(sc.Next(sc.Initialize(), BeginMark))
    push(sc.Initialize())
    head = 0
    while head < len(order) and len(order) < limit:
        for b in range(256):
            push(sc.Next(order[head], b))
        head += 1
    return order[:limit]


def random_strings(rng, alphabet, count, max_len):
    a = np.frombuffer(alphabet, np.uint8)
    return [bytes(rng.choice(a, size=int(k))) for k in rng.integers(0, max_len, size=count)]


@pytest.mark.parametrize("name", sorted(EDGE))
def test_edge_image_loads_and_host_concept_matches_oracle(name):
    e = EDGE[name]
    sc = host_scanner(e["image"])
    info = sc.info()
    assert (info.states, info.letters, info.regexps) == (e["states"], e["letters"], e["regexps"])
    assert not sc.Empty()
    orc = Oracle(e["image"])
    assert (orc.states, orc.letters, orc.regexps) == (e["states"], e["letters"], e["regexps"])
    rng = np.random.default_rng(sum(name.encode()))
    strings = random_strings(rng, ALPHABETS[name], 300, 80) + [b""]
    corpus, offs = csr(strings)
    for begin, end in ((True, True), (False, False), (True, False), (False, True)):
        final, mask, state = orc.run(corpus, offs, begin=begin, end=end, shortcuts=False)
        for k, s in enumerate(strings):
            st = sc.Initialize()
            if begin:
                st = sc.Next(st, BeginMark)
            for b in s:
                st = sc.Next(st, b)
            if end:
                st = sc.Next(st, EndMark)
            assert sc.StateIndex(st) == state[k], (name, begin, end, s)
            assert sc.Final(st) == bool(final[k]), (name, begin, end, s)
            assert sum(1 << r for r in sc.AcceptedRegexps(st) if r < 32) == mask[k], (name, begin, end, s)


def test_edge_image_properties():
    """What make_edge_images.py asserted when it wrote the images."""
    wide = host_scanner(EDGE["wide"]["image"])
    assert wide.Size() > 65536
    assert wide.info().table_bytes == wide.Size() * wide.LettersCount() * 4          # 32-bit cells
    for name in ("anchored", "glued"):
        sc = host_scanner(EDGE[name]["image"])
        assert sc.Next(sc.Initialize(), BeginMark) != sc.Initialize(), name
    sc = host_scanner(EDGE["all_final"]["image"])
    todo, seen = [sc.Initialize()], {sc.Initialize()}
    while todo:
        s = todo.pop()
        for c in list(range(256)) + [BeginMark, EndMark]:
            t = sc.Next(s, c)
            if t not in seen:
                seen.add(t)
                todo.append(t)
    assert all(sc.Final(s) for s in seen)
    sc = host_scanner(EDGE["none_hot"]["image"])
    assert sc.Size() > MAX_HOT and not any(sc.Final(s) for s in static_hot_order(sc, MAX_HOT))
    sc = host_scanner(EDGE["absorbing"]["image"])
    absorbing = [s for s in range(sc.Size()) if sc.Final(s) and all(sc.Next(s, b) == s for b in range(256))]
    assert absorbing
    # the images narrower than 65 536 states keep 16-bit cells
    for name in ("anchored", "glued", "none_hot"):
        sc = host_scanner(EDGE[name]["image"])
        assert sc.info().table_bytes == sc.Size() * sc.LettersCount() * 2, name
