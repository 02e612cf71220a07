"""One string over the grid (pire_gpu_run_string), the parts that need no GPU: a host-only handle is refused, the
fixtures of tests/golden/string_images.json.xz still have the property each stands for, and the oracle's run from a
given state (tests/string_oracle.py) agrees with the host Scanner concept on the golden vectors."""
import base64
import json
import lzma
import os

import numpy as np
import pytest

from conftest import GOLDEN, HERE
from refpire import Oracle
from string_oracle import run_from

BEGIN_MARK, END_MARK = 258, 259


def load_string_images():
    """name -> {"image": bytes, "states", "letters", "regexps", "patterns"}"""
    with open(os.path.join(HERE, "golden", "string_images.json.xz"), "rb") as f:
        d = json.loads(lzma.decompress(f.read()))["images"]
    return {name: dict(e, image=lzma.decompress(base64.b64decode(e["image_xz"]))) for name, e in d.items()}


STRING_IMAGES = load_string_images()


def host_scanner(image):
    from pire_b200 import Scanner
    return Scanner(image, device=-1)


def walk(sc, st, text):
    for b in text:
        st = sc.Next(st, b)
    return st


def test_host_only_handle_is_refused():
    import pire_b200 as P
    from pire_b200 import _native as N
    sc = host_scanner(STRING_IMAGES["parity"]["image"])
    assert N.lib.pire_gpu_run_string(sc._h, None, 0, N.RUN_BEGIN, None, None, None, None, None) == -4       # ENODEVICE
    with pytest.raises(P.PireGpuError) as ex:
        P.StringRunner(sc).Begin().End().State()
    assert ex.value.code == -4
    with pytest.raises(P.PireGpuError) as ex:
        P.StringRunner(sc, state=1).State()
    assert ex.value.code == -4


def test_string_image_properties():
    """What make_string_images.py asserted when it wrote the images, on host-only scanners."""
    par = host_scanner(STRING_IMAGES["parity"]["image"])
    assert par.Size() == STRING_IMAGES["parity"]["states"]
    even = par.Next(par.Initialize(), BEGIN_MARK)
    odd = par.Next(even, ord("a"))
    for _ in range(2 * par.Size() + 2):                      # no run of a's brings the two walks together
        assert even != odd
        even, odd = par.Next(even, ord("a")), par.Next(odd, ord("a"))

    sh = host_scanner(STRING_IMAGES["shift11"]["image"])
    todo, states = [sh.Initialize()], {sh.Initialize()}
    while todo:
        s = todo.pop()
        for c in b"ab":
            t = sh.Next(s, c)
            if t not in states:
                states.add(t)
                todo.append(t)
    assert len(states) >= 2048
    rng = np.random.default_rng(11)
    for _ in range(8):                                       # eleven bytes bring every state to one
        text = bytes(rng.choice(np.frombuffer(b"ab", np.uint8), size=11))
        assert len({walk(sh, s, text) for s in states}) == 1
    s = sh.Initialize()                                      # ten do not
    assert walk(sh, sh.Next(s, ord("a")), b"b" * 10) != walk(sh, s, b"b" * 10)


@pytest.mark.parametrize("case", GOLDEN, ids=lambda c: c.name)
def test_oracle_run_from_state_matches_host_concept(case):
    """string_oracle.run_from against the host Scanner concept (pire_gpu_next & co.), from every state (at most 64,
    spread over the scanner) and with every mark pair."""
    orc = Oracle(case.image)
    sc = host_scanner(case.image)
    size = sc.Size()
    starts = sorted(set(range(0, size, max(1, size // 64))) | {sc.Initialize()})
    for text in case.strings[:8]:
        for st in starts:
            for begin in (False, True):
                for end in (False, True):
                    s = sc.Next(st, BEGIN_MARK) if begin else st
                    s = walk(sc, s, text)
                    if end:
                        s = sc.Next(s, END_MARK)
                    mask = sum(1 << r for r in sc.AcceptedRegexps(s) if r < 32)
                    assert run_from(orc, np.frombuffer(text, np.uint8), st, begin, end) == (int(sc.Final(s)), mask, s)
    assert run_from(orc, np.zeros(4, np.uint8), size) == (0, 0, 0xFFFFFFFF)
