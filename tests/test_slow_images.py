"""SlowScanner images on the host, no GPU: host-only handles (device -1) ingest every fixture and synthesized image, the
host concept (pire_gpu_slow_initial / next / final) equals the reference and the numpy oracle, and every malformed
image is refused."""
import ctypes as C
import struct

import numpy as np
import pytest

import pire_b200 as P
from pire_b200 import _native as N
from slow_fixtures import SLOW
import synth_nfa as SN

EIMAGE, EUNSUPPORTED, ENODEVICE = -2, -5, -4
BEGIN_MARK, END_MARK = 258, 259


def create(image, device=-1):
    h = C.c_void_p()
    buf = (C.c_char * max(1, len(image))).from_buffer_copy(image or b"\0")
    rc = N.lib.pire_gpu_slow_scanner_create(buf, len(image), device, C.byref(h))
    if rc == 0:
        N.lib.pire_gpu_slow_scanner_destroy(h)
    return rc


def keep_mask(states):
    """Words of a set with the bits at or past `states` cleared."""
    words = (states + 31) // 32
    m = np.full(words, 0xFFFFFFFF, np.uint32)
    if states % 32:
        m[-1] = (1 << (states % 32)) - 1
    return m


def walk(sc, data, start, begin, end):
    """Runner(sc[, st]) [.Begin()] .Run(data) [.End()] on the host concept; a start set's bits past Size() dropped."""
    cur = sc.Initialize() if start is None else np.asarray(start, np.uint32) & keep_mask(sc.Size())
    if begin:
        cur = sc.Next(cur, BEGIN_MARK)
    for b in data:
        cur = sc.Next(cur, b)
    if end:
        cur = sc.Next(cur, END_MARK)
    return sc.Final(cur), cur


@pytest.mark.parametrize("e", SLOW, ids=lambda e: e.name)
def test_fixture_ingest(e):
    sc = P.SlowScanner(e.image, -1)
    assert (sc.Size(), sc.LettersCount(), sc.Empty(), sc.RegexpsCount()) == (e.states, e.letters, e.empty, 0 if e.empty else 1)
    info = sc.info()
    assert info.set_words == e.words and info.device == -1 and info.table_bytes > 0


@pytest.mark.parametrize("e", SLOW, ids=lambda e: e.name)
def test_fixture_host_concept_equals_reference(e):
    sc = P.SlowScanner(e.image, -1)
    for key in ((True, True, False), (False, False, True), (True, False, True)):
        final, sets = e.runs[key]
        for i, s in enumerate(e.strings):
            f, cur = walk(sc, s, e.start_sets[i] if key[2] else None, key[0], key[1])
            assert f == final[i] and (cur == sets[i]).all(), (key, i)


def test_slow_ut_vectors():
    e = next(x for x in SLOW if x.name == "slow_ut")
    sc = P.SlowScanner(e.image, -1)
    assert [walk(sc, s, None, True, True)[0] for s in e.strings] == [True, False, False]     # pire_ut.cpp:707-713


def test_golden_cases_agree_with_dfa_bits():
    from conftest import GOLDEN
    by_name = {e.name: e for e in SLOW}
    checked = 0
    for c in GOLDEN:
        e = by_name.get("golden/" + c.name)
        if e is None:
            continue
        final, _ = e.runs[(c.begin, c.end, False)]
        assert final.astype(int).tolist() == c.final, c.name
        checked += 1
    assert checked >= 40


@pytest.mark.parametrize("fam", [f[0] for f in SN.FAMILIES])
def test_synth_host_concept_equals_oracle(fam):
    nfa = SN.family(fam)
    sc = P.SlowScanner(nfa.image(), -1)
    assert sc.Size() == nfa.states and sc.LettersCount() == nfa.letters and not sc.Empty()
    rng = np.random.default_rng(len(fam))
    for k in range(6 if nfa.states < 1000 else 2):
        data = rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8).tobytes()
        start = None
        if k % 2:
            start = rng.integers(0, 1 << 32, nfa.words, dtype=np.uint64).astype(np.uint32)
        begin, end = bool(k & 2), bool(k & 1)
        want_f, want_set = nfa.run(data, None if start is None else nfa.unpack(start), begin, end)
        got_f, got_set = walk(sc, data, start, begin, end)
        assert got_f == want_f and (got_set == want_set).all(), k


def test_4097_states_unsupported():
    nfa = SN.random_nfa(14, 4097, 2, 1.0)
    assert create(nfa.image()) == EUNSUPPORTED
    assert b"4097" in N.lib.pire_gpu_last_error()
    assert create(SN.random_nfa(13, 4096, 2, 1.0).image()) == 0


def test_empty_image_is_null():
    nfa = SN.random_nfa(1, 5, 2)
    sc = P.SlowScanner(nfa.image(empty=True), -1)
    assert sc.Empty() and sc.Size() == 1 and sc.RegexpsCount() == 0 and sc.LettersCount() == 1
    cur = sc.Initialize()
    assert not sc.Final(cur) and not sc.Final(sc.Next(cur, ord("a")))


def _small():
    return SN.SynthNfa(3, 2, 1, [0] * 264, [False, True, False],
                       [[[1], [0, 2]], [[], [2, 2]], [[0], [1]]])


def _layout(image, S, L):
    """Byte offsets of the sections of a SlowScanner image: locals, empty, letters, finals, jumpPos, jumps, end."""
    pad = lambda v: (v + 7) // 8 * 8
    loc, emp = 24, 48
    let = 56
    fin = let + 264 * 8
    pos = fin + pad(S)
    jmp = pos + (S * L + 1) * 8
    total = struct.unpack_from("<Q", image, jmp - 8)[0]
    return {"locals": loc, "empty": emp, "letters": let, "finals": fin, "pos": pos, "jumps": jmp, "end": jmp + pad(4 * total)}


def _poke(image, off, fmt, value):
    b = bytearray(image)
    struct.pack_into(fmt, b, off, value)
    return bytes(b)


def test_malformed_images_refused():
    nfa = _small()
    good = nfa.image()
    assert create(good) == 0
    L = _layout(good, 3, 2)
    assert L["end"] == len(good)
    bad = {
        "magic": _poke(good, 0, "<I", 0x12345678),
        "version": _poke(good, 4, "<I", 5),
        "ptr_size": _poke(good, 8, "<I", 4),
        "word_size": _poke(good, 12, "<I", 8),
        "type_scanner": _poke(good, 16, "<I", 1),
        "hdr_size": _poke(good, 20, "<I", 48),
        "no_states": _poke(good, L["locals"], "<Q", 0),
        "no_letters": _poke(good, L["locals"] + 8, "<Q", 0),
        "start_past": _poke(good, L["locals"] + 16, "<Q", 3),
        "states_huge": _poke(good, L["locals"], "<Q", 1 << 62),
        "letters_huge": _poke(good, L["locals"] + 8, "<Q", (1 << 64) - 1),
        "letter_past": _poke(good, L["letters"] + 8 * ord("x"), "<Q", 2),
        "begin_letter_past": _poke(good, L["letters"] + 8 * BEGIN_MARK, "<Q", 7),
        "jump_past": _poke(good, L["jumps"], "<I", 3),
        "pos_first": _poke(good, L["pos"], "<Q", 1),
        "pos_back": _poke(good, L["pos"] + 16, "<Q", 0),
        "pos_past": _poke(good, L["pos"] + 6 * 8, "<Q", 1 << 40),
    }
    # 7 jumps: the last section is 28 bytes and 4 bytes of padding, which Load reads too (L["end"] - 4 cuts inside it)
    for cut in (0, 10, 30, L["empty"] + 4, L["letters"] + 100, L["finals"] + 1, L["finals"] + 4, L["pos"] + 20,
                L["jumps"] + 4, L["end"] - 4, L["end"] - 1):
        bad["cut_%d" % cut] = good[:cut]
    for name, image in bad.items():
        assert create(image) == EIMAGE, name
    # Epsilon's letter is never stepped: any value is accepted, as Load accepts it
    assert create(_poke(good, L["letters"] + 8 * 257, "<Q", 99)) == 0


def test_null_and_bad_arguments():
    assert N.lib.pire_gpu_slow_scanner_create(None, 0, -1, C.byref(C.c_void_p())) == EIMAGE
    assert N.lib.pire_gpu_slow_scanner_create(None, 0, -1, None) == -1


def test_dfa_create_refuses_slow_image():
    image = SLOW[0].image
    h = C.c_void_p()
    buf = (C.c_char * len(image)).from_buffer_copy(image)
    assert N.lib.pire_gpu_scanner_create(buf, len(image), -1, C.byref(h)) == EIMAGE
    assert N.lib.pire_gpu_last_error() == b"Serialized regexp incompatible with your system"


def test_host_only_run_is_enodevice():
    sc = P.SlowScanner(SLOW[0].image, -1)
    assert N.lib.pire_gpu_slow_run_batch(sc._h, None, None, 0, 1, 0, None, None, None, None) == ENODEVICE
    with pytest.raises(ValueError):
        sc.Next(np.zeros(sc.set_words + 1, np.uint32), 0)
    assert N.lib.pire_gpu_slow_next(sc._h, sc.Initialize().ctypes.data, 260, np.zeros(8, np.uint32).ctypes.data) == -1
