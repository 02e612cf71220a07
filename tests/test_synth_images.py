"""The synthesized automata of tests/synth_dfa.py are images Pire itself accepts and reads as intended, so that a GPU
disagreement in test_gpu_synth.py is a kernel bug and not a flaw in the fixtures:

* every family's image is byte-identical across two generations;
* the image loads as a host-only handle whose Scanner concept (info, Next, Final, StateIndex, AcceptedRegexps, the
  cell width) equals the generator's tables;
* the C oracle (oracle/pire_oracle.c) over the image equals the walker for run -- plain, and with the exit-mask
  shortcuts, which checks the masks -- and for prefix, suffix and HalfFinalScanner counts;
* the reference itself, when oracle/_ref is built, loads the image and agrees on run (Scanner, ExitMasks), prefix,
  suffix and, loaded as a HalfFinalScanner, counts."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import refpire  # noqa: E402
import synth_dfa as SD  # noqa: E402

FAMILIES = sorted(SD.FAMILIES)
BIG = {"width_65536", "width_65537"}


def sample_strings(seed, n=120, max_len=70):
    """Random strings of every length up to max_len, some a multiple of 16 (the shortcut's word) and some empty."""
    rng = np.random.default_rng(seed)
    lens = list(rng.integers(0, max_len, n)) + [0, 16, 32, 48, 64, 17, 15]
    return [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in lens]


def test_families_are_deterministic():
    for name in FAMILIES:
        assert SD.FAMILIES[name]().image() == SD.family(name).image(), name


@pytest.mark.parametrize("name", FAMILIES)
def test_host_handle_reads_the_tables(name):
    import pire_b200 as P
    d = SD.family(name)
    sc = P.Scanner(d.image(), -1)
    info = sc.info()
    assert (info.states, info.letters, info.regexps, info.initial, info.empty) == (d.states, d.letters, d.regexps, d.initial, 0)
    assert info.table_bytes == d.states * d.letters * (4 if d.states > 65536 else 2)
    rng = np.random.default_rng(7)
    states = range(d.states) if d.states <= 400 else rng.integers(0, d.states, 400).tolist() + [d.states - 1]
    chars = list(range(256)) + [SD.BEGIN_MARK, SD.END_MARK]
    for s in states:
        row = [sc.Next(s, c) for c in chars]
        want = [d.step(s, c) for c in chars]
        assert row == want, (name, s)
        assert sc.Final(s) == bool(d.final[s]) and sc.Dead(s) == bool(d.dead[s]), (name, s)
        assert sc.AcceptedRegexps(s) == d.accept[s], (name, s)
        assert sc.StateIndex(s) == s


@pytest.mark.parametrize("name", FAMILIES)
def test_oracle_equals_walker(name):
    d = SD.family(name)
    orc = refpire.Oracle(d.image())
    strings = sample_strings(hash(name) % 1000, n=40 if name in BIG else 120)
    corpus, offs = refpire.csr(strings)
    for begin in (False, True):
        for end in (False, True):
            want = d.run(strings, begin=begin, end=end)
            for shortcuts in (False, True):
                got = orc.run(corpus, offs, begin=begin, end=end, shortcuts=shortcuts)
                for g, w, what in zip(got, want, ("final", "mask", "state")):
                    np.testing.assert_array_equal(g, w, err_msg="%s run %s begin=%d end=%d shortcuts=%d" % (
                        name, what, begin, end, shortcuts))
            counts, fin = refpire.oracle_count(orc, corpus, offs, begin=begin, end=end)
            wc, wf, _ = d.count(strings, begin=begin, end=end)
            np.testing.assert_array_equal(counts, wc, err_msg="%s counts" % name)
            np.testing.assert_array_equal(fin, wf, err_msg="%s count final" % name)
            for shortest in (False, True):
                np.testing.assert_array_equal(
                    refpire.oracle_prefix(orc, corpus, offs, shortest=shortest, through_begin=begin, through_end=end),
                    d.prefix(strings, shortest, begin, end), err_msg="%s prefix shortest=%d" % (name, shortest))
                np.testing.assert_array_equal(
                    refpire.oracle_suffix(orc, corpus, offs, shortest=shortest, through_end=end, through_begin=begin),
                    d.suffix(strings, shortest, end, begin), err_msg="%s suffix shortest=%d" % (name, shortest))


def _ref():
    if not refpire.have_ref():
        pytest.skip("oracle/_ref not built (make ref)")
    return refpire.Ref()


@pytest.mark.parametrize("name", FAMILIES)
def test_reference_counts_equal_walker(name):
    """The reference loads the image as a HalfFinalScanner (the same format): its counts, and the Final() of the state
    each run ends in, equal the walker's."""
    ref = _ref()
    d = SD.family(name)
    image = d.image()
    hf = ref.load_half_final(image)
    assert (hf.size, hf.regexps) == (d.states, d.regexps)
    assert hf.save() == image                                   # Save() of the loaded scanner writes the same bytes
    strings = sample_strings(hash(name) % 1000 + 1, n=40 if name in BIG else 120)
    corpus, offs = refpire.csr(strings)
    for begin in (False, True):
        for end in (False, True):
            counts, fin = hf.count(corpus, offs, begin=begin, end=end)
            wc, wf, _ = d.count(strings, begin=begin, end=end)
            np.testing.assert_array_equal(counts, wc, err_msg="%s reference counts begin=%d end=%d" % (name, begin, end))
            np.testing.assert_array_equal(fin, wf, err_msg="%s reference count final begin=%d end=%d" % (name, begin, end))
            np.testing.assert_array_equal(fin, d.run(strings, begin=begin, end=end)[0], err_msg="%s run final" % name)


@pytest.mark.parametrize("name", FAMILIES)
def test_reference_equals_walker(name):
    """The reference loads the image as a Pire::Scanner and agrees on run (ExitMasks shortcuts), prefix and suffix."""
    ref = _ref()
    if not ref.can_load:
        pytest.skip("oracle/_ref was built from an oracle/ref_capi.cpp without pref_load (rebuild with make ref)")
    d = SD.family(name)
    image = d.image()
    sc = ref.load(image)
    assert (sc.size, sc.letters, sc.regexps, sc.initial) == (d.states, d.letters, d.regexps, d.initial)
    assert sc.save() == image
    strings = sample_strings(hash(name) % 1000 + 1, n=40 if name in BIG else 120)
    corpus, offs = refpire.csr(strings)
    for begin in (False, True):
        for end in (False, True):
            got = sc.run(corpus, offs, begin=begin, end=end, variant=0)
            for g, w, what in zip(got, d.run(strings, begin=begin, end=end), ("final", "mask", "state")):
                np.testing.assert_array_equal(g, w, err_msg="%s reference run %s begin=%d end=%d" % (name, what, begin, end))
            for shortest in (False, True):
                np.testing.assert_array_equal(sc.prefix(corpus, offs, shortest=shortest, through_begin=begin, through_end=end,
                                                        variant=0),
                                              d.prefix(strings, shortest, begin, end),
                                              err_msg="%s reference prefix shortest=%d" % (name, shortest))
                np.testing.assert_array_equal(sc.suffix(corpus, offs, shortest=shortest, through_end=end, through_begin=begin,
                                                        variant=0),
                                              d.suffix(strings, shortest, end, begin),
                                              err_msg="%s reference suffix shortest=%d" % (name, shortest))
