#!/usr/bin/env python
"""Writes tests/golden/slow_images.json.xz: Pire::SlowScanner images compiled by the reference, with the reference's
answers (tests/test_slow_images.py, tests/test_gpu_slow.py).

    slow_ut      a.{30}$ and the three strings of pire_ut.cpp:707-713 (Slow)
    golden/<n>   every single-pattern case of pire_golden.json compiled as a SlowScanner; with the case's marks its
                 Final() equals the DFA's golden bits (asserted here)
    empty        SlowScanner::Null() (pire_ut.cpp:829, BasicTestEmptySaveLoadMmap<SlowScanner>)
    approx1/2    internationalization with distance 1 and 2 (Compile<SlowScanner>(distance), approximate matching)
    heavy/<n>    patterns whose DFA does not fit in 20 000 states (Fsm::Determine fails): a.{30}$, x.{40}$, ... --
                 the NFAs the fallback of Pire::Regexp (easy.h:205-215) exists for

Each entry holds the image (xz, base64), Size(), GetLettersCount(), Empty(), whether Determine(20000) succeeded, and
strings with, for each of the four mark combinations (begin, end), Final() and the State's set after the run (W =
ceil(Size() / 32) words per string) from Initialize(), and from a seeded random start set per string.

It needs oracle/_ref (oracle/build_ref.sh) and the reference tree ($PIRE_REF, default /root/reference): it compiles
tests/golden/slow_ref.cpp, a C face over Pire::SlowScanner, into a temporary directory.  It is deterministic: a second
run writes a byte-identical file.
"""
import base64
import ctypes as C
import json
import lzma
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "slow_images.json.xz")
REF = os.environ.get("PIRE_REF", "/root/reference")
LIB = os.path.join(ROOT, "oracle", "_ref")

HEAVY = [
    ("a30", rb"a.{30}$", "ab.\n"),
    ("x40", rb"x.{40}$", "xy.\n"),
    ("ab20cd20", rb"(a|b).{20}(c|d).{20}$", "abcde"),
    ("d3_50_d3", rb"\d{3}.{50}\d{3}$", "0123x"),
    ("foo64bar", rb"foo.{64}bar", "fobar"),
    ("a100", rb"a.{100}$", "ab"),
    ("error200", rb"^.{0,80}error.{200}$", "erox"),
]


def build_helper(tmp):
    so = os.path.join(tmp, "libslowref.so")
    subprocess.run(["g++", "-std=c++11", "-O2", "-w", "-fPIC", "-shared", "-DPIRE_NO_CONFIG", "-include", "limits",
                    "-I" + REF, "-I" + os.path.join(REF, "pire"), "-I" + os.path.join(LIB, "gen"),
                    os.path.join(HERE, "slow_ref.cpp"), "-L" + LIB, "-lpire_ref", "-Wl,-rpath," + LIB, "-o", so], check=True)
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.slow_ref_compile.restype = C.c_uint64
    lib.slow_ref_compile.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_int), vp,
                                     C.c_uint64]
    lib.slow_ref_null.restype = C.c_uint64
    lib.slow_ref_null.argtypes = [vp, C.c_uint64]
    lib.slow_ref_run.restype = C.c_uint64
    lib.slow_ref_run.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint64, C.c_int, C.c_int, vp, C.c_uint64, vp, vp,
                                 C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
    return lib


def compile_slow(lib, pattern, options="", distance=0, max_size=20000):
    """(SlowScanner image, whether Fsm::Determine(max_size) succeeded); max_size 0 is Determine()'s own limit."""
    det = C.c_int(0)
    n = lib.slow_ref_compile(pattern, len(pattern), options.encode(), distance, max_size, C.byref(det), None, 0)
    assert n, pattern
    buf = C.create_string_buffer(n)
    assert lib.slow_ref_compile(pattern, len(pattern), options.encode(), distance, max_size, C.byref(det), buf, n) == n
    return buf.raw, bool(det.value)


def run(lib, image, strings, begin, end, starts=None, words=1):
    n = len(strings)
    corpus = np.frombuffer(b"".join(strings) + b"\0", np.uint8)
    offsets = np.zeros(n + 1, np.uint64)
    offsets[1:] = np.cumsum([len(s) for s in strings])
    final = np.zeros(max(n, 1), np.uint8)
    letters, empty = C.c_uint64(0), C.c_int(0)
    sets = np.zeros(max(n, 1) * words, np.uint32)
    st = None if starts is None else np.ascontiguousarray(starts, np.uint32)
    size = lib.slow_ref_run(image, len(image), corpus.ctypes.data, offsets.ctypes.data, n, int(begin), int(end),
                            None if st is None else st.ctypes.data, words, final.ctypes.data, sets.ctypes.data,
                            C.byref(letters), C.byref(empty))
    assert size, "reference refused the image"
    return int(size), int(letters.value), bool(empty.value), final[:n].tolist(), sets[: n * words]


def entry(lib, name, image, strings, determinable, seed, patterns=None):
    size, letters, empty, _, _ = run(lib, image, [], True, True)
    words = (size + 31) // 32
    rng = np.random.default_rng(seed)
    starts = rng.integers(0, 1 << 32, len(strings) * words, dtype=np.uint64).astype(np.uint32)
    starts &= rng.integers(0, 1 << 32, starts.size, dtype=np.uint64).astype(np.uint32)   # sparser sets
    e = {"name": name, "image": base64.b64encode(lzma.compress(image)).decode(), "states": size, "letters": letters,
         "empty": empty, "determinable": determinable, "strings": [s.hex() for s in strings],
         "start_sets": starts.tobytes().hex(), "runs": []}
    if patterns is not None:
        e["patterns"] = patterns
    for begin in (False, True):
        for end in (False, True):
            for from_sets in (False, True):
                _, _, _, final, sets = run(lib, image, strings, begin, end, starts if from_sets else None, words)
                e["runs"].append({"begin": begin, "end": end, "from_sets": from_sets, "final": final,
                                  "sets": sets.tobytes().hex()})
    return e


def random_strings(rng, alphabet, count, max_len, plant=None):
    out = []
    for k in range(count):
        n = int(rng.integers(0, max_len + 1))
        s = bytes(rng.choice(np.frombuffer(alphabet.encode(), np.uint8), n).tolist())
        if plant is not None and k % 2 == 0 and n >= len(plant):
            at = int(rng.integers(0, n - len(plant) + 1))
            s = s[:at] + plant + s[at + len(plant):]
        out.append(s)
    return out


def main():
    entries = []
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_helper(tmp)
        rng = np.random.default_rng(20261019)

        image, det = compile_slow(lib, rb"a.{30}$")
        ut = [b"....a..............................", b"....a...............................", b"....a............................."]
        e = entry(lib, "slow_ut", image, ut, det, 1)
        assert [r["final"] for r in e["runs"] if r["begin"] and r["end"] and not r["from_sets"]] == [[1, 0, 0]]   # RunRegexp
        entries.append(e)

        with open(os.path.join(HERE, "pire_golden.json")) as f:
            cases = json.load(f)["cases"]
        for c in cases:
            if len(c["patterns"]) != 1:
                continue
            pat, opts = c["patterns"][0]
            image, det = compile_slow(lib, bytes.fromhex(pat), opts)
            strings = [bytes.fromhex(s) for s in c["strings"]]
            e = entry(lib, "golden/" + c["name"], image, strings, det, len(entries), patterns=c["patterns"])
            want = [r["final"] for r in e["runs"] if r["begin"] == bool(c["begin"]) and r["end"] == bool(c["end"])
                    and not r["from_sets"]]
            assert want == [c["final"]], c["name"]
            entries.append(e)

        buf = C.create_string_buffer(4096)
        n = lib.slow_ref_null(buf, 4096)
        e = entry(lib, "empty", buf.raw[:n], [b"", b"a string", b"a"], False, 2)
        assert e["empty"] and e["states"] == 1
        entries.append(e)

        word = b"internationalization"
        for d in (1, 2):
            image, det = compile_slow(lib, word, "", d)
            strings = [b"internationalisation", b"internationalization", b"xx intrnationalization yy", b"interzzzionalization",
                       b"", b"nationalization"] + random_strings(rng, "inter", 10, 200, plant=b"internatonalizaton")
            entries.append(entry(lib, "approx%d" % d, image, strings, det, 3 + d))

        for name, pat, alphabet in HEAVY:
            image, det = compile_slow(lib, pat)
            strings = random_strings(rng, alphabet, 24, 600) + [b"", b"a" * 31, b"x" * 41, b"foo" + b"." * 64 + b"bar"]
            entries.append(entry(lib, "heavy/" + name, image, strings, det, len(entries)))
            assert not det, name

    data = json.dumps({"note": "generated by tests/golden/make_slow_images.py from the reference", "entries": entries},
                      sort_keys=True).encode()
    with open(OUT, "wb") as f:
        f.write(lzma.compress(data, preset=9))
    print("%s: %d entries, %d bytes" % (OUT, len(entries), os.path.getsize(OUT)))


if __name__ == "__main__":
    sys.exit(main())
