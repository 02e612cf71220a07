"""ctypes faces of the two checkers (TEST INFRASTRUCTURE):

* ``Ref``    -- the real reference, compiled from /root/reference into
               oracle/_ref/libpire_ref.so by oracle/build_ref.sh;
* ``Oracle`` -- the plain-C restatement oracle/pire_oracle.c over the
               reference's serialised scanner image.

Nothing under pire_b200/ imports this module.
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libpire_ref.so")
ORACLE_SO = os.path.join(ROOT, "oracle", "libpire_oracle.so")

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


def have_ref():
    return os.path.exists(REF_SO)


def _ptr(arr, typ):
    return None if arr is None else arr.ctypes.data_as(typ)


class RefScanner:
    """A compiled reference scanner (all variants)."""

    def __init__(self, lib, handle):
        self._lib, self._h = lib, handle

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.pref_free(self._h)
            self._h = None

    empty = property(lambda s: bool(s._lib.pref_empty(s._h)))
    size = property(lambda s: s._lib.pref_size(s._h))
    letters = property(lambda s: s._lib.pref_letters_count(s._h))
    regexps = property(lambda s: s._lib.pref_regexps_count(s._h))
    initial = property(lambda s: s._lib.pref_initial_index(s._h))

    def next(self, state, ch):
        return self._lib.pref_next_index(self._h, state, ch)

    def final(self, state):
        return bool(self._lib.pref_final(self._h, state))

    def dead(self, state):
        return bool(self._lib.pref_dead(self._h, state))

    def accepted(self, state):
        ids = (C.c_uint64 * 256)()
        k = self._lib.pref_accepted(self._h, state, ids, 256)
        return [int(ids[i]) for i in range(min(k, 256))]

    def save(self):
        n = self._lib.pref_save(self._h, None, 0)
        buf = (C.c_uint8 * n)()
        self._lib.pref_save(self._h, buf, n)
        return bytes(buf)

    def prefix(self, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_begin=False, through_end=False,
               variant=2):
        """Pire::LongestPrefix / ShortestPrefix per string: length or -1.  variant 0 = Scanner
        (ExitMasks), 2 = NonrelocScannerNoMask."""
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            n = len(offsets) - 1 if n is None else n
        out = np.zeros(n, np.int64)
        rc = self._lib.pref_prefix_batch(self._h, variant, int(shortest), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                         int(through_begin), int(through_end), out.ctypes.data_as(C.POINTER(C.c_int64)))
        assert rc == 0
        return out

    def suffix(self, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_end=False, through_begin=False,
               variant=2):
        """Pire::LongestSuffix / ShortestSuffix per string (walked from its last byte): length or -1."""
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            n = len(offsets) - 1 if n is None else n
        out = np.zeros(n, np.int64)
        rc = self._lib.pref_suffix_batch(self._h, variant, int(shortest), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                         int(through_end), int(through_begin), out.ctypes.data_as(C.POINTER(C.c_int64)))
        assert rc == 0
        return out

    def run(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, variant=1, threads=1,
            want=("final", "mask", "state")):
        """Runner(sc).[Begin()].Run(str).[End()] per string (run.h:365-392)."""
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            n = len(offsets) - 1 if n is None else n
        elif n is None:
            n = len(corpus) // fixed_len if fixed_len else 0
        final = np.zeros(n, np.uint8) if "final" in want else None
        mask = np.zeros(n, np.uint32) if "mask" in want else None
        state = np.zeros(n, np.uint32) if "state" in want else None
        rc = self._lib.pref_run_batch(self._h, variant, _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                      int(begin), int(end), threads, _ptr(final, u8p), _ptr(mask, u32p),
                                      _ptr(state, u32p))
        assert rc == 0
        return final, mask, state


class RefHalfFinal:
    """A reference HalfFinalScanner (pire/scanners/half_final.h)."""

    def __init__(self, lib, handle):
        self._lib, self._h = lib, handle

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.pref_hf_free(self._h)
            self._h = None

    empty = property(lambda s: bool(s._lib.pref_hf_empty(s._h)))
    size = property(lambda s: s._lib.pref_hf_size(s._h))
    regexps = property(lambda s: s._lib.pref_hf_regexps_count(s._h))

    def save(self):
        n = self._lib.pref_hf_save(self._h, None, 0)
        buf = (C.c_uint8 * n)()
        self._lib.pref_hf_save(self._h, buf, n)
        return bytes(buf)

    def count(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, threads=1):
        """tests/count_ut.cpp:54-63 per string: (counts[n, regexps] u32, final[n] u8)."""
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            n = len(offsets) - 1 if n is None else n
        elif n is None:
            n = len(corpus) // fixed_len if fixed_len else 0
        counts = np.zeros((n, max(1, self.regexps)), np.uint32)
        final = np.zeros(n, np.uint8)
        rc = self._lib.pref_hf_count_batch(self._h, _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n, int(begin), int(end),
                                           threads, _ptr(counts, u32p), _ptr(final, u8p))
        assert rc == 0
        return counts, final


class Ref:
    def __init__(self):
        if not have_ref():
            raise RuntimeError("oracle/_ref/libpire_ref.so missing: run oracle/build_ref.sh (needs /root/reference)")
        lib = C.CDLL(REF_SO)
        lib.pref_compile.restype = C.c_void_p
        lib.pref_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]
        lib.pref_glue.restype = C.c_void_p
        lib.pref_glue.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]
        lib.pref_empty_scanner.restype = C.c_void_p
        lib.pref_free.argtypes = [C.c_void_p]
        for f in ("pref_size", "pref_letters_count", "pref_regexps_count", "pref_initial_index"):
            getattr(lib, f).restype = C.c_uint64
            getattr(lib, f).argtypes = [C.c_void_p]
        lib.pref_empty.argtypes = [C.c_void_p]
        lib.pref_next_index.restype = C.c_uint64
        lib.pref_next_index.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32]
        lib.pref_final.argtypes = [C.c_void_p, C.c_uint64]
        lib.pref_dead.argtypes = [C.c_void_p, C.c_uint64]
        lib.pref_accepted.restype = C.c_uint64
        lib.pref_accepted.argtypes = [C.c_void_p, C.c_uint64, u64p, C.c_uint64]
        lib.pref_save.restype = C.c_uint64
        lib.pref_save.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        lib.pref_run_batch.argtypes = [C.c_void_p, C.c_int, u8p, u64p, C.c_uint64, C.c_uint64, C.c_int, C.c_int,
                                       C.c_int, u8p, u32p, u32p]
        lib.pref_prefix_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, u8p, u64p, C.c_uint64, C.c_uint64, C.c_int, C.c_int,
                                          C.POINTER(C.c_int64)]
        lib.pref_suffix_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, u8p, u64p, C.c_uint64, C.c_uint64, C.c_int, C.c_int,
                                          C.POINTER(C.c_int64)]
        lib.pref_hardware_threads.restype = C.c_uint
        lib.pref_hf_compile.restype = C.c_void_p
        lib.pref_hf_compile.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_size_t]
        lib.pref_hf_glue.restype = C.c_void_p
        lib.pref_hf_glue.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]
        lib.pref_hf_load.restype = C.c_void_p
        lib.pref_hf_load.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        lib.pref_hf_free.argtypes = [C.c_void_p]
        lib.pref_hf_empty.argtypes = [C.c_void_p]
        for f in ("pref_hf_size", "pref_hf_regexps_count"):
            getattr(lib, f).restype = C.c_uint64
            getattr(lib, f).argtypes = [C.c_void_p]
        lib.pref_hf_save.restype = C.c_uint64
        lib.pref_hf_save.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        lib.pref_hf_count_batch.argtypes = [C.c_void_p, u8p, u64p, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, u32p, u8p]
        self.lib = lib

    def compile_half_final(self, pattern, opts="", mode=0):
        """mode 0 = HalfFinalScanner(fsm); 1..5 = the counters of count_ut.cpp:503-520."""
        if isinstance(pattern, str):
            pattern = pattern.encode("latin-1")
        err = C.create_string_buffer(512)
        h = self.lib.pref_hf_compile(pattern, opts.encode(), mode, err, len(err))
        if not h:
            raise ValueError(err.value.decode(errors="replace"))
        return RefHalfFinal(self.lib, h)

    def load_half_final(self, image):
        """Scanner::Load of a stored HalfFinalScanner image."""
        err = C.create_string_buffer(512)
        h = self.lib.pref_hf_load(bytes(image), len(image), err, len(err))
        if not h:
            raise ValueError(err.value.decode(errors="replace"))
        return RefHalfFinal(self.lib, h)

    def glue_half_final(self, a, b, max_size=0):
        err = C.create_string_buffer(512)
        h = self.lib.pref_hf_glue(a._h, b._h, max_size, err, len(err))
        if not h:
            raise ValueError(err.value.decode(errors="replace"))
        return RefHalfFinal(self.lib, h)

    def compile(self, pattern, opts=""):
        if isinstance(pattern, str):
            pattern = pattern.encode("latin-1")
        err = C.create_string_buffer(512)
        h = self.lib.pref_compile(pattern, opts.encode(), err, len(err))
        if not h:
            raise ValueError(err.value.decode(errors="replace"))
        return RefScanner(self.lib, h)

    def glue(self, a, b, max_size=0):
        err = C.create_string_buffer(512)
        h = self.lib.pref_glue(a._h, b._h, max_size, err, len(err))
        if not h:
            raise ValueError(err.value.decode(errors="replace"))
        return RefScanner(self.lib, h)

    def glue_all(self, patterns):
        """tools/bench/bench.cpp:108-132: glue left to right."""
        sc = None
        for pat, opts in patterns:
            one = self.compile(pat, opts)
            sc = one if sc is None else self.glue(sc, one)
            if sc.empty:
                raise ValueError("Scanner gluing failed at regexp %r - pattern too complicated" % (pat,))
        return sc

    def empty_scanner(self):
        return RefScanner(self.lib, self.lib.pref_empty_scanner())

    def hardware_threads(self):
        return int(self.lib.pref_hardware_threads())


class _OracleStruct(C.Structure):
    _fields_ = [("states", C.c_uint32), ("letters", C.c_uint32), ("regexps", C.c_uint32),
                ("final_table_size", C.c_uint32), ("initial", C.c_uint64), ("shortcutting", C.c_uint64),
                ("header_cells", C.c_uint32), ("row_cells", C.c_uint32), ("empty", C.c_int),
                ("letter_of", C.c_void_p), ("final_tab", C.c_void_p), ("final_idx", C.c_void_p),
                ("trans", C.c_void_p)]


class Oracle:
    """oracle/pire_oracle.c over one serialised scanner image."""
    _lib = None

    def __init__(self, image):
        if Oracle._lib is None:
            if not os.path.exists(ORACLE_SO):
                raise RuntimeError("oracle/libpire_oracle.so missing: run `make` (or __graft_entry__.build())")
            lib = C.CDLL(ORACLE_SO)
            lib.pire_oracle_load.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(_OracleStruct)]
            lib.pire_oracle_run_batch.restype = None
            lib.pire_oracle_run_batch.argtypes = [C.POINTER(_OracleStruct), u8p, u64p, C.c_uint64, C.c_uint64,
                                                  C.c_int, C.c_int, C.c_int, u8p, u32p, u32p]
            lib.pire_oracle_prefix_batch.restype = None
            lib.pire_oracle_prefix_batch.argtypes = [C.POINTER(_OracleStruct), u8p, u64p, C.c_uint64, C.c_uint64, C.c_int,
                                                     C.c_int, C.c_int, C.POINTER(C.c_int64)]
            lib.pire_oracle_suffix_batch.restype = None
            lib.pire_oracle_suffix_batch.argtypes = [C.POINTER(_OracleStruct), u8p, u64p, C.c_uint64, C.c_uint64, C.c_int,
                                                     C.c_int, C.c_int, C.POINTER(C.c_int64)]
            lib.pire_oracle_count_batch.restype = None
            lib.pire_oracle_count_batch.argtypes = [C.POINTER(_OracleStruct), u8p, u64p, C.c_uint64, C.c_uint64, C.c_int,
                                                    C.c_int, u32p, u8p]
            Oracle._lib = lib
        # keep an 8-byte aligned private copy alive for the views
        self._buf = np.frombuffer(bytes(image) + b"\0" * 8, dtype=np.uint8).copy()
        base = self._buf.ctypes.data
        assert base % 8 == 0
        self._sc = _OracleStruct()
        rc = Oracle._lib.pire_oracle_load(C.c_void_p(base), len(image), C.byref(self._sc))
        if rc != 0:
            raise ValueError("pire_oracle_load failed: %d" % rc)
        self.states, self.letters, self.regexps = self._sc.states, self._sc.letters, self._sc.regexps
        self.empty = bool(self._sc.empty)

    def run(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, shortcuts=False):
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            n = len(offsets) - 1 if n is None else n
        elif n is None:
            n = len(corpus) // fixed_len if fixed_len else 0
        final = np.zeros(n, np.uint8)
        mask = np.zeros(n, np.uint32)
        state = np.zeros(n, np.uint32)
        Oracle._lib.pire_oracle_run_batch(C.byref(self._sc), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                          int(begin), int(end), int(shortcuts), _ptr(final, u8p), _ptr(mask, u32p),
                                          _ptr(state, u32p))
        return final, mask, state


def oracle_count(orc, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True):
    """HalfFinalScanner counting through the oracle port: (counts[n, regexps], final[n])."""
    corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
    if offsets is not None:
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1 if n is None else n
    elif n is None:
        n = len(corpus) // fixed_len if fixed_len else 0
    counts = np.zeros((n, max(1, orc.regexps)), np.uint32)
    final = np.zeros(n, np.uint8)
    Oracle._lib.pire_oracle_count_batch(C.byref(orc._sc), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n, int(begin),
                                        int(end), _ptr(counts, u32p), _ptr(final, u8p))
    return counts, final


def oracle_prefix(orc, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_begin=False, through_end=False):
    corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
    if offsets is not None:
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1 if n is None else n
    out = np.zeros(n, np.int64)
    Oracle._lib.pire_oracle_prefix_batch(C.byref(orc._sc), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                         int(through_begin), int(through_end), int(shortest),
                                         out.ctypes.data_as(C.POINTER(C.c_int64)))
    return out


def oracle_suffix(orc, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_end=False, through_begin=False):
    corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
    if offsets is not None:
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1 if n is None else n
    out = np.zeros(n, np.int64)
    Oracle._lib.pire_oracle_suffix_batch(C.byref(orc._sc), _ptr(corpus, u8p), _ptr(offsets, u64p), fixed_len, n,
                                         int(through_end), int(through_begin), int(shortest),
                                         out.ctypes.data_as(C.POINTER(C.c_int64)))
    return out


def csr(strings):
    """Concatenate byte strings into the (corpus, offsets[n+1]) form of the batch API.
    Alignment cases (pire_ut.cpp Aligned@729) arise from the lengths of the
    preceding strings; callers interleave junk strings to shift them."""
    offs = np.zeros(len(strings) + 1, np.uint64)
    total = 0
    for i, s in enumerate(strings):
        total += len(s)
        offs[i + 1] = total
    corpus = np.frombuffer(b"".join(strings) + b"\0" * 32, dtype=np.uint8).copy()
    return corpus, offs


# ----------------------------------------------------------------------------- the reference's answers, stored
#
# The tests that compare with the reference (``ref`` fixture) run without it too: every scanner image the reference
# compiled for them and a SHA-256 of every answer it gave are kept in tests/golden/reference_answers.json.xz.  Without
# oracle/_ref the answers are recomputed by the oracle over the stored image and must hash to what the reference
# returned; where the oracle cannot give the reference's answer (the default scanner's LongestPrefix on 16-byte
# boundaries, accepted-regexp lists) the answer itself is stored.  PIRE_RECORD_REFERENCE=<file> with oracle/_ref
# built records what a test session asks of the reference into <file> (on top of the committed answers).

import base64
import hashlib
import json
import lzma

STORED_ANSWERS = os.path.join(ROOT, "tests", "golden", "reference_answers.json.xz")
_DATA_DIR = os.path.join(ROOT, "pire_b200", "data")


def _sha(*parts):
    h = hashlib.sha256()
    for p in parts:
        if isinstance(p, np.ndarray):
            a = np.ascontiguousarray(p)
            h.update(str((a.dtype.str, a.shape)).encode())
            h.update(a.reshape(-1).view(np.uint8).data)
        elif isinstance(p, (bytes, bytearray)):
            h.update(bytes(p))
        else:
            h.update(repr(p).encode())
        h.update(b"|")
    return h.hexdigest()


def _call_key(op, image_sha, corpus, offsets, params):
    corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
    offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
    return _sha(op, image_sha, params, corpus, b"" if offsets is None else offsets)[:24]


def _answer_sha(arrays):
    return _sha(*["-" if a is None else a for a in arrays])[:24]


def _pack(a):
    a = np.ascontiguousarray(a)
    return {"dtype": a.dtype.str, "shape": list(a.shape), "xz": base64.b64encode(lzma.compress(a.tobytes())).decode()}


def _unpack(d):
    return np.frombuffer(lzma.decompress(base64.b64decode(d["xz"])), dtype=np.dtype(d["dtype"])).reshape(d["shape"]).copy()


class AnswerStore:
    def __init__(self, path=STORED_ANSWERS):
        self.images, self.ops, self.calls = {}, {}, {}
        if os.path.exists(path):
            with open(path, "rb") as f:
                d = json.loads(lzma.decompress(f.read()))
            self.images, self.ops, self.calls = d["images"], d["ops"], d["calls"]
        self._bytes = {}

    def save(self, path):
        blob = json.dumps({"images": self.images, "ops": self.ops, "calls": self.calls}, sort_keys=True, separators=(",", ":"))
        with open(path, "wb") as f:
            f.write(lzma.compress(blob.encode(), preset=9 | lzma.PRESET_EXTREME))

    def add_image(self, image, meta):
        sha = _sha(image)[:24]
        if sha not in self.images:
            entry = dict(meta)
            for name in sorted(os.listdir(_DATA_DIR)):                # the package's own images are not stored twice
                with open(os.path.join(_DATA_DIR, name), "rb") as f:
                    if lzma.decompress(f.read()) == image:
                        entry["data"] = name
                        break
            else:
                entry["hex"] = image.hex()                                # the file as a whole is compressed
            self.images[sha] = entry
        return sha

    def image(self, sha):
        if sha not in self._bytes:
            e = self.images[sha]
            if "data" in e:
                with open(os.path.join(_DATA_DIR, e["data"]), "rb") as f:
                    self._bytes[sha] = lzma.decompress(f.read())
            else:
                self._bytes[sha] = bytes.fromhex(e["hex"])
        return self._bytes[sha]


def _oracle_answer(orc, op, corpus, offsets, fixed_len, n, kw):
    """The oracle's answer to one of the reference's batch calls, as the tuple of arrays the reference returns."""
    if op == "run":
        return orc.run(corpus, offsets, fixed_len=fixed_len, n=n, begin=kw["begin"], end=kw["end"], shortcuts=True)
    if op == "prefix":
        return (oracle_prefix(orc, corpus, offsets, fixed_len=fixed_len, n=n, shortest=kw["shortest"],
                              through_begin=kw["through_begin"], through_end=kw["through_end"]),)
    if op == "suffix":
        return (oracle_suffix(orc, corpus, offsets, fixed_len=fixed_len, n=n, shortest=kw["shortest"],
                              through_end=kw["through_end"], through_begin=kw["through_begin"]),)
    return oracle_count(orc, corpus, offsets, fixed_len=fixed_len, n=n, begin=kw["begin"], end=kw["end"])


def _batch_n(corpus, offsets, fixed_len, n):
    if offsets is not None:
        return len(offsets) - 1 if n is None else n
    return (len(corpus) // fixed_len if fixed_len else 0) if n is None else n


class StoredScanner:
    """A scanner the reference compiled, with the reference's answers: recorded from a live one (``live`` given, the
    answers are checked against nothing and stored) or replayed through the oracle (``live`` None)."""

    def __init__(self, store, sha, live=None):
        self._store, self._sha, self._live = store, sha, live
        meta = store.images[sha]
        self.empty, self.size, self.letters, self.regexps = meta["empty"], meta["size"], meta["letters"], meta["regexps"]
        self._orc = None

    @property
    def _h(self):
        return self._live._h

    def save(self):
        return self._store.image(self._sha)

    def oracle(self):
        if self._orc is None:
            self._orc = Oracle(self.save())
        return self._orc

    def accepted(self, state):
        key = "accepted:%s:%d" % (self._sha, state)
        if self._live is not None:
            self._store.calls[key] = {"value": self._live.accepted(state)}
        return list(self._store.calls[key]["value"])

    def _batch(self, op, corpus, offsets, fixed_len, n, kw, want, live_call):
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
        n = _batch_n(corpus, offsets, fixed_len, n)
        key = _call_key(op, self._sha, corpus, offsets, (fixed_len, n, sorted(kw.items())) + ((tuple(want),) if want else ()))
        if self._live is not None:
            got = live_call()
            mine = _oracle_answer(self.oracle(), op, corpus, offsets, fixed_len, n, kw)
            entry = {"sha": _answer_sha(got)}
            if any(g is None for g in got):
                entry["none"] = [i for i, g in enumerate(got) if g is None]
            if _answer_sha(got) != _answer_sha([None if g is None else m for g, m in zip(got, mine)]):
                entry["value"] = [None if g is None else _pack(g) for g in got]
            self._store.calls[key] = entry
            return got
        if key not in self._store.calls:
            raise KeyError("no stored reference answer for this %s call (record it with PIRE_RECORD_REFERENCE and "
                           "oracle/_ref built)" % op)
        entry = self._store.calls[key]
        if "value" in entry:
            out = tuple(None if v is None else _unpack(v) for v in entry["value"])
        else:
            out = _oracle_answer(self.oracle(), op, corpus, offsets, fixed_len, n, kw)
        out = tuple(None if i in entry.get("none", ()) else a for i, a in enumerate(out))
        assert _answer_sha(out) == entry["sha"], "the answer differs from the reference's stored one (%s)" % op
        return out

    def run(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, variant=1, threads=1,
            want=("final", "mask", "state")):
        kw = dict(begin=bool(begin), end=bool(end), variant=variant)
        live = lambda: self._live.run(corpus, offsets, fixed_len, n, begin, end, variant, threads, want)   # noqa: E731
        out = self._batch("run", corpus, offsets, fixed_len, n, kw, want, live)
        return tuple(a if name in want else None for a, name in zip(out, ("final", "mask", "state")))

    def prefix(self, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_begin=False, through_end=False, variant=2):
        kw = dict(shortest=bool(shortest), through_begin=bool(through_begin), through_end=bool(through_end), variant=variant)
        live = lambda: (self._live.prefix(corpus, offsets, fixed_len, n, shortest, through_begin, through_end, variant),)   # noqa: E731
        return self._batch("prefix", corpus, offsets, fixed_len, n, kw, None, live)[0]

    def suffix(self, corpus, offsets=None, fixed_len=0, n=None, shortest=False, through_end=False, through_begin=False, variant=2):
        kw = dict(shortest=bool(shortest), through_begin=bool(through_begin), through_end=bool(through_end), variant=variant)
        live = lambda: (self._live.suffix(corpus, offsets, fixed_len, n, shortest, through_end, through_begin, variant),)   # noqa: E731
        return self._batch("suffix", corpus, offsets, fixed_len, n, kw, None, live)[0]

    def count(self, corpus, offsets=None, fixed_len=0, n=None, begin=True, end=True, threads=1):
        kw = dict(begin=bool(begin), end=bool(end))
        live = lambda: self._live.count(corpus, offsets, fixed_len, n, begin, end, threads)   # noqa: E731
        return self._batch("count", corpus, offsets, fixed_len, n, kw, None, live)


class StoredRef:
    """``Ref``'s face over an AnswerStore: replays it, or (``live`` = a Ref) records into it."""

    def __init__(self, store=None, live=None):
        self.store = AnswerStore() if store is None else store
        self._live = live

    def _op(self, key, make):
        key = _sha(*key)[:24]
        if self._live is not None:
            try:
                sc = make()
            except ValueError as ex:
                self.store.ops[key] = {"error": str(ex)}
                raise
            meta = {"empty": bool(sc.empty), "size": int(sc.size), "regexps": int(sc.regexps),
                    "letters": int(sc.letters) if hasattr(sc, "letters") else None}
            self.store.ops[key] = {"image": self.store.add_image(sc.save(), meta)}
            return StoredScanner(self.store, self.store.ops[key]["image"], sc)
        if key not in self.store.ops:
            raise KeyError("no stored reference scanner for this call (record it with PIRE_RECORD_REFERENCE and oracle/_ref built)")
        entry = self.store.ops[key]
        if "error" in entry:
            raise ValueError(entry["error"])
        return StoredScanner(self.store, entry["image"])

    def compile(self, pattern, opts=""):
        if isinstance(pattern, str):
            pattern = pattern.encode("latin-1")
        return self._op(("compile", pattern, opts), lambda: self._live.compile(pattern, opts))

    def glue(self, a, b, max_size=0):
        return self._op(("glue", a._sha, b._sha, max_size), lambda: self._live.glue(a._live, b._live, max_size))

    def glue_all(self, patterns):
        return self._op(("glue_all", [(bytes(p), o) for p, o in patterns]), lambda: self._live.glue_all(patterns))

    def compile_half_final(self, pattern, opts="", mode=0):
        if isinstance(pattern, str):
            pattern = pattern.encode("latin-1")
        return self._op(("compile_half_final", pattern, opts, mode), lambda: self._live.compile_half_final(pattern, opts, mode))

    def glue_half_final(self, a, b, max_size=0):
        return self._op(("glue_half_final", a._sha, b._sha, max_size), lambda: self._live.glue_half_final(a._live, b._live, max_size))

    def hardware_threads(self):
        return os.cpu_count() or 1
