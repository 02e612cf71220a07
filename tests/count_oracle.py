"""HalfFinalScanner counting of one string from any state on the oracle (TEST INFRASTRUCTURE): the independent answer for
pire_gpu_count_string's resume tests.  It walks string_oracle.StringWalk one symbol at a time with pire_oracle_step and
counts, after every step, each regexp pire_oracle_accepted lists for a final state.  Nothing under pire_b200/ imports it."""
import ctypes as C

import numpy as np

from string_oracle import BEGIN_MARK, END_MARK, StringWalk


def count_from(orc, text, start=None, begin=True, end=True):
    """HalfFinalScanner counting of one string on the oracle, from Initialize() (its TakeAction counted,
    half_final.h:136-141) or from the StateIndex `start` (not counted: the run that reached it did): one
    pire_oracle_step per byte, and after every step one count for each regexp pire_oracle_accepted lists for a final
    state (TakeAction, half_final.h:154-163).  Returns (counts as a list of ints, the StringWalk result); nothing is
    counted from a start outside the scanner.  A byte at a time in Python: for short texts."""
    w = StringWalk(orc, start)
    counts = [0] * max(1, orc.regexps)
    if not w.valid:
        return counts, w.result()
    lib, sc = w._lib, w._sc
    ids = (C.c_uint64 * 4096)()

    def take(st):
        if lib.pire_oracle_final(sc, st):
            for i in range(min(lib.pire_oracle_accepted(sc, st, ids, 4096), 4096)):
                counts[ids[i]] += 1

    if start is None:
        take(w._st)
    symbols = ([BEGIN_MARK] if begin else []) + [int(b) for b in np.asarray(text, dtype=np.uint8)] + ([END_MARK] if end else [])
    for ch in symbols:
        w._st = lib.pire_oracle_step(sc, w._st, ch)
        take(w._st)
    return counts, w.result()
