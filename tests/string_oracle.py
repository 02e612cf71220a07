"""Runner(sc, st).[Begin()].Run(text).[End()] on the oracle (TEST INFRASTRUCTURE): the run of one string from any
state, the independent answer for pire_gpu_run_string's resume tests.  It drives the entries of oracle/pire_oracle.c
that already take a state -- pire_oracle_step and pire_oracle_run -- from a StateIndex (a state of the oracle is the
byte offset of its row, StateIndex times the row size, multi.h:281-284).  Nothing under pire_b200/ imports it."""
import ctypes as C

import numpy as np

from refpire import Oracle, _OracleStruct

BEGIN_MARK, END_MARK = 258, 259
_bound = False


def _lib():
    global _bound
    lib = Oracle._lib
    if not _bound:
        sp = C.POINTER(_OracleStruct)
        lib.pire_oracle_step.restype = C.c_uint64
        lib.pire_oracle_step.argtypes = [sp, C.c_uint64, C.c_uint]
        lib.pire_oracle_run.restype = C.c_uint64
        lib.pire_oracle_run.argtypes = [sp, C.c_uint64, C.c_void_p, C.c_void_p]
        lib.pire_oracle_initial.restype = C.c_uint64
        lib.pire_oracle_initial.argtypes = [sp]
        lib.pire_oracle_final.argtypes = [sp, C.c_uint64]
        lib.pire_oracle_state_index.restype = C.c_uint64
        lib.pire_oracle_state_index.argtypes = [sp, C.c_uint64]
        lib.pire_oracle_accepted.restype = C.c_size_t
        lib.pire_oracle_accepted.argtypes = [sp, C.c_uint64, C.POINTER(C.c_uint64), C.c_size_t]
        _bound = True
    return lib


class StringWalk:
    """One string on the oracle, fed in pieces: ``StringWalk(orc, start).Begin().Run(a).Run(b).End().result()``.
    start = a StateIndex, or None for Initialize()."""

    def __init__(self, orc, start=None):
        self._orc, self._lib = orc, _lib()
        self._sc = C.byref(orc._sc)
        self.valid = start is None or 0 <= start < orc.states
        if start is None:
            self._st = self._lib.pire_oracle_initial(self._sc)
        else:
            self._st = int(start) * orc._sc.row_cells * 4 if self.valid else 0

    def Begin(self):
        if self.valid:
            self._st = self._lib.pire_oracle_step(self._sc, self._st, BEGIN_MARK)
        return self

    def Run(self, text):
        text = np.ascontiguousarray(text, dtype=np.uint8)
        if self.valid and text.size:
            base = text.ctypes.data
            self._st = self._lib.pire_oracle_run(self._sc, self._st, base, base + text.size)
        return self

    def End(self):
        if self.valid:
            self._st = self._lib.pire_oracle_step(self._sc, self._st, END_MARK)
        return self

    def result(self):
        """(final, accept mask of the ids below 32, StateIndex); (0, 0, 0xFFFFFFFF) for a start outside the scanner."""
        if not self.valid:
            return 0, 0, 0xFFFFFFFF
        ids = (C.c_uint64 * 4096)()
        k = self._lib.pire_oracle_accepted(self._sc, self._st, ids, 4096)
        mask = 0
        for i in range(min(k, 4096)):
            if ids[i] < 32:
                mask |= 1 << ids[i]
        return (int(self._lib.pire_oracle_final(self._sc, self._st)), mask,
                int(self._lib.pire_oracle_state_index(self._sc, self._st)))


def run_from(orc, text, start=None, begin=True, end=True):
    w = StringWalk(orc, start)
    if begin:
        w.Begin()
    w.Run(text)
    if end:
        w.End()
    return w.result()
