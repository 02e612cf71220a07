"""pire_b200 -- H100-native (sm_90a) implementation of Pire's inner DFA scan path.

Only what the path needs lives here:
    csrc/         sm_90a CUDA kernels + the extern "C" boundary (include/pire_b200.h)
    _native.py    ctypes binding of that boundary (fails loudly if the .so is missing)
    scanner.py    Python mirror of Pire's Scanner / Runner / Matches for batches, StringRunner, StringCounter and
                  StringMatchEnds for one long string, BatchCounter and BatchMatchEnds for many streams,
                  MatchStarts for the starts of either's matches
    workloads.py  the BASELINE.json pattern sets and synthetic corpora
    dist.py       shard-by-string + the one bitmap all-reduce
"""
from ._native import PireGpuError, RUN_BEGIN, RUN_END, VARIANT_AUTO, VARIANT_PLAIN, VARIANT_PRED, VARIANT_PRIV, VARIANT_LOOK  # noqa: F401
from .scanner import (Batch, BatchCounter, BatchMatchEnds, BeginMark, EndMark, HalfFinalCount, HalfFinalResult, LongestPrefix, LongestSuffix, Matches,  # noqa: F401
                      MatchStarts, MatchStartsResult, NO_START, RunHelper, Runner, Scanner, ShortestPrefix, ShortestSuffix, StringCounter, StringMatchEnds, StringRunner)
