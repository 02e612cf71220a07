#!/usr/bin/env bash
# memcheck and racecheck over tools/sanitize_run.py; logs under $OUT (default sanitizer_out/).
OUT=${OUT:-sanitizer_out}; mkdir -p "$OUT"
timeout 1200 compute-sanitizer --tool memcheck --error-exitcode 7 python tools/sanitize_run.py > $OUT/sanitizer_memcheck.log 2>&1; echo "memcheck exit $?" | tee -a $OUT/sanitizer_memcheck.log
tail -6 $OUT/sanitizer_memcheck.log
timeout 1200 compute-sanitizer --tool racecheck --error-exitcode 7 python tools/sanitize_run.py > $OUT/sanitizer_racecheck.log 2>&1; echo "racecheck exit $?" | tee -a $OUT/sanitizer_racecheck.log
tail -6 $OUT/sanitizer_racecheck.log
