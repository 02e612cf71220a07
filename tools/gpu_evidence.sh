#!/usr/bin/env bash
# Evidence run at bench size: launch list + one full ncu capture of the chosen scan kernel, per workload.
# Nsight Compute reports under $OUT (default evidence_out/).
OUT=${OUT:-evidence_out}; mkdir -p "$OUT"
for wl in ${WORKLOADS:-glue10 headline}; do
  timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 80 --csv --log-file $OUT/launches_$wl.csv \
      python bench.py --workload $wl --steps 3 --warmup 3 --no-e2e --no-cpu > $OUT/ncu_launches_$wl.log 2>&1
  timeout 1200 ncu --set full --clock-control none --import-source on -k regex:Scan -s 8 -c 1 -f -o $OUT/prof_full_$wl \
      python bench.py --workload $wl --steps 3 --warmup 3 --no-e2e --no-cpu > $OUT/ncu_full_$wl.log 2>&1
done
if [ -n "${MIXED:-}" ]; then
  timeout 1200 ncu --set full --clock-control none --import-source on -k regex:ScanGeneric -s 6 -c 1 -f -o $OUT/prof_full_utf8mixed \
      python bench.py --workload utf8mixed --steps 2 --warmup 3 --no-e2e --no-cpu --variant plain > $OUT/ncu_full_utf8mixed.log 2>&1
fi
ls -la $OUT/*.ncu-rep
