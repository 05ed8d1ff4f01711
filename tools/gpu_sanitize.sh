#!/bin/bash
# compute-sanitizer over the kernel modes; one log per run under LOG_DIR.
#   tools/gpu_sanitize.sh LOG_DIR
OUT=${1:?usage: tools/gpu_sanitize.sh LOG_DIR}
mkdir -p "$OUT"
S=/usr/local/cuda/bin/compute-sanitizer
for mode in auto fast-split fast-noprune tile queue; do
  for tool in memcheck racecheck; do
    timeout 600 $S --tool $tool --print-limit 20 python tools/sanitize_target.py $mode \
      > "$OUT/${tool}_${mode}.log" 2>&1
    echo "$tool $mode rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' "$OUT/${tool}_${mode}.log" | tail -1)"
  done
done
for tool in synccheck initcheck; do
  timeout 600 $S --tool $tool --print-limit 20 python tools/sanitize_target.py auto \
    > "$OUT/${tool}_auto.log" 2>&1
  echo "$tool auto rc=$? $(grep -E 'ERROR SUMMARY' "$OUT/${tool}_auto.log" | tail -1)"
done
# the region allow-list and the forced full chain evaluation
timeout 600 $S --tool memcheck --print-limit 20 python tools/sanitize_target.py auto full \
  > "$OUT/memcheck_auto_fullchain.log" 2>&1
echo "memcheck auto fullchain rc=$? $(grep -E 'ERROR SUMMARY' "$OUT/memcheck_auto_fullchain.log" | tail -1)"
# every native buffer freed by the time the store is closed
timeout 600 $S --tool memcheck --leak-check full --print-limit 20 python tools/sanitize_target.py auto \
  > "$OUT/memcheck_auto_leaks.log" 2>&1
echo "memcheck auto leaks rc=$? $(grep -E 'ERROR SUMMARY|LEAK SUMMARY' "$OUT/memcheck_auto_leaks.log" | tail -2 | tr '\n' ' ')"
