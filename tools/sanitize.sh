#!/bin/bash
# Run on a machine with the GPU: compute-sanitizer memcheck and racecheck over small encodes that reach every kernel
# family; the logs are the evidence kept under profiles/ (SURVEY 5: the reference relies on ASan/valgrind jobs).
#   tools/sanitize.sh [log directory, default profiles]
OUT=${1:-profiles}
mkdir -p "$OUT"
for TOOL in memcheck racecheck; do
  OPTS=(); [ $TOOL = memcheck ] && OPTS=(--leak-check full)   # the closed encoders must leave no device allocation behind
  timeout 900 compute-sanitizer --tool $TOOL "${OPTS[@]}" --print-limit 20 python tools/sanitize_cases.py > "$OUT/sanitizer_$TOOL.log" 2>&1
  echo "== $TOOL: exit $?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|sanitize cases done|Error:|hazard|Leaked" "$OUT/sanitizer_$TOOL.log" | head -8
done
