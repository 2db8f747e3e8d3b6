#!/bin/bash
# Development aid, runs on the GPU box: stage times of the default pipeline for a list of "variant[,ENV=VAL...]" specs.
#   tools/ab2.sh main unroll2 main      (variants built by tools/build_variant.sh, here: unroll2 -DT3_PRED_UNROLL=2)
# BENCH_ARGS overrides the bench arguments (default: 64 images of 3840x2160, baseline + trellis).
export B200JPEG_BENCH_CACHE=/dev/shm
ARGS=${BENCH_ARGS:---batch 64 --steps 3 --warmup 3}
for SPEC in "$@"; do
  V=${SPEC%%,*}; ENVS=""; [ "$SPEC" != "$V" ] && ENVS=$(echo "${SPEC#*,}" | tr ',' ' ')
  [ "$V" = "main" ] && LV="" || LV=$V
  TAG=$(echo "$SPEC" | tr ',=' '__')
  env $ENVS B200JPEG_LIB_VARIANT=$LV B200JPEG_CHUNK_IMAGES=64 B200JPEG_STREAMS=1 timeout 200 python bench.py $ARGS --no-cpu-baseline --no-e2e > gpurun_out/ab_$TAG.json 2> gpurun_out/ab_$TAG.err
  python - "$TAG" <<'PY'
import json, sys
v = sys.argv[1]
try:
    d = json.load(open(f"gpurun_out/ab_{v}.json")); s = d["roofline"]["stage_ms"]
    print(f"{v:28s} {d['ms_per_step']:7.3f} ms  " + " ".join(f"{k}={x:.2f}" for k, x in s.items() if x >= 0.005))
except Exception as e:
    print(v, "FAILED", e, open(f"gpurun_out/ab_{v}.err").read()[-400:])
PY
done
