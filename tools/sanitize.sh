#!/bin/bash
# compute-sanitizer memcheck + racecheck + initcheck of the smoke frame (tiger 256x256, MSAA16 and area AA) plus a frame that
# exercises clips / blends / gradients / images (tools/sanitize_frame.py). Logs land in sanitizer_logs/.
# Usage (GPU box): tools/sanitize.sh [tag]
tag=${1:-r2}
mkdir -p sanitizer_logs
for tool in memcheck racecheck initcheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitize_frame.py > sanitizer_logs/sanitizer_${tool}_${tag}.log 2>&1
  echo "$tool rc=$?" >> sanitizer_logs/sanitizer_${tool}_${tag}.log
  tail -4 sanitizer_logs/sanitizer_${tool}_${tag}.log
done
