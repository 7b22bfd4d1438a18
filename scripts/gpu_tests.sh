#!/bin/bash
# Runs every GPU test file in its own process (a sticky CUDA error in one file must not poison the rest),
# one log per file and a summary under the output directory.  usage: scripts/gpu_tests.sh <output dir>
out=${1:?usage: gpu_tests.sh <output dir>}
mkdir -p "$out"
: > "$out/summary.txt"
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,memory.total --format=csv > "$out/gpu.txt" 2>&1
for f in tests/test_*_gpu.py; do
  n=$(basename $f .py)
  timeout 900 python -m pytest $f -q -m gpu -s -x --no-header -p no:cacheprovider > "$out/$n.log" 2>&1
  echo "$n exit=$? $(tail -1 "$out/$n.log")" | tee -a "$out/summary.txt"
done
