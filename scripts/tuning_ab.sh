#!/bin/bash
# A/B of the tuning knobs whose defaults are compiled into the kernels (DESIGN.md section 3): forward CTAs per SM and the
# encode-loop unroll on the render bench, the scatter generation on the train bench.  One bench JSON line per setting,
# the default setting first and last (its spread is the noise floor of the comparison).
# usage: scripts/tuning_ab.sh <output dir> [steps]
out=${1:?usage: tuning_ab.sh <output dir> [steps]}
steps=${2:-50}
mkdir -p "$out"
b() { python bench.py --gpus 1 --steps "$steps" --warmup 5 --no-cpu-baseline --no-companions "$@"; }
b --mode render > "$out/render_default_a.json"
HRF_FWD_CTAS=4 b --mode render > "$out/render_ctas4_unroll4.json"
HRF_FWD_CTAS=6 HRF_FWD_UNROLL=1 b --mode render > "$out/render_ctas6_unroll1.json"
HRF_FWD_UNROLL=2 b --mode render > "$out/render_unroll2.json"
HRF_FWD_UNROLL=4 b --mode render > "$out/render_unroll4.json"
b --mode render > "$out/render_default_b.json"
b > "$out/train_default_a.json"
for g in 1 2 4 5; do HRF_SCATTER=$g b > "$out/train_scatter$g.json"; done
HRF_SCATTER_CTAS=6 b > "$out/train_scatter3_ctas6.json"
b > "$out/train_default_b.json"
