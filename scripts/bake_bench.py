"""Learned occupancy bake benchmark (hrf_bake_occupancy through toolbox/learned_occupancy.bake_occupancy_grid): the bench
model of `--segments` baked over the make_scene hull at G = 256, `--steps` frames after `--warmup`, frames cycled, L2
flushed between steps, CUDA events around each bake.  Prints one JSON line: ms per frame, evaluated samples/s (8 per hull
voxel), hull / live / baked voxel fractions, the SURVEY 8d-convention bytes (3 072 B per evaluated sample: 2 048 B of
table gathers + 1 024 B of vector taps; positions are generated in the kernel, so no per-sample stream) and the card's
name and power limit.
    python scripts/bake_bench.py [--segments 50] [--steps 20] [--warmup 5]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

BYTES_PER_SAMPLE = 3072


def gpu_identity(index):
    """Card name and power limit, read beside the numbers they qualify."""
    name, limit = torch.cuda.get_device_name(index), None
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        pass
    return {"name": name, "power_limit_w": limit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--G", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bake_bench.py needs a CUDA device (the bake has no CPU path)")
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.learned_occupancy import ALPHA_THRE, bake_occupancy_grid

    dev = torch.device("cuda:0")
    G, step_size = a.G, 4e-4
    model, frames = make_model(tuple(a.segments), seed=123, device=dev)
    hull = torch.from_numpy(np.ascontiguousarray(make_scene(num_images=1, G=G)["grids"][0])).to(dev)
    n_hull = int((hull != 0).sum())
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    w = max(a.warmup, 1)
    for i in range(w):
        flush.zero_()
        bake_occupancy_grid(model, frames[i % len(frames)], hull, step_size)
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(a.steps)]
    for i in range(a.steps):
        flush.zero_()
        ev[i][0].record()
        bake_occupancy_grid(model, frames[(w + i) % len(frames)], hull, step_size)
        ev[i][1].record()
    torch.cuda.synchronize()
    ms = sum(e[0].elapsed_time(e[1]) for e in ev) / a.steps
    out, max_sigma = bake_occupancy_grid(model, frames[(w + a.steps - 1) % len(frames)], hull, step_size,
                                         return_max_sigma=True)
    live = (hull != 0) & ((1 - torch.exp(-max_sigma * step_size)) >= ALPHA_THRE)
    n_vox = G ** 3
    samples_per_s = 8 * n_hull / (ms * 1e-3)
    print(json.dumps({
        "metric": "bake_ms_per_frame", "value": ms, "unit": "ms/frame", "higher_is_better": False, "steps": a.steps,
        "warmup": w, "gpu": gpu_identity(0), "samples_per_s": samples_per_s,
        "algorithmic_bytes_per_sample": BYTES_PER_SAMPLE, "algorithmic_gb_per_s": BYTES_PER_SAMPLE * samples_per_s / 1e9,
        "config": {"workload": f"learned occupancy bake, make_scene hull G={G}, segment_sizes={tuple(a.segments)}, one frame "
                               "per step (compaction + bake kernel + dilate-and-AND)",
                   "l2": "flushed between timed steps (256 MiB memset)", "render_step_size": step_size,
                   "alpha_thre": ALPHA_THRE, "hull_voxels": n_hull, "hull_fraction": n_hull / n_vox,
                   "live_fraction": int(live.sum()) / n_vox, "baked_fraction": int((out != 0).sum()) / n_vox,
                   "note": "the bench model's random tables give density almost everywhere, so the live fraction here says "
                           "nothing about real scenes; gathers served by L2 count as algorithmic bytes"}}))


if __name__ == "__main__":
    main()
