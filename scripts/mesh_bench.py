"""Mesh extraction benchmark (toolbox/mesh_extraction: hrf_density_lattice, then hrf_marching_cubes_count / _emit).
Two workloads on the bench model of `--segments`: the lattice over the make_scene hull at G = 256, and a dense lattice
(every vertex) at G = 512.  `--steps` frames after `--warmup`, frames cycled, L2 flushed before each of the two timed
phases, CUDA events around the lattice and around marching cubes (which includes its one count readback).  The
iso-level is the median of the first frame's evaluated lattice values (the bench model's random tables have no real
surface, so this gives a dense, noisy mesh: a heavy case for marching cubes).  Prints one JSON line: ms per frame of
each phase, lattice samples/s, vertex and face counts, and the card's name and power limit.
    python scripts/mesh_bench.py [--segments 50] [--steps 10] [--warmup 3]
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bake_bench import gpu_identity  # noqa: E402


def run(model, frames, G, mask, steps, warmup, flush):
    from humanrf_b200.toolbox.mesh_extraction import density_lattice, marching_cubes

    def lattice(frame):
        return density_lattice(model, frame, mask) if mask is not None else density_lattice(model, frame, resolution=G)

    first = lattice(frames[0])
    evaluated = first != 0 if mask is not None else torch.ones_like(first, dtype=torch.bool)
    level = float(torch.median(first[evaluated]))
    n_eval = int(evaluated.sum())
    for i in range(max(warmup, 1)):
        marching_cubes(lattice(frames[i % len(frames)]), level)
    torch.cuda.synchronize()
    t_lat, t_mc, nv, nf = [], [], [], []
    for i in range(steps):
        frame = frames[(warmup + i) % len(frames)]
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        flush.zero_()
        e[0].record()
        lat = lattice(frame)
        e[1].record()
        flush.zero_()
        e[2].record()
        mesh = marching_cubes(lat, level)
        e[3].record()
        torch.cuda.synchronize()
        t_lat.append(e[0].elapsed_time(e[1]))
        t_mc.append(e[2].elapsed_time(e[3]))
        nv.append(int(mesh.vertices.shape[0]))
        nf.append(int(mesh.faces.shape[0]))
    ms_lat, ms_mc = float(np.mean(t_lat)), float(np.mean(t_mc))
    return {"G": G, "lattice": "hull" if mask is not None else "dense", "level": level,
            "evaluated_vertices": n_eval, "evaluated_fraction": n_eval / (G + 1) ** 3,
            "lattice_ms": ms_lat, "marching_cubes_ms": ms_mc, "lattice_samples_per_s": n_eval / (ms_lat * 1e-3),
            "vertices_mean": float(np.mean(nv)), "faces_mean": float(np.mean(nf))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench.py needs a CUDA device (mesh extraction has no CPU path)")
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene

    dev = torch.device("cuda:0")
    model, frames = make_model(tuple(a.segments), seed=123, device=dev)
    hull = torch.from_numpy(np.ascontiguousarray(make_scene(num_images=1, G=256)["grids"][0])).to(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    workloads = [run(model, frames, 256, hull, a.steps, a.warmup, flush),
                 run(model, frames, 512, None, a.steps, a.warmup, flush)]
    w = workloads[0]
    print(json.dumps({
        "metric": "mesh_extract_ms_per_frame", "value": w["lattice_ms"] + w["marching_cubes_ms"], "unit": "ms/frame",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu": gpu_identity(0), "workloads": workloads,
        "config": {"model": f"bench model, segment_sizes={tuple(a.segments)}", "hull": "make_scene grid 0, G=256",
                   "l2": "flushed before each timed phase (256 MiB memset)",
                   "value": "hull workload, lattice + marching cubes (incl. its count readback)"}}))


if __name__ == "__main__":
    main()
