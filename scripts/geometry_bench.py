"""Geometry score benchmark (toolbox/geometry_metrics: hrf_mesh_distance).  Workload: the bench model's G = 256 hull
mesh (mesh_bench.py's, about 2.1 M faces) of frame 0 against the same extraction of another frame, `--samples` points
per side (1 M).  One direction is one hrf_mesh_distance call; `--steps` calls per direction after `--warmup`, L2
flushed before each, CUDA events around each call.  A separate torch.profiler run of one call per direction splits the
kernel time into sampling (source prep, weights, scan, sample kernel, query-order sort), tree build (target prep, Morton
keys, sort, leaves, refit) and queries (query + finish kernels).  Prints one JSON line with the card's name and power
limit.
    python scripts/geometry_bench.py [--samples 1000000] [--steps 10] [--warmup 3]
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


def meshes(dev):
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.mesh_extraction import density_lattice, marching_cubes

    model, frames = make_model((50,), seed=123, device=dev)
    hull = torch.from_numpy(np.ascontiguousarray(make_scene(num_images=1, G=256)["grids"][0])).to(dev)
    lat = density_lattice(model, frames[0], hull)
    level = float(torch.median(lat[lat != 0]))
    return (marching_cubes(lat, level, normals=False),
            marching_cubes(density_lattice(model, frames[5], hull), level, normals=False))


def phases(src, dst, n):
    """Kernel time of one call split into the three phases, from a torch.profiler trace (ms)."""
    from torch.profiler import ProfilerActivity, profile

    from humanrf_b200.toolbox.geometry_metrics import mesh_distance

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mesh_distance(src, dst, n, 1)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
                 and "Memset" not in e.name), key=lambda e: e.time_range.start)
    names = [e.name for e in ev]
    preps = [i for i, nm in enumerate(names) if "prep_kernel" in nm]
    q = next(i for i, nm in enumerate(names) if "query_kernel" in nm)
    t = [e.time_range.elapsed_us() / 1e3 for e in ev]
    return {"sampling_ms": sum(t[:preps[1]]), "build_ms": sum(t[preps[1]:q]), "query_ms": sum(t[q:]),
            "kernels": len(ev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("geometry_bench.py needs a CUDA device (the mesh distance has no CPU path)")
    from humanrf_b200.toolbox.geometry_metrics import mesh_distance

    dev = torch.device("cuda:0")
    src, dst = meshes(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    n = a.samples
    result = {}
    for name, (x, y) in (("pred_to_ref", (src, dst)), ("ref_to_pred", (dst, src))):
        for i in range(max(a.warmup, 1)):
            mesh_distance(x, y, n, i)
        torch.cuda.synchronize()
        times = []
        for i in range(a.steps):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            flush.zero_()
            e[0].record()
            out, _, _, _ = mesh_distance(x, y, n, a.warmup + i)
            e[1].record()
            torch.cuda.synchronize()
            times.append(e[0].elapsed_time(e[1]))
        result[name] = {"call_ms": float(np.mean(times)), "call_ms_min": float(np.min(times)),
                        "mean_distance": float(out[0]), **phases(x, y, n)}
    total = result["pred_to_ref"]["call_ms"] + result["ref_to_pred"]["call_ms"]
    print(json.dumps({
        "metric": "geometry_score_ms_per_frame", "value": total, "unit": "ms/frame", "higher_is_better": False,
        "steps": a.steps, "warmup": a.warmup, "gpu": gpu_identity(0), "samples_per_side": n,
        "faces": [int(src.faces.shape[0]), int(dst.faces.shape[0])], "directions": result,
        "config": {"meshes": "bench model segment_sizes=(50,), make_scene hull G=256, frames 0 and 5, median level",
                   "l2": "flushed before each timed call (256 MiB memset)",
                   "value": "both directions, one hrf_mesh_distance call each (CUDA events)",
                   "phases": "kernel time of one profiled call (torch.profiler)"}}))


if __name__ == "__main__":
    main()
