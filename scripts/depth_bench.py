"""Cost of the depth map in the fused render kernel (hrf_render_fused_depth against hrf_render_fused).
Render workload of bench.py (bench model of `--segments`, 4096 rays x 512 samples) in both kernel variants: encode
(every candidate), and MLPs on the features of a prune pass (the survivors of prune_samples).  Then a 1028x752 image
through TileShardedRenderer: render_range against render_range_maps.  The two arms of each pair alternate step by step
in one process, L2 flushed before every timed call, CUDA events around it; `--steps` timed calls per arm after
`--warmup`.  Prints one JSON line: ms per call of each arm, the overhead in %, and the card's name and power limit.
    python scripts/depth_bench.py [--segments 50] [--steps 20] [--warmup 5]
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

RAYS, SPR = 4096, 512


def ab(fa, fb, steps, warmup, flush):
    """Alternating timed calls of fa and fb (A first on even steps, B first on odd ones); ms per call of each."""
    for _ in range(warmup):
        fa(), fb()
    torch.cuda.synchronize()
    t = {0: [], 1: []}
    for i in range(steps):
        for k in ((0, 1) if i % 2 == 0 else (1, 0)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            flush.zero_()
            e0.record()
            (fa if k == 0 else fb)()
            e1.record()
            torch.cuda.synchronize()
            t[k].append(e0.elapsed_time(e1))
    a, b = float(np.mean(t[0])), float(np.mean(t[1]))
    return {"plain_ms": a, "depth_ms": b, "overhead_pct": 100.0 * (b - a) / a,
            "plain_ms_median": float(np.median(t[0])), "depth_ms_median": float(np.median(t[1]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_bench.py needs a CUDA device (the render kernels have no CPU path)")
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.volume_rendering import _reusable_features, prune_samples, ray_offsets, render_fused

    dev = torch.device("cuda:0")
    model, frames = make_model(tuple(a.segments), seed=123, device=dev)
    b = synthetic_rays(RAYS, SPR, frames, seed=123)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    bg = torch.rand(RAYS, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    off = ray_offsets(g["ri"], RAYS)

    def encode(depth):
        return lambda: render_fused(model, g["o"], g["d"], g["frames"], g["t"], g["ri"], RAYS, bg, ray_offsets_dev=off,
                                    want_depth=depth)

    ib = InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                    sample_distances=g["t"].clone().view(-1, 1), ray_indices=g["ri"].clone())
    prune_samples(ib, model, is_training=False)
    reuse = _reusable_features(ib, model)
    pt, pri = ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous()

    def from_feat(depth):
        return lambda: render_fused(model, g["o"], g["d"], g["frames"], pt, pri, RAYS, bg, reuse=reuse, want_depth=depth)

    # the two arms compute the same colour and weights sum
    for f in (encode, from_feat):
        x, y = f(False)(), f(True)()
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])

    W, H, G = 1028, 752, 256
    sc = make_scene(num_images=1, width=W, height=H, G=G, portrait_every=0)
    og = OccupanyGrid(G, 1)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    cam = dict(frame_numbers=t(sc["frame_numbers"]), camera_numbers=t(sc["camera_numbers"]),
               grid_handles=torch.tensor([og.add_grid(t(sc["grids"][0]))], dtype=torch.int64, device=dev),
               landscape=t(sc["landscape"]), inverse_krs=t(sc["inverse_krs"]), camera_origins=t(sc["camera_origins"]),
               aabb=t(sc["aabb"]), G=G, width=W, height=H)
    r = TileShardedRenderer(model, og, rays_per_batch=262144)

    workloads = {
        "render_encode": ab(encode(False), encode(True), a.steps, a.warmup, flush),
        "render_from_prune_features": ab(from_feat(False), from_feat(True), a.steps, a.warmup, flush),
        "image": ab(lambda: r.render_range(cam, 0, W * H), lambda: r.render_range_maps(cam, 0, W * H), a.steps,
                    a.warmup, flush),
    }
    workloads["render_encode"]["samples"] = int(g["t"].shape[0])
    workloads["render_from_prune_features"]["samples"] = int(pt.shape[0])
    workloads["image"]["candidate_samples"] = r.last_stats.get("candidate_samples")
    print(json.dumps({
        "metric": "depth_overhead_pct", "value": workloads["render_encode"]["overhead_pct"], "unit": "%",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu_identity": gpu_identity(0),
        "workloads": workloads,
        "config": {"model": f"bench model, segment_sizes={tuple(a.segments)}",
                   "render": f"{RAYS} rays x {SPR} samples, background per ray; hrf_render_fused vs hrf_render_fused_depth",
                   "image": f"{W}x{H} make_scene view, G={G}, 262144 rays/batch; render_range vs render_range_maps",
                   "l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events, arms alternated",
                   "value": "encode variant, (depth - plain) / plain"}}))


if __name__ == "__main__":
    main()
