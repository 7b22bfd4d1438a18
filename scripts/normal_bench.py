"""Cost of the position gradient (hrf_field_position_grad) and of normal maps.
1. The kernel alone on the survivors of prune_samples on bench.py's render workload (bench model of `--segments`,
   4096 rays x 512 samples), its workspace filled once by hrf_field_backward_mlp (d_sigma = 1), timed against the
   density-only field forward (encode + sigma MLP) over the same samples: "one encode pass" as a yardstick.
2. A 1028x752 image through TileShardedRenderer.render_range_maps without and with normals.
The two arms of each pair alternate call by call in one process, L2 flushed before every timed call, CUDA events
around it; medians over `--steps` timed calls per arm after `--warmup`.  Prints one JSON line with the card's name and
power limit.
    python scripts/normal_bench.py [--segments 50] [--steps 100] [--warmup 10]
"""
import argparse
import ctypes as C
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


def ab(fa, fb, steps, warmup, flush, names):
    """Alternating timed calls of fa and fb (A first on even steps, B first on odd ones); median ms of each."""
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
    a, b = float(np.median(t[0])), float(np.median(t[1]))
    return {f"{names[0]}_ms_median": a, f"{names[1]}_ms_median": b, "ratio": b / a,
            f"{names[0]}_ms_p10_p90": [float(np.percentile(t[0], 10)), float(np.percentile(t[0], 90))],
            f"{names[1]}_ms_p10_p90": [float(np.percentile(t[1], 10)), float(np.percentile(t[1], 90))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normal_bench.py needs a CUDA device (the kernels have no CPU path)")
    from humanrf_b200 import _lib as L
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.volume_rendering import _reusable_features, prune_samples

    dev = torch.device("cuda:0")
    lib = L.lib()
    model, frames = make_model(tuple(a.segments), seed=123, device=dev)
    nat = model.native()
    b = synthetic_rays(RAYS, SPR, frames, seed=123)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2

    ib = InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                    sample_distances=g["t"].clone().view(-1, 1), ray_indices=g["ri"].clone())
    prune_samples(ib, model, is_training=False)
    saved, src, _ = _reusable_features(ib, model)
    pt, pri = ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous()
    n = int(pt.shape[0])
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], pt, pri)
    ws = torch.empty(n * 40, dtype=torch.float32, device=dev)
    ones = torch.ones(n, dtype=torch.float32, device=dev)
    L.check(lib.hrf_field_backward_mlp(C.byref(nat.field), C.byref(samples), ones.data_ptr(), None, None, saved.data_ptr(),
                                       src.data_ptr(), None, None, ws.data_ptr(), L.stream()))
    d_pos = torch.empty((n, 3), dtype=torch.float32, device=dev)
    sigma = torch.empty(n, dtype=torch.float32, device=dev)

    def position_grad():
        L.check(lib.hrf_field_position_grad(C.byref(nat.field), C.byref(samples), ws.data_ptr(), d_pos.data_ptr(), L.stream()))

    def encode():
        L.check(lib.hrf_field_forward(C.byref(nat.field), C.byref(samples), 0, 0, sigma.data_ptr(), None, None, None, None,
                                      L.stream()))

    position_grad()
    first = d_pos.clone()
    position_grad()
    assert torch.equal(first, d_pos) and torch.isfinite(d_pos).all()

    W, H, G = 1028, 752, 256
    sc = make_scene(num_images=1, width=W, height=H, G=G, portrait_every=0)
    og = OccupanyGrid(G, 1)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    cam = dict(frame_numbers=t(sc["frame_numbers"]), camera_numbers=t(sc["camera_numbers"]),
               grid_handles=torch.tensor([og.add_grid(t(sc["grids"][0]))], dtype=torch.int64, device=dev),
               landscape=t(sc["landscape"]), inverse_krs=t(sc["inverse_krs"]), camera_origins=t(sc["camera_origins"]),
               aabb=t(sc["aabb"]), G=G, width=W, height=H)
    r = TileShardedRenderer(model, og, rays_per_batch=262144)
    x, y = r.render_range_maps(cam, 0, W * H), r.render_range_maps(cam, 0, W * H, normals=True)
    assert all(torch.equal(p, q) for p, q in zip(x, y[:3]))

    workloads = {
        "position_grad": ab(encode, position_grad, a.steps, a.warmup, flush, ("density_forward", "position_grad")),
        "image": ab(lambda: r.render_range_maps(cam, 0, W * H), lambda: r.render_range_maps(cam, 0, W * H, normals=True),
                    a.steps, a.warmup, flush, ("maps", "maps_normals")),
    }
    workloads["position_grad"]["samples"] = n
    workloads["image"]["candidate_samples"] = r.last_stats.get("candidate_samples")
    print(json.dumps({
        "metric": "position_grad_ms", "value": workloads["position_grad"]["position_grad_ms_median"], "unit": "ms",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu_identity": gpu_identity(0),
        "workloads": workloads,
        "config": {"model": f"bench model, segment_sizes={tuple(a.segments)}",
                   "position_grad": f"survivors of prune_samples on {RAYS} rays x {SPR} samples; against "
                                    "hrf_field_forward mode 0 (encode + sigma MLP) on the same samples",
                   "image": f"{W}x{H} make_scene view, G={G}, 262144 rays/batch; render_range_maps without / with normals",
                   "l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events, arms alternated, medians"}}))


if __name__ == "__main__":
    main()
