"""Mesh rasteriser and depth score benchmark (toolbox/mesh_depth: hrf_rasterize_mesh, hrf_depth_metrics).  Workload: the
bench model's G = 256 hull mesh of frame 0 (geometry_bench.py's, about 2.1 M faces), seen by the first make_scene camera
(the bench scene's units, distance 2 from the centre), at 1028x752 and 4112x3008.  Per view, `--steps` calls of each
after `--warmup`, L2 flushed before each, CUDA events around each, medians:
  - rasterize_mesh (z, mask, face; no hits), with faces / s and fragments / s (fragments = sum of hits of one call with
    hits);
  - depth_scores of that view against a perturbed copy, with its bytes (two float32 z and two uint8 masks per pixel)
    against 3.35 TB/s;
  - TileShardedRenderer.render_range_maps of the same view (what render_depth_map renders) as the yardstick.
Prints one JSON line with the card's name and power limit.
    python scripts/raster_bench.py [--steps 10] [--warmup 3]
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
from geometry_bench import meshes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


class Camera:
    """make_scene's camera 0 as CameraData fields: RDF, looking at the origin, focal 1.773863, centred principal point."""

    def __init__(self, width, height):
        from scipy.spatial.transform import Rotation

        rng = np.random.default_rng(0)                      # make_scene(seed=0)'s first draw is camera 0's height
        a = 0.3
        pos = np.array([2.0 * np.cos(a), rng.uniform(-0.4, 0.4), 2.0 * np.sin(a)])
        fwd = -pos / np.linalg.norm(pos)
        right = np.cross(fwd, [0.0, -1.0, 0.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        self.width, self.height = width, height
        self.rotation_axisangle = Rotation.from_matrix(np.stack([right, down, fwd], 1)).as_rotvec()
        self.translation = pos
        self.focal_length = np.array([1.773863, 1.773863 * width / height])
        self.principal_point = np.array([0.5, 0.5])


def timed(fn, steps, warmup, flush):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        flush.zero_()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    return float(np.median(t)), float(np.min(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raster_bench.py needs a CUDA device (the rasteriser has no CPU path)")
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.mesh_depth import depth_scores, rasterize_mesh

    dev = torch.device("cuda:0")
    mesh, _ = meshes(dev)
    nf = int(mesh.faces.shape[0])
    model, _ = make_model((50,), seed=123, device=dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    views = {}
    for W, H in ((1028, 752), (4112, 3008)):
        cam = Camera(W, H)
        r = rasterize_mesh(mesh, cam, hits=True)
        fragments = int(r.hits.sum())
        covered = int((r.mask != 0).sum())
        assert int(r.error[0]) == 0 and int(r.skipped[0]) == 0
        raster_ms, raster_min = timed(lambda: rasterize_mesh(mesh, cam), a.steps, a.warmup, flush)
        pred = (r.z + 1e-3 * torch.randn(r.z.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(1)))
        pred = torch.where(r.mask != 0, pred, torch.zeros_like(pred)).contiguous()
        metrics_ms, metrics_min = timed(lambda: depth_scores(pred, r.mask, r.z, r.mask), a.steps, a.warmup, flush)
        nbytes = W * H * (4 + 1 + 4 + 1)
        sc = make_scene(num_images=1, width=W, height=H, G=256, portrait_every=0)
        og = OccupanyGrid(256, 1)
        tables = dict(frame_numbers=t(sc["frame_numbers"]), camera_numbers=t(sc["camera_numbers"]),
                      grid_handles=torch.tensor([og.add_grid(t(sc["grids"][0]))], dtype=torch.int64, device=dev),
                      landscape=t(sc["landscape"]), inverse_krs=t(sc["inverse_krs"]),
                      camera_origins=t(sc["camera_origins"]), aabb=t(sc["aabb"]), G=256, width=W, height=H)
        rend = TileShardedRenderer(model, og, rays_per_batch=262144)
        render_ms, _ = timed(lambda: rend.render_range_maps(tables, 0, W * H), max(a.steps // 2, 2), 1, flush)
        views[f"{W}x{H}"] = {
            "raster_ms": raster_ms, "raster_ms_min": raster_min, "faces_per_s": nf / (raster_ms * 1e-3),
            "fragments": fragments, "covered_pixels": covered, "fragments_per_s": fragments / (raster_ms * 1e-3),
            "depth_metrics_ms": metrics_ms, "depth_metrics_ms_min": metrics_min, "depth_metrics_bytes": nbytes,
            "depth_metrics_hbm_share": nbytes / HBM_BYTES_PER_S / (metrics_ms * 1e-3),
            "render_depth_map_ms": render_ms}
        del og, rend
    print(json.dumps({
        "metric": "raster_ms_1028x752", "value": views["1028x752"]["raster_ms"], "unit": "ms", "higher_is_better": False,
        "steps": a.steps, "warmup": a.warmup, "gpu": gpu_identity(0), "faces": nf, "views": views,
        "config": {"mesh": "bench model segment_sizes=(50,), make_scene hull G=256, frame 0, median level",
                   "camera": "make_scene camera 0 (distance 2, focal 1.773863), landscape",
                   "l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events, median",
                   "render_depth_map": "TileShardedRenderer.render_range_maps of the same view, 262144 rays/batch",
                   "hbm": "depth_metrics bytes / 3.35 TB/s over its time"}}))


if __name__ == "__main__":
    main()
