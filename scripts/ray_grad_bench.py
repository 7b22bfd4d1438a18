"""Cost of the gradients with respect to the rays (hrf_field_backward_mlp_dirs, hrf_ray_gradients).
1. On the survivors of prune_samples on bench.py's render workload (bench model of `--segments`, 4096 rays x 512
   samples): the MLP backward without and with d_directions, and hrf_ray_gradients against hrf_field_position_grad on
   the same samples.
2. render() forward + backward of that batch with origins, directions and distances requiring grad, trainable model
   (scatter included) against frozen model (no scatter).
3. One refine_camera iteration at 16384 rays of a 256x192 synthetic camera: (time of 11 iterations - time of 1) / 10.
Pairs alternate call by call in one process, L2 flushed before every timed call, CUDA events around it; medians over
`--steps` timed calls per arm after `--warmup`.  Prints one JSON line with the card's name and power limit.
    python scripts/ray_grad_bench.py [--segments 50] [--steps 50] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bake_bench import gpu_identity  # noqa: E402
from normal_bench import ab  # noqa: E402

RAYS, SPR = 4096, 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ray_grad_bench.py needs a CUDA device (the kernels have no CPU path)")
    from humanrf_b200 import _lib as L
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.camera_refinement import refine_camera
    from humanrf_b200.volume_rendering import _reusable_features, prune_samples, render

    dev = torch.device("cuda:0")
    lib = L.lib()
    model, frames = make_model(tuple(a.segments), seed=123, device=dev)
    nat = model.native()
    b = synthetic_rays(RAYS, SPR, frames, seed=123)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2

    def batch():
        ib = InputBatch(ray_origins=g["o"].clone(), ray_directions=g["d"].clone(), frame_numbers=g["frames"].view(-1, 1),
                        unique_frame_numbers=torch.unique(g["frames"]).view(-1, 1),
                        sample_distances=g["t"].clone().view(-1, 1), ray_indices=g["ri"].clone())
        prune_samples(ib, model, is_training=False)
        return ib

    ib = batch()
    saved, src, kept_off = _reusable_features(ib, model)
    pt, pri = ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous()
    n = int(pt.shape[0])
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], pt, pri)
    ws = torch.empty(n * 40, dtype=torch.float32, device=dev)
    ones, ones3 = torch.ones(n, device=dev), torch.ones((n, 3), device=dev)
    d_mlp = torch.zeros(model.mlp_grad_elems, device=dev)
    d_dir = torch.empty((n, 3), device=dev)
    d_pos = torch.empty((n, 3), device=dev)
    g_o, g_d, g_t = torch.empty((RAYS, 3), device=dev), torch.empty((RAYS, 3), device=dev), torch.empty(n, device=dev)
    args = lambda: (C.byref(nat.field), C.byref(samples), ones.data_ptr(), ones3.data_ptr(), None, saved.data_ptr(),  # noqa: E731
                    src.data_ptr(), d_mlp.data_ptr(), None)

    def mlp():
        L.check(lib.hrf_field_backward_mlp(*args(), ws.data_ptr(), L.stream()))

    def mlp_dirs():
        L.check(lib.hrf_field_backward_mlp_dirs(*args(), d_dir.data_ptr(), ws.data_ptr(), L.stream()))

    def position_grad():
        L.check(lib.hrf_field_position_grad(C.byref(nat.field), C.byref(samples), ws.data_ptr(), d_pos.data_ptr(), L.stream()))

    def ray_grads():
        L.check(lib.hrf_ray_gradients(d_pos.data_ptr(), d_dir.data_ptr(), pt.data_ptr(), g["d"].data_ptr(),
                                      kept_off.data_ptr(), RAYS, g_o.data_ptr(), g_d.data_ptr(), g_t.data_ptr(), L.stream()))

    mlp_dirs(), position_grad(), ray_grads()
    first = g_d.clone()
    ray_grads()
    assert torch.equal(first, g_d) and torch.isfinite(g_d).all()

    def render_bwd(frozen):
        def run():
            for q in model.parameters():
                q.requires_grad_(not frozen)
                q.grad = None
            x = batch()
            x.ray_origins.requires_grad_(True)
            x.ray_directions.requires_grad_(True)
            x.sample_distances.requires_grad_(True)
            out = render(x, model, torch.zeros(3, device=dev), is_training=False)
            (out.color.sum() + out.weights_sum.sum()).backward()
        return run

    workloads = {
        "mlp_backward": ab(mlp, mlp_dirs, a.steps, a.warmup, flush, ("mlp_backward", "mlp_backward_dirs")),
        "ray_gradients": ab(position_grad, ray_grads, a.steps, a.warmup, flush, ("position_grad", "ray_gradients")),
        "render_backward": ab(render_bwd(False), render_bwd(True), a.steps, a.warmup, flush,
                              ("prune_render_fwd_bwd_trainable", "prune_render_fwd_bwd_frozen")),
    }
    for q in model.parameters():
        q.requires_grad_(True)
        q.grad = None
    workloads["mlp_backward"]["samples"] = n
    workloads["ray_gradients"]["rays"] = RAYS

    ds = SyntheticDataset(width=256, height=192, G=64)
    loader = DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192, camera_numbers=(0,),
                frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])
    teacher, _ = make_model((6,), seed=7, table_std=1.0, device=dev)

    def refine(k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        refine_camera(teacher, loader, 0, [16], iterations=k, rays_per_step=16384)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    refine(2)
    per = [(refine(11) - refine(1)) / 10 * 1e3 for _ in range(max(3, a.steps // 10))]
    workloads["refine_iteration"] = {"ms_median": float(np.median(per)), "rays": 16384, "image": "256x192"}
    print(json.dumps({
        "metric": "mlp_backward_dirs_ms", "value": workloads["mlp_backward"]["mlp_backward_dirs_ms_median"], "unit": "ms",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu_identity": gpu_identity(0),
        "workloads": workloads,
        "config": {"model": f"bench model, segment_sizes={tuple(a.segments)}",
                   "samples": f"survivors of prune_samples on {RAYS} rays x {SPR} samples",
                   "render_backward": "prune_samples + render() + backward, origins / directions / distances requiring grad",
                   "refine_iteration": "(refine_camera 11 iterations - 1 iteration) / 10, 16384 rays of a 256x192 view",
                   "l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events, arms alternated, medians"}}))


if __name__ == "__main__":
    main()
