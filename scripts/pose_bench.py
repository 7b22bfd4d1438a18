"""Cost of camera pose refinement in the fused train step (FusedTrainer(camera_poses=...), DESIGN.md §3.14).
1. FusedTrainer.step on bench.py's train workload (bench model of `--segments`, 4096 rays x 512 samples, the initial
   model's own render as the target, lr 1e-6, reuse="feat+grid"), its rays spread over 8 cameras: without and with
   camera_poses.  The two trainers own separate copies of the model and alternate call by call; L2 flushed before every
   timed call, CUDA events around it, medians over `--steps` calls per arm after `--warmup`.
2. Each new kernel alone, CUDA events around `--reps` back-to-back launches: hrf_camera_pose_grad at 4096, 65536 and
   300000 rays over 8 and 160 cameras, hrf_camera_pose_step with 160 cameras and 200 pool slots.
Prints one JSON line with the card's name and power limit.
    python scripts/pose_bench.py [--segments 50] [--steps 50] [--warmup 5] [--reps 200]
"""
import argparse
import json
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bake_bench import gpu_identity  # noqa: E402
from normal_bench import ab  # noqa: E402

RAYS, SPR = 4096, 512


def tables(num_cameras, slot_cameras, dev):
    """The camera and pool-slot tables a DataLoader holds, for cameras on a ring (synthetic_scene.make_scene)."""
    from humanrf_b200.synthetic_scene import make_scene

    sc = make_scene(num_images=num_cameras, width=96, height=72, portrait_every=0)
    B = len(slot_cameras)
    return SimpleNamespace(all_inverse_krs=torch.from_numpy(sc["inverse_krs"]).to(dev).contiguous(),
                           all_camera_origins=torch.from_numpy(sc["camera_origins"]).to(dev).contiguous(),
                           camera_numbers=tuple(range(num_cameras)),
                           inverse_krs_cuda=torch.zeros((B, 3, 3), device=dev),
                           camera_origins_cuda=torch.zeros((B, 3), device=dev),
                           camera_numbers_cuda=torch.tensor(slot_cameras, dtype=torch.int32, device=dev))


def per_launch_ms(fn, reps):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_bench.py needs a CUDA device (the kernels have no CPU path)")
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.training import FusedTrainer
    from humanrf_b200.volume_rendering import render

    dev = torch.device("cuda:0")
    out = {"gpu": gpu_identity(0), "workload": f"bench.py train: segments {a.segments}, {RAYS} rays x {SPR} samples, 8 cameras"}
    b = synthetic_rays(RAYS, SPR, list(range(15, 15 + sum(a.segments))), seed=123)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    cams = (b["cams"] % 8).to(dev).contiguous()
    trainers = []
    for poses in (False, True):
        model, frames = make_model(tuple(a.segments), seed=123, device=dev)
        if not trainers:        # the target: the initial model's own render (bench.py's stationary workload)
            with torch.no_grad():
                r = render(InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                                      sample_distances=g["t"].view(-1, 1), ray_indices=g["ri"]), model, None, is_training=False)
                w = r.weights_sum.clamp(min=1e-6)
                g["rgba"] = torch.cat((r.color / w, r.weights_sum), dim=1).clamp(0, 1).contiguous()
        cp = CameraPoses(tables(8, list(range(8)), dev), lr=1e-6) if poses else None
        trainers.append(FusedTrainer(model, lr=1e-6, reuse="feat+grid", camera_poses=cp))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    step = [lambda tr=tr: tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], RAYS, cameras=cams)
            for tr in trainers]
    out["train_step"] = ab(step[0], step[1], a.steps, a.warmup, flush, ("without_poses", "with_poses"))
    out["survivors"] = int(trainers[1].last["samples"])
    poses = trainers[1].camera_poses
    assert int(poses.ray_count.sum()) == RAYS and int(poses.error[0]) == 0

    kern = {}
    rng = np.random.default_rng(0)
    for C_ in (8, 160):
        cp = CameraPoses(tables(C_, list(range(min(C_, 200))), dev))
        cp.omega.copy_(torch.from_numpy(rng.standard_normal((C_, 3)) * 0.01))
        for R in (4096, 65536, 300000):
            d = torch.nn.functional.normalize(torch.randn(R, 3, device=dev), dim=1).contiguous()
            g_o, g_d = torch.randn(R, 3, device=dev), torch.randn(R, 3, device=dev)
            c = torch.randint(0, C_, (R,), dtype=torch.int32, device=dev)
            kern[f"pose_grad_R{R}_C{C_}_ms"] = per_launch_ms(lambda: cp.accumulate(g_o, g_d, d, c, R), a.reps)
    cp = CameraPoses(tables(160, [i % 160 for i in range(200)], dev))
    cp.ray_count.fill_(1)
    cp.pose_grad.normal_()
    kern["pose_step_C160_B200_ms"] = per_launch_ms(lambda: cp.step(0), a.reps)
    out["kernels"] = kern
    print(json.dumps(out))


if __name__ == "__main__":
    main()
