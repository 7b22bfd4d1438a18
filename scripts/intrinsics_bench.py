"""Cost of intrinsics refinement in the fused train step (CameraPoses(intrinsics=True), DESIGN.md §3.15).
1. FusedTrainer.step on bench.py's train workload (as scripts/pose_bench.py: bench model of `--segments`, 4096 rays x
   512 samples, the initial model's own render as the target, lr 1e-6, reuse="feat+grid", rays over 8 cameras) in three
   configurations: no camera_poses, poses only, poses plus intrinsics.  The three trainers own separate copies of the
   model and alternate call by call; L2 flushed before every timed call, CUDA events around it; median and p10-p90 over
   `--steps` calls per arm after `--warmup`.
2. Each new kernel alone, CUDA events around `--reps` back-to-back launches, beside the pose-only kernels on the same
   inputs: hrf_camera_calib_grad at 4096, 65536 and 300000 rays over 8 and 160 cameras, hrf_camera_calib_step with
   160 cameras and 200 pool slots.
Prints one JSON line with the card's name and power limit.
    python scripts/intrinsics_bench.py [--segments 50] [--steps 50] [--warmup 5] [--reps 200]
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
from pose_bench import RAYS, SPR, per_launch_ms, tables  # noqa: E402


def calib_tables(num_cameras, slot_cameras, dev):
    """pose_bench's tables plus the cameras intrinsics refinement reads its base focal lengths and rotations from
    (synthetic_scene.SyntheticDataset's ring; the timing does not depend on their values)."""
    from humanrf_b200.synthetic_scene import SyntheticDataset

    t = tables(num_cameras, slot_cameras, dev)
    t.cameras = SyntheticDataset(num_cameras=num_cameras, width=96, height=72).cameras
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("intrinsics_bench.py needs a CUDA device (the kernels have no CPU path)")
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
    arms = ("no_poses", "poses", "poses_intrinsics")
    trainers = []
    for arm in arms:
        model, frames = make_model(tuple(a.segments), seed=123, device=dev)
        if not trainers:        # the target: the initial model's own render (bench.py's stationary workload)
            with torch.no_grad():
                r = render(InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                                      sample_distances=g["t"].view(-1, 1), ray_indices=g["ri"]), model, None, is_training=False)
                w = r.weights_sum.clamp(min=1e-6)
                g["rgba"] = torch.cat((r.color / w, r.weights_sum), dim=1).clamp(0, 1).contiguous()
        cp = None
        if arm != "no_poses":
            cp = CameraPoses(calib_tables(8, list(range(8)), dev), lr=1e-6, intrinsics=arm == "poses_intrinsics",
                             intrinsics_lr=1e-6)
        trainers.append(FusedTrainer(model, lr=1e-6, reuse="feat+grid", camera_poses=cp))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    times = {arm: [] for arm in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(a.warmup + a.steps):
        for arm, tr in zip(arms, trainers):
            flush.zero_()
            torch.cuda.synchronize()
            e0.record()
            tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], RAYS, cameras=cams)
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times[arm].append(e0.elapsed_time(e1))
    out["train_step_ms"] = {arm: {"median": float(np.median(v)), "p10": float(np.percentile(v, 10)),
                                  "p90": float(np.percentile(v, 90))} for arm, v in times.items()}
    for tr in trainers[1:]:
        assert int(tr.camera_poses.ray_count.sum()) == RAYS and int(tr.camera_poses.error[0]) == 0

    kern = {}
    rng = np.random.default_rng(0)
    for C_ in (8, 160):
        pose = CameraPoses(tables(C_, list(range(min(C_, 200))), dev))
        calib = CameraPoses(calib_tables(C_, list(range(min(C_, 200))), dev), intrinsics=True)
        w = torch.from_numpy(rng.standard_normal((C_, 3)) * 0.01)
        pose.omega.copy_(w)
        calib.omega.copy_(w)
        for R in (4096, 65536, 300000):
            d = torch.nn.functional.normalize(torch.randn(R, 3, device=dev), dim=1).contiguous()
            g_o, g_d = torch.randn(R, 3, device=dev), torch.randn(R, 3, device=dev)
            c = torch.randint(0, C_, (R,), dtype=torch.int32, device=dev)
            kern[f"pose_grad_R{R}_C{C_}_ms"] = per_launch_ms(lambda: pose.accumulate(g_o, g_d, d, c, R), a.reps)
            kern[f"calib_grad_R{R}_C{C_}_ms"] = per_launch_ms(lambda: calib.accumulate(g_o, g_d, d, c, R), a.reps)
    for name, intr in (("pose_step", False), ("calib_step", True)):
        cp = CameraPoses(calib_tables(160, [i % 160 for i in range(200)], dev), intrinsics=intr)
        cp.ray_count.fill_(1)
        cp.pose_grad.normal_()
        kern[f"{name}_C160_B200_ms"] = per_launch_ms(lambda: cp.step(0), a.reps)
    out["kernels"] = kern
    print(json.dumps(out))


if __name__ == "__main__":
    main()
