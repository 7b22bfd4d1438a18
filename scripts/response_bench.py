"""Cost of the per-camera colour response in the fused train step (FusedTrainer(camera_responses=...), DESIGN.md §3.17).
FusedTrainer.step on bench.py's train workload (bench model of `--segments`, 4096 rays x 512 samples, the initial model's
own render as the target, lr 1e-6, reuse="feat+grid"), its rays spread over 8 cameras, in three arms: no responses,
responses, responses and poses.  The three trainers own separate copies of the model and take turns call by call (the
order rotates every step); L2 flushed before every timed call, CUDA events around it, median and p10-p90 over `--steps`
calls per arm after `--warmup`.  Also hrf_train_loss_response and hrf_camera_response_step alone at 4096 and 300000
rays over 8 and 160 cameras.  Prints one JSON line with the card's name and power limit.
    python scripts/response_bench.py [--segments 50] [--steps 60] [--warmup 5] [--reps 200]
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
from pose_bench import per_launch_ms, tables  # noqa: E402

RAYS, SPR = 4096, 512
ARMS = ("no_responses", "responses", "responses_and_poses")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("response_bench.py needs a CUDA device (the kernels have no CPU path)")
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.training import FusedTrainer
    from humanrf_b200.volume_rendering import render

    dev = torch.device("cuda:0")
    out = {"gpu": gpu_identity(0), "workload": f"bench.py train: segments {a.segments}, {RAYS} rays x {SPR} samples, 8 cameras"}
    b = synthetic_rays(RAYS, SPR, list(range(15, 15 + sum(a.segments))), seed=123)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    cams = (b["cams"] % 8).to(dev).contiguous()
    trainers = []
    for arm in ARMS:
        model, frames = make_model(tuple(a.segments), seed=123, device=dev)
        if not trainers:        # the target: the initial model's own render (bench.py's stationary workload)
            with torch.no_grad():
                r = render(InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                                      sample_distances=g["t"].view(-1, 1), ray_indices=g["ri"]), model, None, is_training=False)
                w = r.weights_sum.clamp(min=1e-6)
                g["rgba"] = torch.cat((r.color / w, r.weights_sum), dim=1).clamp(0, 1).contiguous()
        ld = tables(8, list(range(8)), dev)
        resp = CameraResponses(ld, lr=1e-6) if arm != "no_responses" else None
        cp = CameraPoses(ld, lr=1e-6) if arm == "responses_and_poses" else None
        trainers.append(FusedTrainer(model, lr=1e-6, reuse="feat+grid", camera_poses=cp, camera_responses=resp))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    steps = [lambda tr=tr: tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], RAYS, cameras=cams)
             for tr in trainers]
    for _ in range(a.warmup):
        for f in steps:
            f()
    torch.cuda.synchronize()
    t = {k: [] for k in range(len(ARMS))}
    for i in range(a.steps):
        for j in range(len(ARMS)):
            k = (i + j) % len(ARMS)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            flush.zero_()
            e0.record()
            steps[k]()
            e1.record()
            torch.cuda.synchronize()
            t[k].append(e0.elapsed_time(e1))
    step = {}
    for k, name in enumerate(ARMS):
        step[f"{name}_ms_median"] = float(np.median(t[k]))
        step[f"{name}_ms_p10_p90"] = [float(np.percentile(t[k], 10)), float(np.percentile(t[k], 90))]
    step["responses_overhead_ms"] = step["responses_ms_median"] - step["no_responses_ms_median"]
    out["train_step"] = step
    resp = trainers[1].camera_responses
    assert int(resp.ray_count.sum()) == RAYS and int(resp.error[0]) == 0

    kern = {}
    for C_ in (8, 160):
        cr = CameraResponses(tables(C_, [0], dev))
        cr.params.normal_(0.0, 0.05)
        cr._write_table()
        for R in (4096, 300000):
            color, wsum = torch.rand(R, 3, device=dev), torch.rand(R, device=dev)
            rgba, bg = torch.rand(R, 4, device=dev), torch.rand(R, 3, device=dev)
            c = torch.randint(0, C_, (R,), dtype=torch.int32, device=dev)
            dc, dw, loss = torch.empty(R, 3, device=dev), torch.empty(R, device=dev), torch.zeros(1, device=dev)
            kern[f"loss_response_R{R}_C{C_}_ms"] = per_launch_ms(
                lambda: cr.loss(color, wsum, rgba, bg, c, R, 0.01, 1e-3, None, dc, dw, loss), a.reps)
        cr.ray_count.fill_(1)
        cr.response_grad.normal_()
        kern[f"response_step_C{C_}_ms"] = per_launch_ms(lambda: cr.step(0), a.reps)
    out["kernels"] = kern
    print(json.dumps(out))


if __name__ == "__main__":
    main()
