"""Cost of camera refinement in data-parallel training (DESIGN.md §3.16).
1. The step entry alone on one GPU: W ranks simulated on one device (W gradient records, every camera touched), CUDA
   events around `--reps` back-to-back launches, at W in {1, 2, 8} x C in {8, 160, 1024} with 200 pool slots, beside the
   single-rank hrf_camera_pose_step and hrf_camera_calib_step.  The records are local here; over NVLink
   (exchange="p2p") the W - 1 peers' records are remote reads.
2. With two or more GPUs visible: FusedTrainer.step on bench.py's train workload (bench model of `--segments`, 4096 rays x
   512 samples per rank, the initial model's own render as the target, lr 1e-6, reuse="feat+grid", rays over 8
   cameras) at world 2 and at the visible GPU count, one process per GPU, for exchanges p2p and nccl.  Per exchange the
   three configurations (no poses, poses, poses with intrinsics) own separate copies of the model and alternate call by
   call; L2 flushed before every timed call, CUDA events around it; rank 0's median and p10-p90 over `--steps` calls
   after `--warmup`.  With fewer GPUs these rows are reported as not measured.
Prints one JSON line with the card's name and power limit.
    python scripts/pose_dp_bench.py [--reps 500] [--segments 50] [--steps 30] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bake_bench import gpu_identity  # noqa: E402
from pose_bench import per_launch_ms  # noqa: E402


def loader(num_cameras, num_slots, dev, seed=0):
    rng = np.random.default_rng(seed)
    cams = [SimpleNamespace(width=96, height=72, focal_length=rng.uniform(0.8, 1.2, 2),
                            principal_point=rng.uniform(0.4, 0.6, 2), rotation_axisangle=rng.standard_normal(3))
            for _ in range(num_cameras)]
    ikr = (np.eye(3) * 1e-3 + rng.standard_normal((num_cameras, 3, 3)) * 2e-4).astype(np.float32)
    return SimpleNamespace(all_inverse_krs=torch.from_numpy(ikr).to(dev),
                           all_camera_origins=torch.from_numpy(rng.standard_normal((num_cameras, 3)).astype(np.float32)).to(dev),
                           camera_numbers=tuple(range(num_cameras)), cameras=cams,
                           inverse_krs_cuda=torch.zeros((num_slots, 3, 3), device=dev),
                           camera_origins_cuda=torch.zeros((num_slots, 3), device=dev),
                           camera_numbers_cuda=torch.from_numpy(rng.integers(0, num_cameras, num_slots).astype(np.int32)).to(dev))


RAYS, SPR = 4096, 512
CONFIGS = ("none", "poses", "poses+intrinsics")


def _train_rank(rank, world, port, segments, steps, warmup, q):
    """One rank of the FusedTrainer.step measurement; rank 0 puts its rows on `q`."""
    import torch.distributed as dist

    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.training import FusedTrainer
    from humanrf_b200.volume_rendering import render

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    if world > 1:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    b = synthetic_rays(RAYS, SPR, list(range(15, 15 + sum(segments))), seed=123 + rank)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    cams = (b["cams"] % 8).to(dev).contiguous()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    rows = []
    for exchange in ("p2p", "nccl"):
        trainers = []
        for mode in CONFIGS:
            model, _ = make_model(tuple(segments), seed=123, device=dev)
            if "rgba" not in g:     # the target: the initial model's own render (bench.py's stationary workload)
                with torch.no_grad():
                    r = render(InputBatch(ray_origins=g["o"], ray_directions=g["d"], frame_numbers=g["frames"].view(-1, 1),
                                          sample_distances=g["t"].view(-1, 1), ray_indices=g["ri"]), model, None,
                               is_training=False)
                    w = r.weights_sum.clamp(min=1e-6)
                    g["rgba"] = torch.cat((r.color / w, r.weights_sum), dim=1).clamp(0, 1).contiguous()
            cp = None
            if mode != "none":
                cp = CameraPoses(loader(8, 8, dev), lr=1e-6, intrinsics=mode == "poses+intrinsics", world_size=world)
            trainers.append(FusedTrainer(model, lr=1e-6, reuse="feat+grid", world_size=world, exchange=exchange,
                                         camera_poses=cp))
        times = [[] for _ in trainers]
        for i in range(warmup + steps):
            order = range(len(trainers)) if i % 2 == 0 else reversed(range(len(trainers)))
            for k in order:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                flush.zero_()
                e0.record()
                trainers[k].step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], RAYS, cameras=cams)
                e1.record()
                torch.cuda.synchronize()
                if i >= warmup:
                    times[k].append(e0.elapsed_time(e1))
        for tr, mode, t in zip(trainers, CONFIGS, times):
            if tr.camera_poses is not None:
                tr.camera_poses.check()
            rows.append({"exchange": exchange if world > 1 else "local", "world": world, "poses": mode,
                         "step_ms_median": float(np.median(t)),
                         "step_ms_p10_p90": [float(np.percentile(t, 10)), float(np.percentile(t, 90))]})
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        for tr in trainers:
            tr.close()
        del trainers
    if rank == 0:
        q.put(rows)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def train_rows(world, segments, steps, warmup):
    """FusedTrainer.step rows at `world` ranks: one process per GPU (world 1 runs in this process)."""
    import queue as queue_mod

    import torch.multiprocessing as mp

    if world == 1:
        q = queue_mod.Queue()
        _train_rank(0, 1, 0, segments, steps, warmup, q)
        return q.get()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000 + world
    procs = [ctx.Process(target=_train_rank, args=(r, world, port, segments, steps, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    rows = q.get(timeout=1800)
    for p in procs:
        p.join(timeout=300)
        if p.exitcode != 0:
            raise RuntimeError(f"a rank of the world-{world} measurement exited with {p.exitcode}")
    return rows


def main():
    from humanrf_b200 import _lib as L
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=500)
    ap.add_argument("--segments", type=int, nargs="+", default=[50])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_dp_bench needs a GPU")
    dev = torch.device("cuda", 0)
    lib = L.lib()
    rows = []
    for calib in (False, True):
        for C_ in (8, 160, 1024):
            p = CameraPoses(loader(C_, 200, dev), lr=1e-9, final_lr_ratio=1.0, fixed_cameras=(), intrinsics=calib)
            p.pose_grad.copy_(torch.randn(C_, 6, device=dev) * 1e-3)
            if calib:
                p.intrinsics_grad.copy_(torch.randn(C_, 4, device=dev) * 1e-3)
            p.ray_count.fill_(10)
            single = lambda: p.step(0)        # noqa: E731
            rows.append({"entry": "hrf_camera_calib_step" if calib else "hrf_camera_pose_step", "world": 1,
                         "cameras": C_, "us": 1e3 * per_launch_ms(single, args.reps)})
            for W in (1, 2, 8):
                records = [p.record] + [p.record.clone() for _ in range(W - 1)]
                rec = L.CameraGradRecords()
                for r, t in enumerate(records):
                    rec.record[r] = t.data_ptr()
                rec.world, rec.rank = W, 0
                if calib:
                    fn = lambda: L.check(lib.hrf_camera_calib_step_ranks(   # noqa: E731
                        C.byref(p._desc), C.byref(p._idesc), C.byref(rec), p.error.data_ptr(), 1e-9, 1e-9, 0.9, 0.99,
                        1e-15, L.stream()))
                else:
                    fn = lambda: L.check(lib.hrf_camera_pose_step_ranks(    # noqa: E731
                        C.byref(p._desc), C.byref(rec), p.error.data_ptr(), 1e-9, 0.9, 0.99, 1e-15, L.stream()))
                rows.append({"entry": "hrf_camera_calib_step_ranks" if calib else "hrf_camera_pose_step_ranks",
                             "world": W, "cameras": C_, "record_bytes": int(p.record.numel()),
                             "us": 1e3 * per_launch_ms(fn, args.reps)})
            p.check()
    for r in rows:
        print(f"{r['entry']:30s} W={r['world']} C={r['cameras']:5d}  {r['us']:8.2f} us/launch")
    n = torch.cuda.device_count()
    if n >= 2:
        train = [row for world in sorted({2, n}) for row in train_rows(world, args.segments, args.steps, args.warmup)]
    else:
        train = [{"exchange": ex, "world": 2, "poses": mode, "step_ms": f"not measured ({n} GPU visible)"}
                 for ex in ("p2p", "nccl") for mode in CONFIGS]
    for r in train:
        print(f"FusedTrainer.step {r['exchange']:5s} world={r['world']} {r['poses']:17s} "
              + (f"{r['step_ms_median']:.3f} ms [{r['step_ms_p10_p90'][0]:.3f}-{r['step_ms_p10_p90'][1]:.3f}]"
                 if "step_ms_median" in r else r["step_ms"]))
    print(json.dumps({"gpu": gpu_identity(0), "gpus_visible": torch.cuda.device_count(), "reps": args.reps,
                      "step_entry": rows, "train_step": train}))


if __name__ == "__main__":
    main()
