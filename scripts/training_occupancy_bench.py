#!/usr/bin/env python
"""Cost and effect of the training occupancy (toolbox/training_occupancy.py, DESIGN.md §3.21) on one GPU.

1. Refresh cost per frame (update + pack, CUDA events) at G = 128 and 256, with the hull voxel counts, and the bytes
   held per frame.
2. On the loose-hull synthetic scene after training with a training occupancy: candidates per loader batch, device
   time of loader next() plus prune_samples, and the share of rays that leave the batch, through the hulls and through
   the learned grids (the same pool, the same draws).
3. Held-out PSNR at equal steps over several seeds, with and without the training occupancy, on the loose-hull scene
   and on the example's teacher scene.

    python scripts/training_occupancy_bench.py [--out DIR] [--seeds 4] [--steps 600]

The whole report is printed as the last line (JSON); with --out it is also written to DIR/training_occupancy_bench.json.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "examples"))


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"unavailable ({e})"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def refresh_cost(G, reps=20):
    from humanrf_b200 import _lib as L
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import ellipsoid_grid

    dev = torch.device("cuda:0")
    m, _ = make_model((50,), seed=1, table_std=0.5, device=dev)
    lib = L.lib()
    out = []
    c = (np.arange(G) + 0.5) / G - 0.5
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    hulls = {"ellipsoids": ellipsoid_grid(G, 0),
             "sphere r=0.42": ((x * x + y * y + z * z <= 0.42 ** 2) * 255).astype(np.uint8)}
    for name, h in hulls.items():
        hull = torch.from_numpy(h).to(dev)
        ws = torch.empty(int(lib.hrf_training_occupancy_workspace_bytes(G)), dtype=torch.uint8, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), G, None, count.data_ptr(), ws.data_ptr(), L.stream()))
        n = int(count.item())
        ids = torch.empty(n, dtype=torch.int32, device=dev)
        L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), G, ids.data_ptr(), count.data_ptr(), ws.data_ptr(),
                                                   L.stream()))
        bound = torch.full((n,), float("inf"), device=dev)
        og = OccupanyGrid(G, 1)
        slot = og.add_grid(hull)
        field = m.native().field

        def once(k):
            L.check(lib.hrf_training_occupancy_update(C.byref(field), 20, G, ids.data_ptr(), count.data_ptr(), n, 0, k,
                                                      0.95, bound.data_ptr(), None, L.stream()))
            L.check(lib.hrf_training_occupancy_pack(ids.data_ptr(), bound.data_ptr(), n, G, 4e-4, 1e-4, slot, None,
                                                    ws.data_ptr(), L.stream()))

        for k in range(3):
            once(k)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        for k in range(reps):
            L.check(lib.hrf_training_occupancy_update(C.byref(field), 20, G, ids.data_ptr(), count.data_ptr(), n, 0, k,
                                                      0.95, bound.data_ptr(), None, L.stream()))
        ev[1].record()
        for k in range(reps):
            L.check(lib.hrf_training_occupancy_pack(ids.data_ptr(), bound.data_ptr(), n, G, 4e-4, 1e-4, slot, None,
                                                    ws.data_ptr(), L.stream()))
        ev[2].record()
        torch.cuda.synchronize()
        upd, pack = ev[0].elapsed_time(ev[1]) / reps, ev[1].elapsed_time(ev[2]) / reps
        out.append({"G": G, "hull": name, "hull_voxels": n, "update_ms": upd, "pack_ms": pack, "refresh_ms": upd + pack,
                    "evaluations_per_s": n / (upd * 1e-3), "bytes_per_frame": 8 * n + 4,
                    "shared_workspace_bytes": int(ws.numel())})
        print(json.dumps(out[-1]), flush=True)
    return out


def loader_cost(state, iters=40):
    """next() + prune_samples(is_training=True) per batch through the learned grids and through the hulls."""
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.volume_rendering import prune_samples

    dl, occ, m, ds = state["loader"], state["training_occupancy"], state["student"], state["dataset"]
    saved = dl.grid_texture_objects_cuda.clone()
    slot_frames = [int(f) for f in dl.frame_numbers_cuda.cpu().tolist()]
    for f in set(slot_frames):
        occ.evaluate(f)
    ring = OccupanyGrid(dl.occupancy_grid_resolution, 2 * dl.buffer_size)
    hull = torch.tensor([ring.add_grid(torch.from_numpy(ds.get_occupancy_grid(f)).cuda().contiguous())
                         for f in slot_frames], dtype=torch.int64, device="cuda")
    learned = torch.tensor([ring.add_grid(occ.grid(f)) for f in slot_frames], dtype=torch.int64, device="cuda")
    dl.batch_size = 4096
    res = {}
    it = iter(dl)
    dl.pause_replacing()                      # the pool stays as it is: both variants draw from the same images
    for kind, handles in (("hull", hull), ("learned", learned)) * 2:     # the second pass is the one recorded
        dl.grid_texture_objects_cuda.copy_(handles)
        torch.manual_seed(0)
        cand = rays = surv = 0
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(iters):
            b = next(it)
            cand += int(b.sample_distances.numel())
            rays += int(b.num_rays)
            prune_samples(b, m, is_training=True)
            surv += int(b.sample_distances.numel())
        ev[1].record()
        torch.cuda.synchronize()
        res[kind] = {"candidates_per_batch": cand / iters, "rays_kept_per_batch": rays / iters,
                     "survivors_per_batch": surv / iters, "next_plus_prune_ms": ev[0].elapsed_time(ev[1]) / iters}
    dl.grid_texture_objects_cuda.copy_(saved)
    res["candidate_ratio"] = res["learned"]["candidates_per_batch"] / res["hull"]["candidates_per_batch"]
    res["rays_leaving_batch"] = 1 - res["learned"]["rays_kept_per_batch"] / res["hull"]["rays_kept_per_batch"]
    res["time_ratio"] = res["learned"]["next_plus_prune_ms"] / res["hull"]["next_plus_prune_ms"]
    res["note"] = ("device time of the whole loop, including each batch's host reads of its ray and sample counts; "
                   "4096 rays per batch, trained student, pool frozen, every pooled frame's grid from the trained "
                   "model")
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for training_occupancy_bench.json (default: print only)")
    ap.add_argument("--seeds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=600)
    a = ap.parse_args()
    import train_synthetic

    report = {"device": device_info()}
    print(json.dumps(report), flush=True)
    report["refresh"] = refresh_cost(128) + refresh_cost(256)
    occ_kw = dict(warmup=256, interval=16)
    _, state = train_synthetic.main(steps=a.steps, log_every=a.steps, quiet=True, return_state=True, loose_hull=True,
                                    training_occupancy=occ_kw)
    report["loader"] = loader_cost(state)
    psnr = {}
    for scene, loose in (("loose_hull", True), ("teacher", False)):
        for variant, kw in (("hull", None), ("training_occupancy", occ_kw)):
            vals, secs = [], []
            for s in range(a.seeds):
                t0 = time.time()
                h, st = train_synthetic.main(steps=a.steps, log_every=a.steps, quiet=True, seed=s, loose_hull=loose,
                                             training_occupancy=kw, return_state=True)
                torch.cuda.synchronize()
                secs.append(time.time() - t0)
                vals.append(h[-1][1])
            psnr[f"{scene}/{variant}"] = {"psnr": vals, "mean": float(np.mean(vals)), "std": float(np.std(vals, ddof=1))
                                          if len(vals) > 1 else 0.0, "wall_s": secs}
            print(scene, variant, json.dumps(psnr[f"{scene}/{variant}"]), flush=True)
    report["psnr"] = psnr
    print(json.dumps(report), flush=True)
    if a.out is not None:
        out = Path(a.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "training_occupancy_bench.json").write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
