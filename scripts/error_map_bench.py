#!/usr/bin/env python
"""The error map (DESIGN.md §3.20) on the GPU.  Cost: accumulate + update + draw per step at the bench's batch for pools
of 64 x 96x72, 200 x 1022x750 and 200 x 4088x3000 pixels in 16- and 32-pixel tiles, one slot reset, the fused train
step with and without a map on a fixed batch, and the loader's next() with and without a map on a pool that reloads a
slot every batch.  Quality (--quality): held-out PSNR of examples/train_synthetic.py's teacher scene, uniform rays
against the error map, at equal steps and at an equal sample budget, per seed.  Prints one JSON line per measurement,
with the card's name and power limit.

    python scripts/error_map_bench.py [--rays 4096] [--iters 200] [--quality --seeds 0 1 2 --steps 200]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from humanrf_b200 import _lib as L  # noqa: E402


def _card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(), "unknown"
    return {"gpu": name, "power_limit": power}


def _timed(fn, iters: int) -> float:
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def map_cost(B: int, W: int, H: int, T: int, R: int, iters: int) -> dict:
    dev = torch.device("cuda:0")
    lib = L.lib()
    ls = torch.ones(B, dtype=torch.bool, device=dev)
    ls[1::3] = False
    g = L.ErrorMapGeometry()
    g.landscape_modes, g.num_slots, g.image_width, g.image_height, g.tile = ls.data_ptr(), B, W, H, T
    n = int(lib.hrf_error_map_num_tiles(C.byref(g), 1.0))
    ema = torch.ones(n, dtype=torch.float32, device=dev)
    s = torch.zeros(n, dtype=torch.int64, device=dev)
    c = torch.zeros(n, dtype=torch.int32, device=dev)
    cdf = torch.empty(n, dtype=torch.int64, device=dev)
    ws = torch.empty(int(lib.hrf_error_map_workspace_bytes(n)), dtype=torch.uint8, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    color, bg = torch.rand(R, 3, device=dev), torch.rand(R, 3, device=dev)
    rgba = torch.rand(R, 4, device=dev)
    pixels = torch.empty(R, dtype=torch.int64, device=dev)
    counter = [0]

    def accumulate():
        L.check(lib.hrf_error_map_accumulate(color.data_ptr(), None, rgba.data_ptr(), bg.data_ptr(), pixels.data_ptr(),
                                             R, None, None, 0, 0.01, C.byref(g), s.data_ptr(), c.data_ptr(),
                                             err.data_ptr(), L.stream()))

    def update():
        L.check(lib.hrf_error_map_update(C.byref(g), ema.data_ptr(), s.data_ptr(), c.data_ptr(), 0.5, 1e-5,
                                         cdf.data_ptr(), ws.data_ptr(), L.stream()))

    def draw():
        L.check(lib.hrf_error_map_draw(cdf.data_ptr(), C.byref(g), 1, counter[0], R, 0.25, pixels.data_ptr(),
                                       L.stream()))
        counter[0] += 1

    update()
    draw()
    t_acc, t_upd, t_draw = _timed(accumulate, iters), _timed(update, iters), _timed(draw, iters)
    t_all = _timed(lambda: (draw(), accumulate(), update()), iters)
    t_reset = _timed(lambda: L.check(lib.hrf_error_map_reset_slots(C.byref(g), 1, 1, 1.0, ema.data_ptr(), L.stream())),
                     iters)
    return {"metric": "error_map_ms_per_step", "pool": f"{B}x{W}x{H}", "tile": T, "tiles": n, "rays": R,
            "accumulate_ms": t_acc, "update_ms": t_upd, "draw_ms": t_draw, "reset_slot_ms": t_reset, "value": t_all,
            "unit": "ms",
            "update_bytes_per_tile": 20, "update_gb_s": 20 * n / (t_upd * 1e-3) / 1e9}


def train_step_cost(R: int, iters: int) -> list:
    import numpy as np

    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.error_map import ErrorMap
    from humanrf_b200.training import FusedTrainer

    dev = torch.device("cuda:0")
    np.random.seed(0)
    ds = SyntheticDataset(num_cameras=64, frames=range(15, 16), width=96, height=72)
    dl = DL(dataset=ds, device="cuda", mode=DL.Mode.TRAINING, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
            space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=R, camera_numbers=tuple(range(64)),
            frame_numbers=(15,), max_buffer_size=64, max_num_frames_per_batch=1, use_mask=False,
            filter_light_bloom=False)
    b = synthetic_rays(R, 32, list(range(15, 65)), seed=4)
    g = {k: v.to(dev).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba")}
    pixels = torch.randint(0, dl.buffer_size * dl.num_pixels_per_camera, (R,), device=dev)
    out = []
    for use in (False, True, False, True):
        m, _ = make_model((50,), seed=1, device=dev)
        em = ErrorMap(dl, tile=16) if use else None
        tr = FusedTrainer(m, error_map=em)

        def step():
            tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, pixels=pixels if use else None)
            if use:
                em.draw(R)
        out.append({"metric": "train_step_ms", "error_map": use, "rays": R, "value": _timed(step, iters), "unit": "ms"})
        dl.ray_source = None
    return out


def loader_next_cost(R: int, iters: int) -> list:
    """next() on a 16-slot pool of 96x72 images over 64 (camera, frame) pairs: one slot reloaded per batch."""
    import numpy as np

    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.error_map import ErrorMap

    out = []
    for use in (False, True, False, True):
        np.random.seed(0)
        ds = SyntheticDataset(num_cameras=32, frames=range(15, 17), width=96, height=72)
        dl = DL(dataset=ds, device="cuda", mode=DL.Mode.TRAINING, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=R, camera_numbers=tuple(range(32)),
                frame_numbers=(15, 16), max_buffer_size=16, max_num_frames_per_batch=2, use_mask=False,
                filter_light_bloom=False)
        if use:
            ErrorMap(dl, tile=16)
        it = iter(dl)
        out.append({"metric": "loader_next_ms", "error_map": use, "rays": R, "slots": dl.buffer_size,
                    "reloads_per_next": dl.replace_per_next, "value": _timed(lambda: next(it), iters), "unit": "ms"})
    return out


def quality(seeds, steps: int) -> list:
    """Held-out PSNR (dB, mean of the held-out camera's first and last frame) after `steps` steps, and after the steps
    that train on steps * samples_max samples, for uniform rays and for the error map."""
    sys.path.insert(0, str(ROOT / "examples"))
    import train_synthetic as T

    samples_max = 200_000
    out = []
    for seed in seeds:
        for name, kw in (("uniform", None), ("error_map", {"tile": 8, "uniform_fraction": 0.25})):
            h, st = T.main(steps=steps, samples_max=samples_max, log_every=steps, quiet=True, return_state=True,
                           seed=seed, error_map=kw)
            hb, sb = T.main(steps=3 * steps, samples_max=samples_max, log_every=3 * steps, quiet=True,
                            return_state=True, seed=seed, error_map=kw, sample_budget=steps * samples_max)
            out.append({"metric": "held_out_psnr_db", "sampling": name, "seed": seed,
                        "equal_steps": {"steps": st["steps"], "samples": st["samples"], "value": h[-1][1]},
                        "equal_samples": {"steps": sb["steps"], "samples": sb["samples"], "value": hb[-1][1]},
                        "initial": h[0][1], "unit": "dB"})
            print(json.dumps(out[-1]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--quality", action="store_true", help="run the held-out PSNR comparison instead of the costs")
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1, 2])
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()
    card = _card()
    if args.quality:
        print(json.dumps({"gpu": card}), flush=True)
        rows = quality(args.seeds, args.steps)
        for name in ("uniform", "error_map"):
            for k in ("equal_steps", "equal_samples"):
                v = [r[k]["value"] for r in rows if r["sampling"] == name]
                print(json.dumps({"metric": "held_out_psnr_db_mean", "sampling": name, "at": k, "value": float(sum(v) / len(v)),
                                  "seeds": args.seeds, "unit": "dB", **card}), flush=True)
        return
    for B, W, H in ((64, 96, 72), (200, 1022, 750), (200, 4088, 3000)):
        for T in (16, 32):
            print(json.dumps({**map_cost(B, W, H, T, args.rays, args.iters), **card}), flush=True)
    for line in train_step_cost(args.rays, args.iters) + loader_next_cost(args.rays, args.iters):
        print(json.dumps({**line, **card}), flush=True)


if __name__ == "__main__":
    main()
