"""The compact model (int8 tables, DESIGN.md §3.19) against the bf16 model it was quantised from, in one process on one
GPU.  bf16 and int8 alternate, `--repeats` times each, and every rate is reported as its median with min and max:

* fused render rays/s on bench.py's render workload (4096 rays x 512 samples, trained-like N(0, 0.05) tables) for each
  of `--segments` (one inference render of the batch: hrf_render_fused through volume_rendering.render_fused);
* the early-stop density pass of prune_samples on the same batch (ms);
* full 1028x752 images through the tile renderer (bench.py --mode image's workload, Mpix/s);
* quantisation time, file bytes against the fp32 state_dict's, and device bytes each model holds.

Every measured window ends in a device synchronise; each shape is warmed up first.  The card's name and power limit are
read in the same process.  Prints one JSON line.
    python scripts/compact_bench.py [--segments 50 100 100,100,50] [--repeats 3] [--steps 20]
"""
import argparse
import io
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_identity():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        pass
    return {"name": name, "power_limit_w": limit}


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def model_bytes(m):
    """Device bytes of every tensor a bf16 HumanRF holds for rendering: fp32 parameters and buffers, and its native
    view (bf16 shadows, transposed vectors, MLP blob)."""
    n = sum(t.numel() * t.element_size() for t in list(m.parameters()) + list(m.buffers()))
    nat = m.native()
    n += sum(s.numel() * 2 for ss in nat.shadows for s in ss) + sum(v.numel() * 4 for v in nat.vec_t) + nat.blob.numel() * 2
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", nargs="+", default=["50", "100", "100,100,50"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-image", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compact_bench needs a CUDA device")
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.compact_model import quantize_model
    from humanrf_b200.volume_rendering import ray_offsets, render_fused

    dev = torch.device("cuda:0")
    out = {"gpu": gpu_identity(), "repeats": args.repeats, "steps": args.steps, "workloads": {}}
    for key in args.segments:
        segs = tuple(int(s) for s in key.split(","))
        m, frames = make_model(segs, seed=123, device=dev)
        torch.cuda.synchronize()
        tq = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            cm = quantize_model(m)
            torch.cuda.synchronize()
            tq.append(time.perf_counter() - t0)
        b = synthetic_rays(4096, 512, frames, seed=0)
        g = {k: v.to(dev).contiguous() for k, v in b.items()}
        o, d, fr = g["o"], g["d"], g["frames"].to(torch.int32)
        t, ri = g["t"].reshape(-1), g["ri"].to(torch.int64)
        R = o.shape[0]
        off = ray_offsets(ri, R)
        res = {"render_rays_per_s": {}, "early_stop_ms": {}}
        models = {"bf16": m, "int8": cm}
        fns = {}
        for name, mod in models.items():
            nat = mod.native()
            samples = nat.samples_rays(o, d, fr, t, ri)
            fns[name] = (lambda mod=mod: render_fused(mod, o, d, fr, t, ri, R, 0.0, ray_offsets_dev=off),
                         lambda nat=nat, samples=samples: nat.density_early_stop(samples, off, R, 4e-4))
            for f in fns[name]:
                timed(f, args.warmup)
        render = {n: [] for n in models}
        es = {n: [] for n in models}
        for _ in range(args.repeats):
            for name in models:
                render[name].append(R / timed(fns[name][0], args.steps))
                es[name].append(1e3 * timed(fns[name][1], args.steps))
        res["render_rays_per_s"] = {n: spread(v) for n, v in render.items()}
        res["early_stop_ms"] = {n: spread(v) for n, v in es.items()}
        res["quantize_s"] = spread(tq)
        buf = io.BytesIO()
        torch.save(m.state_dict(), buf)
        with tempfile.TemporaryDirectory() as tmp:
            cm.save(Path(tmp) / "c.pt")
            fb = (Path(tmp) / "c.pt").stat().st_size
        res["bytes"] = {"state_dict": buf.tell(), "compact_file": fb, "file_over_state_dict": fb / buf.tell(),
                        "device_bf16_model": model_bytes(m), "device_compact_model": cm.device_bytes(),
                        "compact_parts": cm.parts()}
        rms = cm.rms.cpu().numpy()
        res["rms_error"] = {"median": float(np.median(rms)), "max": float(rms.max())}
        res["clip_ratio_counts"] = np.bincount(cm.clip.cpu().numpy().ravel(), minlength=8).tolist()
        out["workloads"][key] = res
        del fns, models, cm, m
        torch.cuda.empty_cache()
    if not args.no_image:
        out["image_mpix_per_s"] = image_rates(args, dev)
    print(json.dumps(out))


def image_rates(args, dev):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.compact_model import quantize_model

    W, H, G = 1028, 752, 256
    m, _ = make_model((50,), seed=123, device=dev)
    cm = quantize_model(m)
    sc = make_scene(num_images=1, width=W, height=H, G=G, portrait_every=0)
    og = OccupanyGrid(G, 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    cam = dict(frame_numbers=t(sc["frame_numbers"]), camera_numbers=t(sc["camera_numbers"]),
               grid_handles=torch.tensor([og.add_grid(t(sc["grids"][0]))], dtype=torch.int64, device=dev),
               landscape=t(sc["landscape"]), inverse_krs=t(sc["inverse_krs"]), camera_origins=t(sc["camera_origins"]),
               aabb=t(sc["aabb"]), G=G, width=W, height=H)
    rs = {"bf16": TileShardedRenderer(m, og, rays_per_batch=262144), "int8": TileShardedRenderer(cm, og, rays_per_batch=262144)}
    for r in rs.values():
        timed(lambda r=r: r.render_image_sharded(cam, 0, 1), max(args.warmup, 3))
    rates = {n: [] for n in rs}
    steps = max(args.steps // 4, 3)
    for _ in range(args.repeats):
        for n, r in rs.items():
            rates[n].append(W * H / timed(lambda r=r: r.render_image_sharded(cam, 0, 1), steps) / 1e6)
    return {n: spread(v) for n, v in rates.items()}


if __name__ == "__main__":
    main()
