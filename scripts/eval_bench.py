"""Time of hrf_image_metrics (csrc/image_metrics.cu) on an ActorsHQ-sized image (4112x3008) and on a quarter-size one
(1028x752), each with a centred-ellipse mask and with a full mask.  L2 flushed before every call, CUDA events around it,
`--warmup` calls then `--steps` timed calls per workload.  Bytes moved: the mask once (ROI pass) plus 7 bytes per pixel
of the ROI and its 3-pixel halo (pred and gt RGB, mask); the bandwidth is reported against the H100 SXM data sheet's
3.35 TB/s.  At 1028x752 one evaluate_sequence view is split into render, metrics and PNG write (host clock around each
phase, synchronised).  Prints one JSON line with the card's name and power limit.
    python scripts/eval_bench.py [--steps 100] [--warmup 10]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bake_bench import gpu_identity  # noqa: E402

PEAK_BW = 3.35e12


def ellipse(W, H):
    y, x = np.mgrid[0:H, 0:W]
    return (((x + 0.5 - W / 2) / (0.35 * W)) ** 2 + ((y + 0.5 - H / 2) / (0.42 * H)) ** 2 <= 1).astype(np.uint8) * 255


def bytes_moved(mask, W, H):
    ys, xs = np.nonzero(mask)
    x0, x1, y0, y1 = max(xs.min() - 3, 0), min(xs.max() + 3, W - 1), max(ys.min() - 3, 0), min(ys.max() + 3, H - 1)
    return W * H + 7 * (x1 - x0 + 1) * (y1 - y0 + 1)


def time_metrics(fn, steps, warmup, flush):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        flush.zero_()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.mean(ts)), float(np.median(ts))


def view_phases(dev, reps):
    """One evaluate_sequence view at 1028x752: render (colour of the fused kernel), quantise + metrics, PNG write."""
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.depth_maps import _Views
    from humanrf_b200.toolbox.evaluation import ground_truth, image_metrics, quantize, write_frame_png

    W, H = 1028, 752
    ds = SyntheticDataset(num_cameras=3, width=W, height=H, G=256)
    dl = DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
            space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=W * H, camera_numbers=(0, 1, 2),
            frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])
    model, _ = make_model((len(ds.frames),), first_frame=ds.frames[0], seed=123, device=dev)
    views = _Views(model, dl, 4e-4, 262144)
    grid = views.hull(15)
    gt, mask = ground_truth(dl, 0, 15)
    gt_d, mask_d = torch.from_numpy(gt).to(dev), torch.from_numpy(mask).to(dev)
    phases = {"render": [], "metrics": [], "png_write": []}
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            color = views.render(0, 15, grid).color
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            out, _ = image_metrics(quantize(color), gt_d, mask_d)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            write_frame_png(os.path.join(tmp, "Cam001_rgb000015.png"), quantize(color))
            t3 = time.perf_counter()
            if i:                                   # the first view warms up
                phases["render"].append(1e3 * (t1 - t0))
                phases["metrics"].append(1e3 * (t2 - t1))
                phases["png_write"].append(1e3 * (t3 - t2))
    return {k: float(np.median(v)) for k, v in phases.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--view-reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench.py needs a CUDA device (the metrics kernel has no CPU path)")
    from humanrf_b200.toolbox.evaluation import image_metrics

    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    workloads = {}
    for W, H in ((4112, 3008), (1028, 752)):
        rng = np.random.default_rng(W)
        gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        pred = np.clip(gt.astype(np.int32) + rng.integers(-20, 21, gt.shape), 0, 255).astype(np.uint8)
        g, p = torch.from_numpy(gt).to(dev), torch.from_numpy(pred).to(dev)
        for kind, mask in (("ellipse", ellipse(W, H)), ("full", np.full((H, W), 255, np.uint8))):
            m = torch.from_numpy(mask).to(dev)
            out = torch.empty(2, dtype=torch.float64, device=dev)
            mean, med = time_metrics(lambda: image_metrics(p, g, m, out=out), a.steps, a.warmup, flush)
            nbytes = bytes_moved(mask, W, H)
            workloads[f"{W}x{H}_{kind}"] = {
                "ms": mean, "ms_median": med, "bytes": int(nbytes), "tb_per_s": nbytes / (mean * 1e-3) / 1e12,
                "share_of_3p35_tb_s": nbytes / (mean * 1e-3) / PEAK_BW, "psnr": float(out[0]), "ssim": float(out[1])}
    phases = view_phases(dev, a.view_reps)
    print(json.dumps({
        "metric": "image_metrics_ms_4112x3008_ellipse", "value": workloads["4112x3008_ellipse"]["ms"], "unit": "ms",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu_identity": gpu_identity(0),
        "workloads": workloads, "view_1028x752_ms": phases,
        "config": {"l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events per call",
                   "bytes": "mask once + 7 B per pixel of the ROI and its 3-pixel halo",
                   "view": "evaluate_sequence phases of one view, bench model, SyntheticDataset hull G=256, "
                           "median of --view-reps, host clock with synchronise"}}))


if __name__ == "__main__":
    main()
