"""Time of hrf_lpips (csrc/lpips.cu) per image pair at 1028x752 and 4112x3008 (ActorsHQ's size), each over the whole
image and over the bounding box of eval_bench.py's centred ellipse (2878x2526 at full size).  Seeded random weights
(the time does not depend on their values).  L2 flushed before every call, CUDA events around it, `--warmup` calls
then `--steps` timed calls per workload.  FLOPs come from the shapes: 2 MACs per pair (both images through the five
convolutions); the rate is reported against the H100 SXM data sheet's 495 TFLOP/s dense TF32, which a power-capped
card may not reach.  At 1028x752 one evaluate_sequence view is split into render, PSNR/SSIM and LPIPS (host clock
around each phase, synchronised).  Prints one JSON line with the card's name and power limit.
    python scripts/lpips_bench.py [--steps 100] [--warmup 10]
"""
import argparse
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
from eval_bench import ellipse, time_metrics  # noqa: E402

PEAK_TF32 = 495e12
CONVS = ((3, 64, 11, 4, 2), (64, 192, 5, 1, 2), (192, 384, 3, 1, 1), (384, 256, 3, 1, 1), (256, 256, 3, 1, 1))


def flops(w, h):
    """2 * multiply-adds of the five convolutions for both images of a w x h pair."""
    from humanrf_b200.toolbox.lpips import tensor_sizes

    sizes = tensor_sizes(w, h)
    macs = 0
    for (cin, cout, ks, _, _), t in zip(CONVS, (1, 3, 5, 6, 7)):
        oh, ow = sizes[t]
        macs += oh * ow * cout * ks * ks * cin
    return 2 * 2 * macs


def seeded_weights(dev):
    import torchvision

    from humanrf_b200.toolbox.lpips import lpips_alex_from_state_dicts

    torch.manual_seed(0)
    alex = torchvision.models.alexnet(weights=None).state_dict()
    lin = {f"lin{k}.model.1.weight": torch.rand(1, c[1], 1, 1) * 0.1 for k, c in enumerate(CONVS)}
    return lpips_alex_from_state_dicts(alex, lin, dev)


def roi_of(mask):
    ys, xs = np.nonzero(mask)
    return [int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1)]


def view_phases(dev, weights, reps):
    """One evaluate_sequence view at 1028x752: render (colour of the fused kernel), quantise + PSNR/SSIM, LPIPS."""
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.depth_maps import _Views
    from humanrf_b200.toolbox.evaluation import ground_truth, image_metrics, quantize
    from humanrf_b200.toolbox.lpips import lpips

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
    phases = {"render": [], "metrics": [], "lpips": []}
    for i in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        color = views.render(0, 15, grid).color
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        pred = quantize(color)
        _, roi = image_metrics(pred, gt_d, mask_d)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        lpips(pred, gt_d, weights, roi=roi)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        if i:                                   # the first view warms up
            phases["render"].append(1e3 * (t1 - t0))
            phases["metrics"].append(1e3 * (t2 - t1))
            phases["lpips"].append(1e3 * (t3 - t2))
    out = {k: float(np.median(v)) for k, v in phases.items()}
    out["roi"] = [int(x) for x in roi.cpu()]
    out["lpips_share_of_view"] = out["lpips"] / (out["render"] + out["metrics"] + out["lpips"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--view-reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lpips_bench.py needs a CUDA device (the LPIPS kernels have no CPU path)")
    from humanrf_b200.toolbox.lpips import lpips, workspace_bytes

    dev = torch.device("cuda:0")
    weights = seeded_weights(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    workloads = {}
    for W, H in ((1028, 752), (4112, 3008)):
        rng = np.random.default_rng(W)
        gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        pred = np.clip(gt.astype(np.int32) + rng.integers(-20, 21, gt.shape), 0, 255).astype(np.uint8)
        g, p = torch.from_numpy(gt).to(dev), torch.from_numpy(pred).to(dev)
        ws = torch.empty(workspace_bytes(W, H), dtype=torch.uint8, device=dev)
        for kind, roi in (("full", [0, 0, W, H]), ("ellipse", roi_of(ellipse(W, H)))):
            r = torch.tensor(roi, dtype=torch.int32, device=dev)
            out = torch.empty((), dtype=torch.float64, device=dev)
            mean, med = time_metrics(lambda: lpips(p, g, weights, roi=r, out=out, workspace=ws), a.steps, a.warmup, flush)
            f = flops(roi[2], roi[3])
            workloads[f"{W}x{H}_{kind}"] = {
                "roi": roi, "ms": mean, "ms_median": med, "gflop": f / 1e9, "tflop_per_s": f / (mean * 1e-3) / 1e12,
                "share_of_495_tflop_s_tf32": f / (mean * 1e-3) / PEAK_TF32, "lpips": float(out)}
        del ws
    phases = view_phases(dev, weights, a.view_reps)
    print(json.dumps({
        "metric": "lpips_ms_4112x3008_full", "value": workloads["4112x3008_full"]["ms"], "unit": "ms",
        "higher_is_better": False, "steps": a.steps, "warmup": a.warmup, "gpu_identity": gpu_identity(0),
        "workloads": workloads, "view_1028x752_ms": phases,
        "config": {"l2": "flushed before each timed call (256 MiB memset)", "timing": "CUDA events per call",
                   "flops": "2 x multiply-adds of the five convolutions, both images",
                   "peak": "H100 SXM data sheet, dense TF32, 495 TFLOP/s; a power-capped card may not reach it",
                   "view": "evaluate_sequence phases of one view, bench model, SyntheticDataset hull G=256, "
                           "median of --view-reps, host clock with synchronise"}}))


if __name__ == "__main__":
    main()
