"""Cost of the held-out response fit (CameraResponses.fit_held_out, DESIGN.md §3.18).
* hrf_response_fit_accumulate alone at 1028x752 and 4112x3008 (full mask): CUDA events over `--reps` back-to-back
  launches, and the rate over the 20 bytes a pixel is read with (colour 12, alpha 4, gt 3, mask 1) against the H100
  SXM data sheet's 3.35 TB/s.
* fit_held_out for 14 cameras x 8 frames at 1028x752 on the bench model (make_model, SyntheticDataset hulls G=256),
  against evaluate_sequence over the same 112 views (no responses, no PNGs): host clock around each call, after one
  warm-up call of each.
Prints one JSON line with the card's name and power limit.
    python scripts/response_fit_bench.py [--reps 200]
"""
import argparse
import json
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
from pose_bench import per_launch_ms  # noqa: E402

HBM_TBS = 3.35
BYTES_PER_PIXEL = 20


def accumulate_rates(dev, reps):
    from types import SimpleNamespace

    from humanrf_b200 import _lib as L
    from humanrf_b200.toolbox.camera_response import FIT_ROW, CameraResponses

    resp = CameraResponses(SimpleNamespace(all_inverse_krs=torch.zeros((160, 3, 3), device=dev),
                                           camera_numbers=tuple(range(160))), fixed_cameras=())
    out = {}
    for W, H in ((1028, 752), (4112, 3008)):
        P = W * H
        g = torch.Generator(device=dev).manual_seed(P)
        color = torch.rand((P, 3), device=dev, generator=g)
        alpha = torch.rand(P, device=dev, generator=g)
        gt = torch.randint(0, 256, (P, 3), dtype=torch.uint8, device=dev, generator=g)
        mask = torch.ones(P, dtype=torch.uint8, device=dev)
        moments = torch.zeros((160, FIT_ROW), dtype=torch.float64, device=dev)
        error = torch.zeros(1, dtype=torch.int32, device=dev)
        ws = torch.empty(int(L.lib().hrf_response_fit_workspace_bytes(P)), dtype=torch.uint8, device=dev)
        ms = per_launch_ms(lambda: resp.accumulate_fit(color, alpha, gt, mask, 5, moments, error, ws), reps)
        rate = BYTES_PER_PIXEL * P / (ms * 1e-3) / 1e12
        out[f"{W}x{H}"] = {"ms": ms, "TB_per_s": rate, "share_of_3.35_TB_per_s": rate / HBM_TBS}
    return out


def fit_vs_eval(dev):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.camera_response import CameraResponses, held_out_fit_pairs
    from humanrf_b200.toolbox.evaluation import evaluate_sequence

    W, H, n_cams, frames = 1028, 752, 15, list(range(15, 25))
    ds = SyntheticDataset(num_cameras=n_cams, width=W, height=H, G=256, frames=frames)
    dl = DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
            space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=W * H, camera_numbers=tuple(range(n_cams)),
            frame_numbers=tuple(frames), max_buffer_size=1, render_sequence=[(0, 15)])
    model, _ = make_model((len(frames),), first_frame=frames[0], seed=123, device=dev)
    held = list(range(1, n_cams))                     # camera 0 holds the gauge
    score = [(c, frames[c % len(frames)]) for c in held]
    pairs = held_out_fit_pairs(score, frames, per_camera=8)
    resp = CameraResponses(dl)
    times = {"fit_held_out": [], "evaluate_sequence": []}
    refused = None
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                resp.fit_held_out(model, dl, pairs)
            except ValueError as e:   # the synthetic images are not the model's renders: a refusal still did every view
                refused = str(e)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            evaluate_sequence(model, dl, pairs, tmp, save_frames=False)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if i:                                     # the first call of each warms up
                times["fit_held_out"].append(t1 - t0)
                times["evaluate_sequence"].append(t2 - t1)
    fit, ev = float(np.median(times["fit_held_out"])), float(np.median(times["evaluate_sequence"]))
    return {"views": len(pairs), "cameras": len(held), "image": f"{W}x{H}", "fit_held_out_s": fit,
            "evaluate_sequence_s": ev, "fit_over_eval": fit / ev, "runs": times,
            "solve_refused": refused}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("response_fit_bench.py needs a CUDA device (the kernels have no CPU path)")
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_identity(0), "accumulate": accumulate_rates(dev, a.reps), "fit_vs_eval": fit_vs_eval(dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
