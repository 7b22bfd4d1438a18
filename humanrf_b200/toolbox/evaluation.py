"""Scores of rendered test views on the GPU, in the ActorsHQ evaluation convention.

``image_metrics`` scores one pair of 8-bit images with ``hrf_image_metrics`` (csrc/image_metrics.cu, contract in
include/humanrf_b200.h): a PSNR over the mask's pixels and scikit-image's SSIM over the mask's bounding rectangle, the
numbers ``actorshq/evaluation/evaluate.py`` writes.  ``evaluate_sequence`` replaces the reference's ``Trainer.test`` +
``evaluate`` pair: it renders each (camera, frame) view, scores it against the dataset's image and mask without the image
leaving the device, optionally writes the 8-bit PNGs ``Trainer.test`` writes, and writes ``metrics.csv`` and
``averages.csv``.  LPIPS is added when weights are given (toolbox/lpips.py); VMAF is not computed.
"""
from __future__ import annotations

import csv
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from .. import _lib as L
from .depth_maps import _check_camera, _check_frame, _Views, camera_name

METRICS = ("PSNR", "SSIM")
METRICS_LPIPS = ("PSNR", "LPIPS", "SSIM")     # evaluate.py's order


@dataclass
class ViewScore:
    """Scores of one view: camera number (0-based), frame, PSNR (dB), SSIM, the ROI (x, y, w, h) and LPIPS (None when
    not computed)."""
    camera: int
    frame: int
    psnr: float
    ssim: float
    roi: tuple
    lpips: float | None = None


def _check_image(t, name, shape):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.device.type != "cuda" or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous uint8 CUDA tensor")
    if tuple(t.shape) != shape:
        raise RuntimeError(f"{name} has shape {tuple(t.shape)}, expected {shape}")


def image_metrics(pred_u8: torch.Tensor, gt_u8: torch.Tensor, mask: torch.Tensor, out: torch.Tensor | None = None):
    """PSNR and SSIM of `pred_u8` against `gt_u8` (uint8 [H,W,3] RGB) under `mask` (uint8 or bool [H,W], non-zero =
    foreground), all contiguous on one CUDA device.  Returns (out float64 [2] = (PSNR, SSIM), roi int32 [4] = (x, y, w,
    h)) on the device without synchronising; `out` may be given (e.g. a row of an [n,2] tensor) and is written in place.
    SSIM is NaN when the ROI is under 7 pixels wide or tall, both are NaN for an empty mask, PSNR is inf for equal
    masked pixels."""
    if not isinstance(pred_u8, torch.Tensor) or pred_u8.dim() != 3 or pred_u8.shape[2] != 3:
        raise RuntimeError("pred_u8 must be an [H,W,3] tensor")
    H, W = int(pred_u8.shape[0]), int(pred_u8.shape[1])
    _check_image(pred_u8, "pred_u8", (H, W, 3))
    _check_image(gt_u8, "gt_u8", (H, W, 3))
    if isinstance(mask, torch.Tensor) and mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    _check_image(mask, "mask", (H, W))
    dev = pred_u8.device
    if gt_u8.device != dev or mask.device != dev:
        raise RuntimeError("pred_u8, gt_u8 and mask must be on one device")
    if out is None:
        out = torch.empty(2, dtype=torch.float64, device=dev)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float64 or out.device != dev or out.shape != (2,)
          or not out.is_contiguous()):
        raise RuntimeError(f"out must be a contiguous float64 [2] tensor on {dev}")
    roi = torch.empty(4, dtype=torch.int32, device=dev)
    ws = torch.empty(int(L.lib().hrf_image_metrics_workspace_bytes(W, H)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(L.lib().hrf_image_metrics(pred_u8.data_ptr(), gt_u8.data_ptr(), mask.data_ptr(), W, H, out.data_ptr(),
                                          roi.data_ptr(), ws.data_ptr(), L.stream()))
    return out, roi


def quantize(color: torch.Tensor) -> torch.Tensor:
    """``(color * 255).to(uint8)``: truncation, as ``Trainer.test``'s ``(x * 255).astype(np.uint8)`` for colours in
    [0, 1]."""
    return (color * 255).to(torch.uint8)


def ground_truth(loader, camera_number: int, frame_number: int):
    """The dataset's image as uint8 [H,W,3] RGB and its mask as bool [H,W] (numpy).  ``get_rgb`` gives BGR (OpenCV's
    order); float images are ``uint8 / 255`` and come back exactly through ``rint(clip(x * 255, 0, 255))``."""
    cam = loader.cameras[camera_number]
    shape = (int(cam.height), int(cam.width))
    rgb = np.asarray(loader.dataset.get_rgb(camera_number, frame_number))
    if rgb.dtype != np.uint8:
        rgb = np.rint(np.clip(rgb.astype(np.float64) * 255.0, 0, 255)).astype(np.uint8)
    m = np.asarray(loader.dataset.get_mask(camera_number, frame_number))
    if rgb.shape != shape + (3,) or m.ndim != 3 or m.shape[:2] != shape:
        raise RuntimeError(f"camera {camera_number} frame {frame_number}: image {rgb.shape} / mask {m.shape} do not "
                           f"match the camera's {shape[0]}x{shape[1]} (height x width)")
    return np.ascontiguousarray(rgb[..., ::-1]), m[..., 0] > 0


def frame_path(out_dir, name: str, frame: int) -> str:
    """``test_frames/<cam>_rgb%06d.png``: the name ``Trainer.test`` gives a view (the dataset image's stem + .png)."""
    return os.path.join(out_dir, "test_frames", f"{name}_rgb{frame:06d}.png")


def write_frame_png(path, rgb_u8) -> None:
    """8-bit colour PNG of an RGB image, written through OpenCV in BGR order as ``Trainer.test`` writes it."""
    import cv2

    img = np.ascontiguousarray(np.asarray(rgb_u8.cpu() if isinstance(rgb_u8, torch.Tensor) else rgb_u8, np.uint8))
    if not cv2.imwrite(str(path), cv2.cvtColor(img, cv2.COLOR_RGB2BGR)):
        raise RuntimeError(f"writing {path} failed")


def write_metric_tables(out_dir, scores) -> None:
    """``metrics.csv`` (camera numbered from 1, frame, PSNR, SSIM per view, in order) and ``averages.csv`` (the mean of
    each metric), laid out as actorshq/evaluation/evaluate.py writes them.  Its LPIPS column, between PSNR and SSIM, is
    written when every score carries an LPIPS."""
    with_lpips = bool(scores) and all(s.lpips is not None for s in scores)
    metrics = METRICS_LPIPS if with_lpips else METRICS
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "metrics.csv"), "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=["camera", "frame", *metrics])
        w.writeheader()
        for s in scores:
            row = {"camera": s.camera + 1, "frame": s.frame, "PSNR": s.psnr, "SSIM": s.ssim}
            if with_lpips:
                row["LPIPS"] = s.lpips
            w.writerow(row)
    with open(os.path.join(out_dir, "averages.csv"), "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=list(metrics))
        w.writeheader()
        row = {"PSNR": float(np.mean([s.psnr for s in scores])), "SSIM": float(np.mean([s.ssim for s in scores]))}
        if with_lpips:
            row["LPIPS"] = float(np.mean([s.lpips for s in scores]))
        w.writerow(row)


@torch.no_grad()
def evaluate_sequence(model, loader, pairs, out_dir, bake: bool = False, save_frames: bool = True,
                      render_step_size: float = 4e-4, rays_per_batch: int = 262144, lpips_weights=None):
    """Renders every (camera_number, frame_number) of `pairs` with `model` through `loader`'s cameras (the colour of
    ``render_depth_map``), quantises it to 8 bits as ``Trainer.test`` does and scores it against the dataset's image and
    mask with ``image_metrics``.  With `save_frames` the views are written as ``out_dir/test_frames/<cam>_rgb%06d.png``
    (<cam> = ``camera_name``), which the reference's ``evaluate(..., result_suffix=".png")`` reads.  Writes
    ``out_dir/metrics.csv`` and ``out_dir/averages.csv``.  Views are rendered from the dataset's hulls, as the reference's
    evaluation loader does; with `bake` each frame's hull is first tightened by ``bake_occupancy_grid`` (once per
    frame).  Cameras and frames are checked before anything is written; the scores are read back once, at the end, and
    a view without a score (empty mask, or an ROI under 7x7 pixels) raises before the tables are written.  With
    `lpips_weights` (``load_lpips_alex``) each view's LPIPS is computed too, on the quantised render against the dataset
    image over the ROI ``image_metrics`` wrote, and the tables gain evaluate.py's LPIPS column; an ROI under 31x31 pixels
    has no LPIPS and raises.  Returns a ``ViewScore`` per pair."""
    from .learned_occupancy import bake_occupancy_grid
    from .lpips import lpips

    pairs = [(_check_camera(loader, c), _check_frame(model, f)) for c, f in pairs]
    if not pairs:
        raise RuntimeError("no (camera, frame) pairs to evaluate")
    views = _Views(model, loader, render_step_size, rays_per_batch)
    dev = views.device
    values = torch.empty(len(pairs), 2 if lpips_weights is None else 3, dtype=torch.float64, device=dev)
    rois = []
    grids = {}
    if save_frames:
        os.makedirs(os.path.join(out_dir, "test_frames"), exist_ok=True)
    for k, (c, frame) in enumerate(pairs):
        if frame not in grids:
            grid = views.hull(frame)
            grids[frame] = bake_occupancy_grid(model, frame, grid, render_step_size) if bake else grid
        pred = quantize(views.render(c, frame, grids[frame]).color)
        gt, mask = ground_truth(loader, c, frame)
        gt = torch.from_numpy(gt).to(dev)
        _, roi = image_metrics(pred, gt, torch.from_numpy(mask).to(dev), out=values[k, :2])
        if lpips_weights is not None:
            lpips(pred, gt, lpips_weights, roi=roi, out=values[k, 2])
        rois.append(roi)
        if save_frames:
            write_frame_png(frame_path(out_dir, camera_name(loader, c), frame), pred)
    v = values.cpu().numpy()
    r = torch.stack(rois).cpu().numpy()
    scores = [ViewScore(c, f, float(v[k, 0]), float(v[k, 1]), tuple(int(x) for x in r[k]),
                        None if lpips_weights is None else float(v[k, 2])) for k, (c, f) in enumerate(pairs)]
    bad = [(s.camera, s.frame) for s in scores if math.isnan(s.psnr) or math.isnan(s.ssim)]
    if bad:
        raise RuntimeError(f"no score for (camera, frame) {bad}: empty mask, or a mask bounding box under 7x7 pixels")
    bad = [(s.camera, s.frame) for s in scores if s.lpips is not None and math.isnan(s.lpips)]
    if bad:
        raise RuntimeError(f"no LPIPS for (camera, frame) {bad}: a mask bounding box under 31x31 pixels")
    write_metric_tables(out_dir, scores)
    return scores
