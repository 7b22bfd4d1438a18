"""Camera pose refinement against a trained, frozen model.

``refine_camera`` adjusts the extrinsics of one camera so that the model's renders from it match that camera's images
at the given frames.  It is built on the ray gradients of ``volume_rendering.render``: the rays are built in torch from
the pose, rendered with the sampler's choice of samples held fixed, and the loss's gradient flows back through
d(ray origins) and d(ray directions) (hrf_field_backward_mlp_dirs, hrf_field_position_grad, hrf_ray_gradients) to the
pose.

The pose increment is delta = (omega, tau) in R^6: R' = exp([omega]x) R and c' = c + tau, with R the camera-to-world
rotation and c the camera centre, both in the loader's normalised scene units inside the loop.  Each iteration:

1. draws a seeded subset of the image's pixels;
2. builds the sampler tables of the view from (R', c'): the transposed inverse KR table and the origin the loader
   keeps in ``all_inverse_krs`` / ``all_camera_origins``;
3. runs the sampler, the density pass with its early stop and the prune, without gradients;
4. recomputes the kept rays' origins and directions in torch from delta, with the sampler's formula
   (d = v / |v|, v = px T[0] + py T[1] + T[2], px, py the pixel centre); they equal the sampler's within a few fp32 ulps;
5. renders them with ``render`` (background 0), the sample distances held constant as in the reference;
6. takes the mean squared error against the image composited on black with its mask, and steps Adam on delta.

The result is returned in the dataset camera's own convention and world units (``rotation_axisangle`` of the
camera-to-world rotation, ``translation`` of the camera centre), so the loader's normalisation is undone and the values
can replace the calibration's entries.  Intrinsics, per-frame poses and several cameras at once are not refined.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np
import torch


@dataclass
class CameraRefinement:
    """Refined extrinsics of one camera in the dataset's convention and world units, and the loss per iteration."""
    rotation_axisangle: np.ndarray          # [3] camera-to-world rotation, axis * angle
    translation: np.ndarray                 # [3] camera centre in world units
    losses: List[float] = field(default_factory=list)
    omega: np.ndarray = None                # [3] the rotation increment exp([omega]x) applied on the left of R
    tau: np.ndarray = None                  # [3] the centre increment, normalised scene units


def _skew(w: torch.Tensor) -> torch.Tensor:
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def rotation_increment(omega: torch.Tensor) -> torch.Tensor:
    """exp([omega]x), differentiable at omega = 0 (the identity there, exactly)."""
    return torch.linalg.matrix_exp(_skew(omega))


def view_table(inverse_kr: torch.Tensor, omega: torch.Tensor) -> torch.Tensor:
    """The sampler's transposed inverse-KR table of the rotated view, float32 [3,3]: (exp([omega]x) M)^T with
    M = inverse_kr^T (= R K^-1), in float64 before the one rounding.  omega = 0 gives `inverse_kr` bit for bit."""
    M = inverse_kr.reshape(3, 3).to(torch.float64).T
    return (rotation_increment(omega.to(torch.float64)) @ M).T.to(torch.float32)


def pixel_rays(table: torch.Tensor, origin: torch.Tensor, pixels: torch.Tensor, width: int):
    """Origins and unit directions [P,3] (float32) of the pixels `pixels` (row-major indices of a landscape image of
    width `width`) for the table and origin of one view: the sampler's formula in torch, differentiable in both."""
    px = (pixels % width).to(torch.float32) + 0.5
    py = torch.div(pixels, width, rounding_mode="floor").to(torch.float32) + 0.5
    v = px[:, None] * table[0] + py[:, None] * table[1] + table[2]
    d = v / torch.linalg.vector_norm(v, dim=1, keepdim=True)
    return origin.to(torch.float32).expand(pixels.shape[0], 3), d


def axisangle_of(R: np.ndarray) -> np.ndarray:
    """Axis * angle of a rotation matrix (the inverse of dataset.cameras.rotation_from_axisangle)."""
    R = np.asarray(R, np.float64)
    c = np.clip((np.trace(R) - 1) / 2, -1.0, 1.0)
    ang = np.arccos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if ang < 1e-7:
        return 0.5 * w
    if np.pi - ang < 1e-6:      # axis from the symmetric part
        k = np.sqrt(np.maximum((np.diag(R) + 1) / 2, 0.0))
        i = int(np.argmax(k))
        k[np.arange(3) != i] = (R[i] + R[:, i])[np.arange(3) != i] / (4 * k[i])
        return ang * k / np.linalg.norm(k)
    return ang / (2 * np.sin(ang)) * w


def refine_camera(model, loader, camera_number: int, frame_numbers: Sequence[int], iterations: int = 1000,
                  rays_per_step: int = 16384, lr: float = 1e-2, final_lr_ratio: float = 1e-3, seed: int = 0,
                  render_step_size: float = 4e-4) -> CameraRefinement:
    """Refines the extrinsics of `loader`'s camera `camera_number` against its images at `frame_numbers` (read from
    ``loader.dataset``: ``get_rgb`` composited on black with ``get_mask``).  `model` is held frozen: its parameters,
    their ``requires_grad`` flags and their ``.grad`` are as they were when this returns.  Adam on the pose increment,
    learning rate decaying exponentially from `lr` to `lr * final_lr_ratio`, frames taken in turn; the pixel subsets are
    drawn from `seed`, so a run is deterministic.  Landscape images only (the loader's TEST-mode convention for the
    view's size)."""
    from ..dataset import ray_sampler_native as rs
    from ..dataset.cameras import rotation_from_axisangle
    from ..dataset.input_batch import InputBatch
    from ..dataset.occupancy_grid_native import OccupanyGrid
    from ..volume_rendering import prune_samples, render
    from .depth_maps import _check_camera, _check_frame

    c = _check_camera(loader, camera_number)
    frames = [_check_frame(model, f) for f in frame_numbers]
    if not frames:
        raise RuntimeError("refine_camera needs at least one frame")
    dev = loader.aabb.device
    cam = loader.cameras[c]
    W, H = int(cam.width), int(cam.height)
    scale = float(loader.scene_scale)
    inverse_kr = loader.all_inverse_krs[c].to(dev)
    c0 = loader.all_camera_origins[c].to(torch.float64).to(dev)

    # per frame: the hull the sampler skips empty space with, and the target image composited on black
    hulls = [torch.from_numpy(np.ascontiguousarray(loader.dataset.get_occupancy_grid(frame_number=f))).to(dev)
             for f in frames]
    G = int(hulls[0].shape[0])
    og = OccupanyGrid(G, len(frames))
    handles = [torch.tensor([og.add_grid(h.contiguous())], dtype=torch.int64, device=dev) for h in hulls]
    targets = []
    for f in frames:
        rgb = torch.as_tensor(np.asarray(loader.dataset.get_rgb(c, f), np.float32)).reshape(H * W, 3)
        mask = torch.as_tensor(np.asarray(loader.dataset.get_mask(c, f), np.float32)).reshape(H * W, 1)
        targets.append((rgb * mask).to(dev))       # trainer.py:379-385, background 0

    params = list(model.parameters())
    flags = [p.requires_grad for p in params]
    grads = [p.grad for p in params]
    delta = torch.zeros(6, dtype=torch.float64, device=dev, requires_grad=True)
    opt = torch.optim.Adam([delta], lr=lr)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, final_lr_ratio ** (1.0 / max(iterations - 1, 1)))
    gen = torch.Generator().manual_seed(int(seed))
    empty_rgba = torch.zeros((0, 4), dtype=torch.uint8, device=dev)
    empty_mask = torch.zeros(0, dtype=torch.bool, device=dev)
    background = torch.zeros(3, dtype=torch.float32, device=dev)
    landscape = torch.tensor([True], device=dev)
    cam_t = torch.tensor([c], dtype=torch.int32, device=dev)
    losses: List[float] = []
    try:
        for p in params:
            p.requires_grad_(False)
        for it in range(iterations):
            k = it % len(frames)
            pixels = torch.randperm(W * H, generator=gen)[:rays_per_step].to(dev)
            with torch.no_grad():
                table = view_table(inverse_kr, delta[:3])
                origin = (c0 + delta[3:]).to(torch.float32)
                o, d, _, fn, cn, _, ray_mask, dist, rel = rs.get_samples_occupancy_minmax(
                    empty_rgba, empty_mask, torch.tensor([frames[k]], dtype=torch.int32, device=dev), cam_t, handles[k],
                    landscape, pixels, table.reshape(1, 3, 3).contiguous(), origin.reshape(1, 3).contiguous(), loader.aabb,
                    G, W, H, render_step_size, False)
            kept = pixels[ray_mask]
            # pixels without a ray render the background (0): they hold no gradient, but count in the mean
            loss_rest = targets[k][pixels[~ray_mask]].square().sum()
            if o.shape[0] == 0:
                losses.append(float(loss_rest) / pixels.shape[0])
                sched.step()
                continue
            ib = InputBatch(ray_origins=o, ray_directions=d, frame_numbers=fn.view(-1, 1),
                            unique_frame_numbers=torch.tensor([[frames[k]]], dtype=torch.int32, device=dev),
                            camera_numbers=cn.view(-1, 1), sample_distances=dist.view(-1, 1), ray_indices=rel.long(),
                            width=W, height=H)
            prune_samples(ib, model, is_training=False, render_step_size=render_step_size)
            # the same rays as functions of delta (the prune's saved features stay valid: the batch's distances and ray
            # indices are untouched)
            ib.ray_origins, ib.ray_directions = pixel_rays(view_table(inverse_kr, delta[:3]), c0 + delta[3:], kept, W)
            out = render(ib, model, background, is_training=False, render_step_size=render_step_size)
            loss = ((out.color - targets[k][kept]).square().sum() + loss_rest) / pixels.shape[0]
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            sched.step()
            losses.append(float(loss.detach()))
    finally:
        for p, f, g in zip(params, flags, grads):
            p.requires_grad_(f)
            p.grad = g

    omega = delta[:3].detach().cpu().numpy()
    tau = delta[3:].detach().cpu().numpy()
    R = rotation_increment(torch.from_numpy(omega)).numpy() @ rotation_from_axisangle(cam.rotation_axisangle)
    # the loader's normalisation c_n = (c_world + scene_offset) * scene_scale, undone for c_n + tau
    translation = (np.asarray(cam.translation, np.float64) + tau) / scale - np.asarray(loader.scene_offset, np.float64)
    return CameraRefinement(rotation_axisangle=axisangle_of(R), translation=translation, losses=losses, omega=omega,
                            tau=tau)
