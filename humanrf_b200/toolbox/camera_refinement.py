"""Camera pose refinement: one camera against a trained, frozen model (``refine_camera``), and every training camera
jointly with the field inside the fused train step (``CameraPoses``).

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
can replace the calibration's entries.  With ``intrinsics=True`` the camera's focal lengths and principal point are
refined too (below).  Per-frame poses are not refined; ``CameraPoses`` refines several cameras at once.

``CameraPoses`` gives every camera of a loader the same increment (omega_c, tau_c), learnt with the field by
``training.FusedTrainer(camera_poses=...)``.  A batch's ray r of camera c was sampled from the current tables, so
o_r = c_c + tau_c and d_r = exp([omega_c]x) d0_r (a rotation keeps unit length: the sampler's normalisation drops out).
With g_o, g_d the per-ray gradients of hrf_ray_gradients, the exact gradients of the stored increments are

    dL/dtau_c   = sum_{r in c} g_o[r]
    dL/domega_c = J_l(omega_c)^T sum_{r in c} (d_r x g_d[r]),
    J_l(w) = I + (1 - cos t)/t^2 [w]x + (t - sin t)/t^3 [w]x^2,  t = |w|   (J_l(0) = I)

(hrf_camera_pose_grad).  As in ``refine_camera``, the sampler's and the prune's choice of samples is not
differentiated.  hrf_camera_pose_step then runs Adam per camera and rewrites the loader's tables on the device.

Intrinsics (``CameraPoses(intrinsics=True)``, ``refine_camera(intrinsics=True)``, DESIGN.md §3.15): camera c also
carries alpha_c = (alpha_x, alpha_y), log focal scales, and beta_c = (beta_x, beta_y), principal-point offsets in units
of the base focal length.  A pixel's base camera coordinates u0 = K0^-1 (px, py, 1) = (x0, y0, 1) become
u' = ((x0 - beta_x) e^-alpha_x, (y0 - beta_y) e^-alpha_y, 1) and d = R' u' / |u'|: fx = fx0 e^alpha_x and
cx = cx0 + fx0 beta_x (same for y).  The sampler table is (exp([omega]x) (M0 B))^T with B = K0 A K0^-1
(``intrinsics_matrix``), so the sampler and the DataLoader are unchanged.  With q = R'^T d_r and
h = R'^T (g_d - d_r (d_r . g_d)):

    dL/dalpha_x = -sum_r q_x h_x,   dL/dbeta_x = -e^-alpha_x sum_r q_z h_x   (same for y)

(hrf_camera_calib_grad), which needs only the rays' directions, g_d and the camera's current rotation R'_c.
"""
from __future__ import annotations

import copy
import csv
import ctypes as C
import hashlib
from dataclasses import dataclass, field
from typing import Iterable, List, Optional, Sequence

import numpy as np
import torch

from .. import _lib as L


@dataclass
class CameraRefinement:
    """Refined extrinsics of one camera in the dataset's convention and world units, and the loss per iteration."""
    rotation_axisangle: np.ndarray          # [3] camera-to-world rotation, axis * angle
    translation: np.ndarray                 # [3] camera centre in world units
    losses: List[float] = field(default_factory=list)
    omega: np.ndarray = None                # [3] the rotation increment exp([omega]x) applied on the left of R
    tau: np.ndarray = None                  # [3] the centre increment, normalised scene units
    focal_length: np.ndarray = None         # [2] refined, normalised by the image size (intrinsics=True only)
    principal_point: np.ndarray = None      # [2] refined, normalised by the image size (intrinsics=True only)
    alpha: np.ndarray = None                # [2] log focal scales (intrinsics=True only)
    beta: np.ndarray = None                 # [2] principal-point offsets / base focal length (intrinsics=True only)


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


def base_intrinsics_of(cam) -> np.ndarray:
    """(fx0, fy0, cx0, cy0) in pixels of a dataset camera: focal length and principal point times the image size, as
    ``projection_matrix_world2pixel`` builds K."""
    w, h = float(cam.width), float(cam.height)
    f, p = np.asarray(cam.focal_length, np.float64), np.asarray(cam.principal_point, np.float64)
    return np.array([w * f[0], h * f[1], w * p[0], h * p[1]])


def intrinsics_matrix(alpha: torch.Tensor, beta: torch.Tensor, intrinsics) -> torch.Tensor:
    """B = K0 A K0^-1 (float64 [3,3], differentiable in alpha and beta): the map of base pixel coordinates to the pixel
    coordinates of the refined camera's ray, [[e^-ax, 0, -cx0 expm1(-ax) - fx0 bx e^-ax], [0, e^-ay, ...], [0, 0, 1]].
    `intrinsics` = (fx0, fy0, cx0, cy0).  alpha = beta = 0 gives the identity exactly."""
    alpha, beta = alpha.to(torch.float64), beta.to(torch.float64)
    fx0, fy0, cx0, cy0 = (float(v) for v in intrinsics)
    ex, ey = torch.exp(-alpha[0]), torch.exp(-alpha[1])
    b02 = -cx0 * torch.expm1(-alpha[0]) - fx0 * beta[0] * ex
    b12 = -cy0 * torch.expm1(-alpha[1]) - fy0 * beta[1] * ey
    z = torch.zeros((), dtype=torch.float64, device=alpha.device)
    one = torch.ones((), dtype=torch.float64, device=alpha.device)
    return torch.stack([torch.stack([ex, z, b02]), torch.stack([z, ey, b12]), torch.stack([z, z, one])])


def calibration_table(inverse_kr: torch.Tensor, omega: torch.Tensor, alpha: torch.Tensor, beta: torch.Tensor,
                      intrinsics) -> torch.Tensor:
    """The sampler's table of the refined view, float32 [3,3]: (exp([omega]x) (M0 B))^T with M0 = inverse_kr^T and
    B = ``intrinsics_matrix``, in float64 (M0 B formed first) before the one rounding.  alpha = beta = 0 gives
    ``view_table(inverse_kr, omega)`` bit for bit."""
    M = inverse_kr.reshape(3, 3).to(torch.float64).T @ intrinsics_matrix(alpha, beta, intrinsics)
    return (rotation_increment(omega.to(torch.float64)) @ M).T.to(torch.float32)


def refined_intrinsics(cam, alpha, beta):
    """(focal_length, principal_point) of `cam` refined by (alpha, beta), in the dataset's convention (normalised by
    the image size): focal_length * e^alpha, principal_point + focal_length * beta."""
    f, p = np.asarray(cam.focal_length, np.float64), np.asarray(cam.principal_point, np.float64)
    alpha, beta = np.asarray(alpha, np.float64), np.asarray(beta, np.float64)
    return f * np.exp(alpha), p + f * beta


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
                  render_step_size: float = 4e-4, intrinsics: bool = False,
                  intrinsics_lr: Optional[float] = None) -> CameraRefinement:
    """Refines the extrinsics of `loader`'s camera `camera_number` against its images at `frame_numbers` (read from
    ``loader.dataset``: ``get_rgb`` composited on black with ``get_mask``).  `model` is held frozen: its parameters,
    their ``requires_grad`` flags and their ``.grad`` are as they were when this returns.  Adam on the pose increment,
    learning rate decaying exponentially from `lr` to `lr * final_lr_ratio`, frames taken in turn; the pixel subsets are
    drawn from `seed`, so a run is deterministic.  Landscape images only (the loader's TEST-mode convention for the
    view's size).  `intrinsics`: also refine the camera's (alpha, beta) (module docstring), with Adam at `intrinsics_lr`
    (default `lr`) on the same schedule; the result then carries the refined focal length and principal point."""
    from .compact_model import require_trainable

    require_trainable(model, "refine_camera")
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
    k0 = base_intrinsics_of(cam)

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
    calib = torch.zeros(4, dtype=torch.float64, device=dev, requires_grad=intrinsics)     # (alpha, beta)
    groups = [{"params": [delta], "lr": lr}]
    if intrinsics:
        groups.append({"params": [calib], "lr": lr if intrinsics_lr is None else float(intrinsics_lr)})
    opt = torch.optim.Adam(groups, lr=lr)

    def table_of():
        if not intrinsics:
            return view_table(inverse_kr, delta[:3])
        return calibration_table(inverse_kr, delta[:3], calib[:2], calib[2:], k0)
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
                table = table_of()
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
            ib.ray_origins, ib.ray_directions = pixel_rays(table_of(), c0 + delta[3:], kept, W)
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
    out = CameraRefinement(rotation_axisangle=axisangle_of(R), translation=translation, losses=losses, omega=omega,
                           tau=tau)
    if intrinsics:
        ab = calib.detach().cpu().numpy()
        out.alpha, out.beta = ab[:2], ab[2:]
        out.focal_length, out.principal_point = refined_intrinsics(cam, out.alpha, out.beta)
    return out


CALIBRATION_COLUMNS = ("name", "w", "h", "rx", "ry", "rz", "tx", "ty", "tz", "fx", "fy", "px", "py")


def _camera_name(cam, c: int) -> str:
    name = getattr(cam, "name", None)
    return str(name) if name else f"Cam{c + 1:03d}"


def pose_gradients(d_origins: torch.Tensor, d_ray_directions: torch.Tensor, ray_directions: torch.Tensor,
                   camera_numbers: torch.Tensor, omega: torch.Tensor):
    """hrf_camera_pose_grad on its own: (pose_grad float32 [C,6], ray_count int32 [C]) of a ray batch, C = len(omega)
    (float64 [C,3]).  Reads the error word back and raises ``RuntimeError`` when a camera number is outside [0, C)."""
    R, C_ = int(ray_directions.shape[0]), int(omega.shape[0])
    for name, t in (("d_origins", d_origins), ("d_ray_directions", d_ray_directions), ("ray_directions", ray_directions)):
        L.require_cuda(t, name, torch.float32)
        if tuple(t.shape) != (R, 3):
            raise RuntimeError(f"{name} must be [{R}, 3], got {tuple(t.shape)}")
    L.require_cuda(camera_numbers, "camera_numbers", torch.int32)
    L.require_cuda(omega, "omega", torch.float64)
    if camera_numbers.numel() != R or tuple(omega.shape) != (C_, 3):
        raise RuntimeError("camera_numbers must hold one entry per ray and omega must be [C, 3]")
    dev = omega.device
    lib = L.lib()
    nbytes = int(lib.hrf_camera_pose_grad_workspace_bytes(C_))
    if nbytes < 0:
        raise RuntimeError(f"{C_} cameras: hrf_camera_pose_grad handles 1 to 1024")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    pose_grad = torch.empty((C_, 6), dtype=torch.float32, device=dev)
    count = torch.empty(C_, dtype=torch.int32, device=dev)
    error = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.hrf_camera_pose_grad(L.ptr(d_origins) if R else None, L.ptr(d_ray_directions) if R else None,
                                         L.ptr(ray_directions) if R else None, L.ptr(camera_numbers) if R else None, R,
                                         omega.data_ptr(), C_, pose_grad.data_ptr(), count.data_ptr(), error.data_ptr(),
                                         ws.data_ptr(), L.stream()))
    if int(error.cpu()[0]):
        raise RuntimeError(f"hrf_camera_pose_grad: a camera number outside [0, {C_})")
    return pose_grad, count


def calibration_gradients(d_origins: torch.Tensor, d_ray_directions: torch.Tensor, ray_directions: torch.Tensor,
                          camera_numbers: torch.Tensor, omega: torch.Tensor, alpha: torch.Tensor, rotations: torch.Tensor):
    """hrf_camera_calib_grad on its own: (pose_grad float32 [C,6], intrinsics_grad float32 [C,4], ray_count int32 [C])
    of a ray batch, for omega (float64 [C,3]), alpha (float64 [C,2]) and the cameras' current rotations R'_c (float32
    [C,3,3]).  Raises ``RuntimeError`` when a camera number is outside [0, C)."""
    R, C_ = int(ray_directions.shape[0]), int(omega.shape[0])
    for name, t in (("d_origins", d_origins), ("d_ray_directions", d_ray_directions), ("ray_directions", ray_directions)):
        L.require_cuda(t, name, torch.float32)
        if tuple(t.shape) != (R, 3):
            raise RuntimeError(f"{name} must be [{R}, 3], got {tuple(t.shape)}")
    L.require_cuda(camera_numbers, "camera_numbers", torch.int32)
    L.require_cuda(omega, "omega", torch.float64)
    L.require_cuda(alpha, "alpha", torch.float64)
    L.require_cuda(rotations, "rotations", torch.float32)
    if camera_numbers.numel() != R or tuple(omega.shape) != (C_, 3) or tuple(alpha.shape) != (C_, 2) \
            or tuple(rotations.shape) != (C_, 3, 3):
        raise RuntimeError("camera_numbers must hold one entry per ray, omega be [C, 3], alpha [C, 2], rotations [C, 3, 3]")
    dev = omega.device
    lib = L.lib()
    nbytes = int(lib.hrf_camera_calib_grad_workspace_bytes(C_))
    if nbytes < 0:
        raise RuntimeError(f"{C_} cameras: hrf_camera_calib_grad handles 1 to 1024")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    pose_grad = torch.empty((C_, 6), dtype=torch.float32, device=dev)
    intr_grad = torch.empty((C_, 4), dtype=torch.float32, device=dev)
    count = torch.empty(C_, dtype=torch.int32, device=dev)
    error = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.hrf_camera_calib_grad(L.ptr(d_origins) if R else None, L.ptr(d_ray_directions) if R else None,
                                          L.ptr(ray_directions) if R else None, L.ptr(camera_numbers) if R else None, R,
                                          omega.data_ptr(), alpha.data_ptr(), rotations.data_ptr(), C_,
                                          pose_grad.data_ptr(), intr_grad.data_ptr(), count.data_ptr(), error.data_ptr(),
                                          ws.data_ptr(), L.stream()))
    if int(error.cpu()[0]):
        raise RuntimeError(f"hrf_camera_calib_grad: a camera number outside [0, {C_})")
    return pose_grad, intr_grad, count


class CameraPoses:
    """Per-camera pose increments (omega_c, tau_c) of every camera of `loader`, learnt jointly with the field by
    ``FusedTrainer(camera_poses=...)``: R'_c = exp([omega_c]x) R_c, c'_c = c_c + tau_c in normalised scene units, the
    convention of ``refine_camera``.  Everything lives on the device: the increments and Adam's moments (float64), one
    Adam step counter per camera, and the base tables (the loader's ``all_inverse_krs`` / ``all_camera_origins`` when
    this object is built, i.e. omega = tau = 0).

    Each train step from `start_step` on, the step reduces its rays' gradients per camera (hrf_camera_pose_grad) and,
    after the field's Adam, runs Adam on every camera that had rays and is not fixed, rewriting ``all_inverse_krs``,
    ``all_camera_origins`` and the pool slots' ``inverse_krs_cuda`` / ``camera_origins_cuda`` on the device
    (hrf_camera_pose_step), so that the loader's next batch is sampled from the refined poses.  Draw each batch after the
    previous step has been enqueued: the gradient assumes the batch's rays come from the current tables.  The learning
    rate decays exponentially from `lr` at `start_step` to `lr * final_lr_ratio` `max_steps` steps later.

    `fixed_cameras` never move.  Moving every camera together with the scene changes no image, so the joint problem has
    no unique solution without an anchor; by default the loader's first training camera holds the gauge.  A camera
    number outside the loader's cameras in a batch stops every later pose update (the step checks a device-side error
    word) and makes ``check()`` and ``state_dict()`` raise.

    `intrinsics=True` also refines each camera's focal lengths and principal point (alpha_c, beta_c; module docstring,
    DESIGN.md §3.15) with the pose: hrf_camera_calib_grad and hrf_camera_calib_step replace the two pose kernels, Adam
    runs on (alpha, beta) at `intrinsics_lr` (decayed on the same schedule: log focal scales and offsets in focal lengths
    are not radians or scene units) and shares the camera's step counter.  It needs ``loader.cameras`` (the base
    intrinsics and rotations).  `fixed_cameras` freeze the intrinsics too.  With `intrinsics=False` nothing differs
    from the pose-only refinement: the same kernels, ``state_dict`` keys and tensors.

    Data-parallel training (DESIGN.md §3.16): build one ``CameraPoses`` per rank over that rank's loader with
    `world_size` and `process_group` set as the trainer's; the construction checks, as a collective, that every rank has
    the same cameras, base tables, fixed cameras and settings (``ValueError`` on every rank otherwise).  Each rank's step
    writes its gradient record (``pose_grad``, ``intrinsics_grad``, ``ray_count``, ``error``: views of ``record``); the
    trainer lets every rank read every record, and every rank takes the same step: the gradient is the rank-ordered sum
    over the ranks divided by `world_size`, a camera seen by any rank moves on every rank, and a bad camera number on
    any rank stops the poses on every rank (``check()`` raises everywhere).  The replicas stay bit-identical, so
    ``state_dict()`` of rank 0 is enough; ``load_state_dict()`` is called on every rank with the same state.

    Not covered: lens distortion, per-frame poses or intrinsics, and pose refinement through the autograd ``render()``
    route (``refine_camera`` does that for one camera)."""

    def __init__(self, loader, lr: float = 2e-3, final_lr_ratio: float = 1e-2, max_steps: int = 50001,
                 start_step: int = 0, fixed_cameras: Optional[Iterable[int]] = None, betas=(0.9, 0.99),
                 eps: float = 1e-15, intrinsics: bool = False, intrinsics_lr: float = 1e-3, world_size: int = 1,
                 process_group=None):
        self.loader = loader
        self.world_size, self.process_group = int(world_size), process_group
        if not 1 <= self.world_size <= L.DP_MAX_WORLD:
            raise ValueError(f"world_size {world_size} outside [1, {L.DP_MAX_WORLD}]")
        self.lr, self.final_lr_ratio, self.max_steps, self.start_step = float(lr), float(final_lr_ratio), int(max_steps), int(start_step)
        self.intrinsics, self.intrinsics_lr = bool(intrinsics), float(intrinsics_lr)
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        for name in ("all_inverse_krs", "all_camera_origins", "inverse_krs_cuda", "camera_origins_cuda", "camera_numbers_cuda"):
            if not getattr(loader, name).is_contiguous():
                raise RuntimeError(f"loader.{name} is not contiguous")
        ikr, org = loader.all_inverse_krs, loader.all_camera_origins
        n = int(ikr.shape[0])
        if tuple(ikr.shape) != (n, 3, 3) or tuple(org.shape) != (n, 3) or ikr.dtype != torch.float32 or org.dtype != torch.float32:
            raise RuntimeError("loader tables must be float32 all_inverse_krs [C,3,3] and all_camera_origins [C,3]")
        if not 1 <= n <= 1024:
            raise RuntimeError(f"{n} cameras: pose refinement handles 1 to 1024")
        dev = ikr.device
        self.device, self.num_cameras = dev, n
        self.base_inverse_krs = ikr.clone()
        self.base_camera_origins = org.clone()
        f64 = dict(dtype=torch.float64, device=dev)
        self.omega = torch.zeros((n, 3), **f64)
        self.tau = torch.zeros((n, 3), **f64)
        self.exp_avg = torch.zeros((n, 6), **f64)
        self.exp_avg_sq = torch.zeros((n, 6), **f64)
        self.steps = torch.zeros(n, dtype=torch.int32, device=dev)
        if fixed_cameras is None:
            fixed_cameras = (int(loader.camera_numbers[0]),)
        fixed = sorted({int(c) for c in fixed_cameras})
        if any(c < 0 or c >= n for c in fixed):
            raise RuntimeError(f"fixed cameras {fixed} outside [0, {n})")
        self.fixed_cameras = tuple(fixed)
        self.fixed = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.fixed[list(fixed)] = 1
        # the gradient record (include/humanrf_b200.h): pose_grad, intrinsics_grad, ray_count and the error word are
        # views of one allocation, what data-parallel ranks exchange
        self.record = torch.zeros(int(L.lib().hrf_camera_grad_record_bytes(n)), dtype=torch.uint8, device=dev)
        self._bind_record()
        ws_bytes = (L.lib().hrf_camera_calib_grad_workspace_bytes if self.intrinsics
                    else L.lib().hrf_camera_pose_grad_workspace_bytes)(n)
        self.workspace = torch.empty(int(ws_bytes), dtype=torch.uint8, device=dev)
        if self.intrinsics:
            self._init_intrinsics(loader, n, dev)
        p = L.CameraPoses()
        p.omega, p.tau, p.exp_avg, p.exp_avg_sq = (t.data_ptr() for t in (self.omega, self.tau, self.exp_avg, self.exp_avg_sq))
        p.step, p.fixed = self.steps.data_ptr(), self.fixed.data_ptr()
        p.base_inverse_krs, p.base_camera_origins = self.base_inverse_krs.data_ptr(), self.base_camera_origins.data_ptr()
        p.inverse_krs, p.camera_origins = ikr.data_ptr(), org.data_ptr()
        p.slot_inverse_krs, p.slot_camera_origins = loader.inverse_krs_cuda.data_ptr(), loader.camera_origins_cuda.data_ptr()
        p.slot_camera_numbers = loader.camera_numbers_cuda.data_ptr()
        p.num_cameras, p.num_slots = n, int(loader.camera_numbers_cuda.numel())
        self._desc = p
        self.rank = 0
        if self.world_size > 1:
            import torch.distributed as dist

            self.rank = dist.get_rank(process_group)
            self._check_replicas_agree()

    def _bind_record(self) -> None:
        n, words = self.num_cameras, self.record.view(torch.int32)
        self.pose_grad = words[:6 * n].view(torch.float32).view(n, 6)           # the last step's, before Adam
        if self.intrinsics:
            self.intrinsics_grad = words[6 * n:10 * n].view(torch.float32).view(n, 4)
        self.ray_count = words[10 * n:11 * n]
        self.error = words[11 * n:]     # sticky: bit 0, a bad camera number; bit 1, one in another rank's batch

    def _adopt_record(self, buffer: torch.Tensor) -> None:
        """Moves the gradient record into `buffer` (uint8, the record's size: peer-visible memory the other ranks read)."""
        with torch.no_grad():
            buffer.copy_(self.record)
        self.record = buffer
        self._bind_record()

    def _replica_config(self) -> dict:
        digest = lambda t: hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()   # noqa: E731
        return {"num_cameras": self.num_cameras, "base_inverse_krs": digest(self.base_inverse_krs),
                "base_camera_origins": digest(self.base_camera_origins), "fixed_cameras": self.fixed_cameras,
                "intrinsics": self.intrinsics,
                "base_intrinsics": digest(self.base_intrinsics) if self.intrinsics else None,
                "lr": self.lr, "intrinsics_lr": self.intrinsics_lr, "final_lr_ratio": self.final_lr_ratio,
                "max_steps": self.max_steps, "start_step": self.start_step, "betas": self.betas, "eps": self.eps}

    def _check_replicas_agree(self) -> None:
        """Collective over `process_group`: every rank must build the same cameras with the same settings, or their
        replicas would step apart.  Every rank gathers every rank's configuration and takes the same decision, so either
        all ranks go on or all raise ``ValueError`` naming the first field that differs."""
        import torch.distributed as dist

        mine = self._replica_config()
        configs = [None] * self.world_size
        dist.all_gather_object(configs, mine, group=self.process_group)
        for name in mine:
            values = [cfg[name] for cfg in configs]
            if any(v != values[0] for v in values):
                raise ValueError(f"CameraPoses differ between the ranks in {name}: every rank needs the same cameras "
                                 "and settings")

    def _init_intrinsics(self, loader, n: int, dev) -> None:
        from ..dataset.cameras import rotation_from_axisangle

        cams = getattr(loader, "cameras", None)
        if cams is None or len(cams) != n:
            raise RuntimeError("intrinsics=True needs loader.cameras, one per row of the loader's tables")
        f64 = dict(dtype=torch.float64, device=dev)
        self.base_intrinsics = torch.tensor(np.stack([base_intrinsics_of(cam) for cam in cams]), **f64)
        # the scene normalisation moves and scales the centres only: the rotations are the dataset's
        self.base_rotations = torch.tensor(np.stack([rotation_from_axisangle(cam.rotation_axisangle) for cam in cams]), **f64)
        self.rotations = self.base_rotations.to(torch.float32).contiguous()      # exp([omega]x) R at omega = 0
        self.alpha = torch.zeros((n, 2), **f64)
        self.beta = torch.zeros((n, 2), **f64)
        self.intrinsics_exp_avg = torch.zeros((n, 4), **f64)
        self.intrinsics_exp_avg_sq = torch.zeros((n, 4), **f64)
        q = L.CameraIntrinsics()
        q.alpha, q.beta = self.alpha.data_ptr(), self.beta.data_ptr()
        q.exp_avg, q.exp_avg_sq = self.intrinsics_exp_avg.data_ptr(), self.intrinsics_exp_avg_sq.data_ptr()
        q.base_intrinsics, q.base_rotations = self.base_intrinsics.data_ptr(), self.base_rotations.data_ptr()
        q.rotations = self.rotations.data_ptr()
        self._idesc = q

    # ---------------------------------------------------------------------------------------------- train step
    def active(self, t: int) -> bool:
        """Whether the train step after `t` completed steps refines the poses."""
        return t >= self.start_step

    def current_lr(self, t: int) -> float:
        """The learning rate of the pose step after `t` completed train steps."""
        return self.lr * self.final_lr_ratio ** min(max(t - self.start_step, 0) / max(self.max_steps, 1), 1.0)

    def current_intrinsics_lr(self, t: int) -> float:
        """The intrinsics' learning rate after `t` completed train steps (the pose's schedule, from `intrinsics_lr`)."""
        return self.intrinsics_lr * self.final_lr_ratio ** min(max(t - self.start_step, 0) / max(self.max_steps, 1), 1.0)

    def accumulate(self, d_origins, d_ray_directions, ray_directions, cameras, num_rays: int) -> int:
        """Enqueues hrf_camera_pose_grad (hrf_camera_calib_grad with intrinsics) into ``pose_grad`` / ``ray_count``
        (and ``intrinsics_grad``); no host read.  Returns the launch count."""
        if self.intrinsics:
            L.check(L.lib().hrf_camera_calib_grad(L.ptr(d_origins), L.ptr(d_ray_directions), L.ptr(ray_directions),
                                                  L.ptr(cameras), int(num_rays), self.omega.data_ptr(),
                                                  self.alpha.data_ptr(), self.rotations.data_ptr(), self.num_cameras,
                                                  self.pose_grad.data_ptr(), self.intrinsics_grad.data_ptr(),
                                                  self.ray_count.data_ptr(), self.error.data_ptr(),
                                                  self.workspace.data_ptr(), L.stream()))
            return 2 if num_rays > 0 else 1
        L.check(L.lib().hrf_camera_pose_grad(L.ptr(d_origins), L.ptr(d_ray_directions), L.ptr(ray_directions),
                                             L.ptr(cameras), int(num_rays), self.omega.data_ptr(), self.num_cameras,
                                             self.pose_grad.data_ptr(), self.ray_count.data_ptr(), self.error.data_ptr(),
                                             self.workspace.data_ptr(), L.stream()))
        return 2 if num_rays > 0 else 1

    def step(self, t: int, records: Optional[Sequence[int]] = None) -> int:
        """Enqueues hrf_camera_pose_step (hrf_camera_calib_step with intrinsics) at the learning rates of step `t`; no
        host read.  Returns the launch count.  `records`: with world_size > 1, the device addresses of every rank's
        gradient record in rank order (this rank's own or a gathered copy of it included); the step then reduces them
        (hrf_camera_pose_step_ranks / hrf_camera_calib_step_ranks) and every rank takes the same step."""
        b1, b2 = self.betas
        if records is not None:
            if len(records) != self.world_size:
                raise ValueError(f"{len(records)} gradient records for world_size {self.world_size}")
            rec = L.CameraGradRecords()
            for r, a in enumerate(records):
                rec.record[r] = a
            rec.world = self.world_size
            rec.rank = self.rank
            if self.intrinsics:
                L.check(L.lib().hrf_camera_calib_step_ranks(C.byref(self._desc), C.byref(self._idesc), C.byref(rec),
                                                            self.error.data_ptr(), self.current_lr(t),
                                                            self.current_intrinsics_lr(t), b1, b2, self.eps, L.stream()))
            else:
                L.check(L.lib().hrf_camera_pose_step_ranks(C.byref(self._desc), C.byref(rec), self.error.data_ptr(),
                                                           self.current_lr(t), b1, b2, self.eps, L.stream()))
            return 1
        if self.intrinsics:
            L.check(L.lib().hrf_camera_calib_step(C.byref(self._desc), C.byref(self._idesc), self.pose_grad.data_ptr(),
                                                  self.intrinsics_grad.data_ptr(), self.ray_count.data_ptr(),
                                                  self.error.data_ptr(), self.current_lr(t), self.current_intrinsics_lr(t),
                                                  b1, b2, self.eps, L.stream()))
            return 1
        L.check(L.lib().hrf_camera_pose_step(C.byref(self._desc), self.pose_grad.data_ptr(), self.ray_count.data_ptr(),
                                             self.error.data_ptr(), self.current_lr(t), b1, b2, self.eps, L.stream()))
        return 1

    def check(self) -> None:
        """Raises ``RuntimeError`` when a batch held a camera number outside the loader's cameras (reads the device)."""
        err = int(self.error.cpu()[0])
        if err & 1:
            raise RuntimeError(f"a train batch held a camera number outside [0, {self.num_cameras}): the poses stopped "
                               "updating at that step")
        if err:
            raise RuntimeError(f"another rank's train batch held a camera number outside [0, {self.num_cameras}): the "
                               "poses stopped updating at that step on every rank")

    # ---------------------------------------------------------------------------------------------- state
    _INTRINSICS_STATE = ("alpha", "beta", "intrinsics_exp_avg", "intrinsics_exp_avg_sq")

    def state_dict(self) -> dict:
        self.check()
        state = {"omega": self.omega.cpu(), "tau": self.tau.cpu(), "exp_avg": self.exp_avg.cpu(),
                 "exp_avg_sq": self.exp_avg_sq.cpu(), "steps": self.steps.cpu(), "fixed_cameras": list(self.fixed_cameras),
                 "base_inverse_krs": self.base_inverse_krs.cpu(), "base_camera_origins": self.base_camera_origins.cpu()}
        if self.intrinsics:
            for name in self._INTRINSICS_STATE + ("base_intrinsics",):
                state[name] = getattr(self, name).cpu()
        return state

    def load_state_dict(self, state: dict) -> None:
        """Restores increments, moments and step counters in place and rewrites the loader's tables from them.  The base
        tables must be the ones this object was built from (same dataset, same normalisation).  A pose-only state loads
        into ``intrinsics=True`` with alpha = beta = 0 and zero moments; a state with refined intrinsics does not load
        into ``intrinsics=False``."""
        names = ["base_inverse_krs", "base_camera_origins"]
        if self.intrinsics and "base_intrinsics" in state:
            names.append("base_intrinsics")
        for name in names:
            if not torch.equal(state[name].to(self.device), getattr(self, name)):
                raise RuntimeError(f"state_dict's {name} differ from the loader's: another dataset or normalisation")
        if not self.intrinsics and any(name in state and bool(torch.as_tensor(state[name]).any())
                                       for name in ("alpha", "beta")):
            raise RuntimeError("state_dict holds refined intrinsics: load it into CameraPoses(..., intrinsics=True)")
        with torch.no_grad():
            for name in ("omega", "tau", "exp_avg", "exp_avg_sq", "steps"):
                getattr(self, name).copy_(state[name])
            if self.intrinsics:
                for name in self._INTRINSICS_STATE:
                    if name in state:
                        getattr(self, name).copy_(state[name])
                    else:
                        getattr(self, name).zero_()
            fixed = sorted(int(c) for c in state["fixed_cameras"])
            self.fixed.zero_()
            self.fixed[fixed] = 1
            self.fixed_cameras = tuple(fixed)
        self._write_tables(self.loader)
        if self.intrinsics:
            with torch.no_grad():
                self.rotations.copy_(self.current_rotations())

    def current_rotations(self) -> torch.Tensor:
        """exp([omega_c]x) R_c per camera, float32 [C,3,3] (intrinsics=True): hrf_camera_calib_grad's rotations."""
        return torch.stack([rotation_increment(self.omega[c]) @ self.base_rotations[c]
                            for c in range(self.num_cameras)]).to(torch.float32).contiguous()

    def tables(self):
        """The refined sampler tables (float32 inverse_krs [C,3,3], camera_origins [C,3]), built with ``view_table``
        (``calibration_table`` with intrinsics)."""
        if self.intrinsics:
            ikr = torch.stack([calibration_table(self.base_inverse_krs[c], self.omega[c], self.alpha[c], self.beta[c],
                                                 self.base_intrinsics[c].tolist()) for c in range(self.num_cameras)])
        else:
            ikr = torch.stack([view_table(self.base_inverse_krs[c], self.omega[c]) for c in range(self.num_cameras)])
        org = (self.base_camera_origins.to(torch.float64) + self.tau).to(torch.float32)
        return ikr.contiguous(), org.contiguous()

    def _write_tables(self, loader) -> None:
        ikr, org = self.tables()
        with torch.no_grad():
            loader.all_inverse_krs.copy_(ikr)
            loader.all_camera_origins.copy_(org)
            cams = loader.camera_numbers_cuda.long()
            ok = cams >= 0
            slots = torch.nonzero(ok).view(-1)
            loader.inverse_krs_cuda[slots] = ikr[cams[slots]]
            loader.camera_origins_cuda[slots] = org[cams[slots]]

    def apply_to(self, other_loader) -> None:
        """Writes the refined tables into another loader over the same dataset (a validation or test loader): its
        ``all_inverse_krs``, ``all_camera_origins`` and the tables of the pool slots that hold a camera."""
        if tuple(other_loader.all_inverse_krs.shape) != (self.num_cameras, 3, 3):
            raise RuntimeError(f"the loader has {other_loader.all_inverse_krs.shape[0]} cameras, not {self.num_cameras}")
        if (float(other_loader.scene_scale) != float(self.loader.scene_scale)
                or not np.array_equal(np.asarray(other_loader.scene_offset), np.asarray(self.loader.scene_offset))):
            raise RuntimeError("the loader normalises the scene differently: not the same dataset")
        self._write_tables(other_loader)

    # ---------------------------------------------------------------------------------------------- export
    def refined_cameras(self) -> list:
        """Copies of the dataset's cameras with the refined extrinsics in the dataset's convention and world units
        (``rotation_axisangle`` of the camera-to-world rotation, ``translation`` of the centre: the loader's
        normalisation undone, as ``refine_camera`` does).  With intrinsics, ``focal_length`` and ``principal_point`` are
        the refined ones (``refined_intrinsics``); otherwise they are copied through."""
        from ..dataset.cameras import rotation_from_axisangle

        omega, tau = self.omega.cpu().numpy(), self.tau.cpu().numpy()
        if self.intrinsics:
            alpha, beta = self.alpha.cpu().numpy(), self.beta.cpu().numpy()
        scale = float(self.loader.scene_scale)
        offset = np.asarray(self.loader.scene_offset, np.float64)
        out = []
        for c, cam in enumerate(self.loader.cameras):      # the loader's cameras: normalised centres, omega = tau = 0
            rc = copy.deepcopy(cam)
            R = rotation_increment(torch.from_numpy(omega[c])).numpy() @ rotation_from_axisangle(cam.rotation_axisangle)
            rc.rotation_axisangle = axisangle_of(R)
            rc.translation = (np.asarray(cam.translation, np.float64) + tau[c]) / scale - offset
            if self.intrinsics:
                rc.focal_length, rc.principal_point = refined_intrinsics(cam, alpha[c], beta[c])
            out.append(rc)
        return out

    def write_calibration_csv(self, path) -> None:
        """The refined cameras as an ActorsHQ ``calibration.csv`` (columns name,w,h,rx,ry,rz,tx,ty,tz,fx,fy,px,py; one row
        per camera; focal length and principal point normalised by the image size, as the dataset's)."""
        with open(path, "w", newline="") as fh:
            w = csv.writer(fh)
            w.writerow(CALIBRATION_COLUMNS)
            for c, cam in enumerate(self.refined_cameras()):
                r, t = np.asarray(cam.rotation_axisangle, np.float64), np.asarray(cam.translation, np.float64)
                f, p = np.asarray(cam.focal_length, np.float64), np.asarray(cam.principal_point, np.float64)
                w.writerow([_camera_name(cam, c), int(cam.width), int(cam.height)]
                           + [repr(float(x)) for x in (*r, *t, *f, *p)])

