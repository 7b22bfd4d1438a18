"""Depth maps and masks of the dataset's meshes, rasterised on the GPU, and scores of rendered depth against them.

``rasterize_mesh`` runs ``hrf_rasterize_mesh`` (csrc/mesh_raster.cu, contract in include/humanrf_b200.h and DESIGN.md
§3.12): what the ActorsHQ toolbox's OpenGL mesh renderer (``renderer --depth --mask``) writes for one camera, the
camera-space z of an RDF camera and the covered pixels, but exact and deterministic, with no GL context.
``export_mesh_depth_sequence`` writes those maps in that renderer's file layout, the layout ``export_depth_sequence``
writes the model's depth in.  ``depth_scores`` runs ``hrf_depth_metrics`` (bias, MAE, RMSE, AbsRel, shares within
thresholds over the pixels both masks cover, and the masks' IoU, precision and recall), and ``evaluate_depth`` scores a
trained model's depth maps against the dataset's meshes view by view, writing ``depth.csv`` and ``depth_averages.csv``.
"""
from __future__ import annotations

import csv
import ctypes as C
import math
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import _lib as L
from ..dataset.cameras import rotation_from_axisangle
from .depth_maps import _check_camera, _check_frame, _Views, depth_path, mask_path, write_depth_exr, write_mask_png
from .geometry_metrics import _check_mesh, read_obj
from .mesh_extraction import Mesh

MAX_TAUS = 8
DEFAULT_TAUS = (0.005, 0.01, 0.02)


@dataclass
class MeshDepth:
    """One rasterised view on the device: z f32 [H,W] (camera-space z in the camera's units, 0 where nothing is
    covered), mask u8 [H,W] (255 / 0), face i32 [H,W] (the visible face, -1 where nothing is covered), hits i32 [H,W]
    (faces covering the pixel centre) or None, error i32 [1] (bit 0: a face index out of range) and skipped i64 [1]
    (faces not drawn because a vertex lies in front of `near` or implausibly far off-screen)."""
    z: torch.Tensor
    mask: torch.Tensor
    face: torch.Tensor
    hits: Optional[torch.Tensor]
    error: torch.Tensor
    skipped: torch.Tensor


def camera_projection(camera, scale: float = 1.0):
    """(world2cam, fxW, fyH, cxW, cyH) of an ActorsHQ ``CameraData``-like camera, all float64: world2cam =
    (inv(cam2world) diag(s, s, s, 1))[:3] as the mesh renderer builds its model-view matrix (vertices scaled by
    `scale`, then seen from an RDF camera), and focal length and principal point in pixels, the principal point measured
    from the image corner.  These are the factors of ``projection_matrix_world2pixel`` (dataset/cameras.py)."""
    W, H = int(camera.width), int(camera.height)
    c2w = np.eye(4)
    c2w[:3, :3] = rotation_from_axisangle(camera.rotation_axisangle)
    c2w[:3, 3] = np.asarray(camera.translation, np.float64)
    m = (np.linalg.inv(c2w) @ np.diag([scale, scale, scale, 1.0]))[:3]
    f, p = np.asarray(camera.focal_length, np.float64), np.asarray(camera.principal_point, np.float64)
    return np.ascontiguousarray(m, np.float64), W * f[0], H * f[1], W * p[0], H * p[1]


@torch.no_grad()
def rasterize_mesh(mesh: Mesh, camera, scale: float = 1.0, near: float = 0.01, far: float = 100.0,
                   hits: bool = False) -> MeshDepth:
    """The depth map and mask of `mesh` seen by `camera` (any object with ``CameraData``'s width, height,
    rotation_axisangle, translation, focal_length and principal_point; pass the dataset's own cameras, in world units,
    not a loader's normalised ones), as the ActorsHQ mesh renderer draws it with ``--scale scale``: nearest face wins,
    both windings draw, near and far clip fragments.  Faces with a vertex in front of `near` are not drawn and are
    counted in ``skipped`` (the renderer would clip them).  Nothing is synchronised."""
    _check_mesh(mesh, "mesh")
    near, far, scale = float(near), float(far), float(scale)
    if not (0 < near <= far < math.inf):
        raise RuntimeError(f"need 0 < near <= far < inf, got near {near}, far {far}")
    if not (math.isfinite(scale) and scale > 0):
        raise RuntimeError(f"scale must be finite and positive, got {scale}")
    m, fx, fy, cx, cy = camera_projection(camera, scale)
    W, H = int(camera.width), int(camera.height)
    if not np.isfinite(m).all() or not all(math.isfinite(x) for x in (fx, fy, cx, cy)):
        raise RuntimeError("the camera's projection is not finite")
    lib = L.lib()
    nv, nf = int(mesh.vertices.shape[0]), int(mesh.faces.shape[0])
    nbytes = int(lib.hrf_rasterize_mesh_workspace_bytes(nv, nf, W, H))
    if nbytes <= 0:
        raise RuntimeError(f"bad rasteriser sizes: {nv} vertices, {nf} faces, {W}x{H} pixels")
    dev = mesh.vertices.device
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    z = torch.empty((H, W), dtype=torch.float32, device=dev)
    mask = torch.empty((H, W), dtype=torch.uint8, device=dev)
    face = torch.empty((H, W), dtype=torch.int32, device=dev)
    h = torch.empty((H, W), dtype=torch.int32, device=dev) if hits else None
    error = torch.empty(1, dtype=torch.int32, device=dev)
    skipped = torch.empty(1, dtype=torch.int64, device=dev)
    m_arr = (C.c_double * 12)(*m.reshape(-1).tolist())
    with torch.cuda.device(dev):
        L.check(lib.hrf_rasterize_mesh(L.ptr(mesh.vertices) if nv else None, nv, L.ptr(mesh.faces) if nf else None, nf,
                                       m_arr, fx, fy, cx, cy, W, H, near, far, z.data_ptr(), mask.data_ptr(),
                                       face.data_ptr(), L.ptr(h), error.data_ptr(), skipped.data_ptr(), ws.data_ptr(),
                                       L.stream()))
    return MeshDepth(z, mask, face, h, error, skipped)


def _camera_name(cameras, c: int) -> str:
    """``camera_name``'s rule over a list of cameras: the camera's `name`, or ``Cam%03d`` numbered from 1."""
    name = getattr(cameras[c], "name", None)
    return str(name) if name else f"Cam{c + 1:03d}"


def _last_use(frames):
    return {f: k for k, f in enumerate(frames)}


@torch.no_grad()
def export_mesh_depth_sequence(cameras, pairs, mesh_dir, out_dir, scale: float = 1.0,
                               mesh_name: str = "Frame{:06d}.obj", near: float = 0.01, far: float = 100.0,
                               device="cuda"):
    """What ``renderer --objs ... --csv ... --depth --mask`` writes, for every (camera_number, frame_number) of `pairs`:
    ``depths/<cam>/<cam>_depth%06d.exr`` (``rasterize_mesh``'s z, float32, 0 on background) and
    ``masks/<cam>/<cam>_mask%06d.png`` (255 where covered) under `out_dir`, <cam> named as ``camera_name`` names it.
    `cameras` is the dataset's camera list (world units), the meshes are ``mesh_dir/mesh_name.format(frame)``, read
    once per frame.  Every camera, frame and file is checked before anything is written; a view with an out-of-range
    face index or a skipped face raises, naming it.  Returns the written (depth, mask) paths."""
    checked = []
    for c, f in pairs:
        c, f = int(c), int(f)
        if not 0 <= c < len(cameras):
            raise RuntimeError(f"camera {c} is not one of the {len(cameras)} cameras")
        if f < 0:
            raise RuntimeError(f"frame {f} is negative")
        checked.append((c, f))
    paths = {f: os.path.join(mesh_dir, mesh_name.format(f)) for _, f in checked}
    missing = sorted({p for p in paths.values() if not os.path.isfile(p)})
    if missing:
        raise RuntimeError(f"missing meshes: {missing}")
    last = _last_use([f for _, f in checked])
    meshes, written = {}, []
    for k, (c, f) in enumerate(checked):
        if f not in meshes:
            meshes[f] = read_obj(paths[f], device=device)
        md = rasterize_mesh(meshes[f], cameras[c], scale, near, far)
        if last[f] == k:
            del meshes[f]
        err, skipped = int(md.error.cpu()[0]), int(md.skipped.cpu()[0])
        name = _camera_name(cameras, c)
        if err or skipped:
            raise RuntimeError(f"camera {name} frame {f}: {paths[f]} has "
                               + ("face indices outside the vertex range" if err else
                                  f"{skipped} faces in front of the near plane ({near})"))
        dp, mp = depth_path(out_dir, name, f), mask_path(out_dir, name, f)
        os.makedirs(os.path.dirname(dp), exist_ok=True)
        os.makedirs(os.path.dirname(mp), exist_ok=True)
        write_depth_exr(dp, md.z)
        write_mask_png(mp, md.mask)
        written.append((dp, mp))
    return written


def _check_taus(taus):
    taus = tuple(float(t) for t in taus)
    if len(taus) > MAX_TAUS:
        raise RuntimeError(f"at most {MAX_TAUS} thresholds, got {len(taus)}")
    if any(not math.isfinite(t) or t < 0 for t in taus):
        raise RuntimeError(f"thresholds must be finite and non-negative, got {taus}")
    return taus


def _flat(t, name, dtype, n=None):
    if isinstance(t, torch.Tensor) and dtype == torch.uint8 and t.dtype == torch.bool:
        t = t.view(torch.uint8)
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"{name} must be a torch.Tensor")
    L.require_cuda(t, name, dtype)
    if n is not None and t.numel() != n:
        raise RuntimeError(f"{name} has {t.numel()} pixels, expected {n}")
    return t


def depth_scores(pred_z, pred_mask, ref_z, ref_mask, taus=DEFAULT_TAUS, out=None):
    """Scores of the depth map `pred_z` against `ref_z` over the pixels both masks cover (B), on the device without
    synchronising: z float32, masks uint8 or bool (non-zero = covered), all contiguous with the same pixel count on
    one CUDA device.  Returns ``(out, counts, error)``: out float64 [4] = (bias, MAE, RMSE, AbsRel) of pred - ref,
    counts int64 [5 + len(taus)] = (|B|, |P|, |R|, |P and R|, |P or R|, then the pixels of B with |pred - ref| <= tau),
    error int32 [1] (bit 0: a pixel of B whose z is not finite and positive).  out is NaN when B is empty or error is
    set; `out` may be given (e.g. a row of an [n,4] float64 tensor)."""
    pred_z = _flat(pred_z, "pred_z", torch.float32)
    n = pred_z.numel()
    pred_mask = _flat(pred_mask, "pred_mask", torch.uint8, n)
    ref_z = _flat(ref_z, "ref_z", torch.float32, n)
    ref_mask = _flat(ref_mask, "ref_mask", torch.uint8, n)
    dev = pred_z.device
    if any(t.device != dev for t in (pred_mask, ref_z, ref_mask)):
        raise RuntimeError("pred_z, pred_mask, ref_z and ref_mask must be on one device")
    taus = _check_taus(taus)
    if out is None:
        out = torch.empty(4, dtype=torch.float64, device=dev)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float64 or out.device != dev or out.shape != (4,)
          or not out.is_contiguous()):
        raise RuntimeError(f"out must be a contiguous float64 [4] tensor on {dev}")
    counts = torch.empty(5 + len(taus), dtype=torch.int64, device=dev)
    error = torch.empty(1, dtype=torch.int32, device=dev)
    lib = L.lib()
    nbytes = int(lib.hrf_depth_metrics_workspace_bytes(n))
    if nbytes <= 0:
        raise RuntimeError(f"bad depth map size: {n} pixels")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    tau_arr = (C.c_double * max(len(taus), 1))(*taus)
    with torch.cuda.device(dev):
        L.check(lib.hrf_depth_metrics(pred_z.data_ptr(), pred_mask.data_ptr(), ref_z.data_ptr(), ref_mask.data_ptr(), n,
                                      tau_arr, len(taus), out.data_ptr(), counts.data_ptr(), error.data_ptr(),
                                      ws.data_ptr(), L.stream()))
    return out, counts, error


@dataclass
class DepthScore:
    """One view's scores, depth in world units: n = pixels both masks cover, bias / mae / rmse / absrel of the model's
    depth minus the mesh's over them, within = share of them with |difference| <= tau per threshold, and the masks'
    iou, precision (share of the model's mask the mesh covers) and recall (share of the mesh's mask the model covers).
    camera is 0-based (``depth.csv`` numbers it from 1, as ``metrics.csv`` does)."""
    camera: int
    frame: int
    n: int
    bias: float
    mae: float
    rmse: float
    absrel: float
    taus: tuple
    within: tuple
    iou: float
    precision: float
    recall: float


def score_from(camera, frame, out, counts, taus) -> DepthScore:
    """A ``DepthScore`` from ``depth_scores``' read-back out and counts."""
    n, p, r, pr, por = (int(x) for x in counts[:5])
    div = lambda a, b: a / b if b else math.nan
    return DepthScore(int(camera), int(frame), n, *(float(x) for x in out), tuple(taus),
                      tuple(div(int(c), n) for c in counts[5:5 + len(taus)]), div(pr, por), div(pr, p), div(pr, r))


def csv_columns(taus):
    """``depth.csv``'s columns."""
    return ["camera", "frame", "n", "bias", "mae", "rmse", "absrel", *[f"within@{t:g}" for t in taus], "iou",
            "precision", "recall"]


def write_depth_tables(out_dir, scores) -> None:
    """``depth.csv`` (one row per view, in order, camera numbered from 1) and ``depth_averages.csv`` (the mean of every
    column but camera and frame)."""
    cols = csv_columns(scores[0].taus)
    rows = [[s.camera + 1, s.frame, s.n, s.bias, s.mae, s.rmse, s.absrel, *s.within, s.iou, s.precision, s.recall]
            for s in scores]
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "depth.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(cols)
        w.writerows(rows)
    with open(os.path.join(out_dir, "depth_averages.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(cols[2:])
        w.writerow([float(np.mean([r[k] for r in rows])) for k in range(2, len(cols))])


@torch.no_grad()
def evaluate_depth(model, loader, pairs, reference_dir, out_dir, taus=DEFAULT_TAUS, mask_threshold: float = 0.5,
                   bake: bool = True, reference_name: str = "Frame{:06d}.obj", scale: float = 1.0,
                   near: float = 0.01, far: float = 100.0, render_step_size: float = 4e-4,
                   rays_per_batch: int = 262144):
    """Scores the model's depth against the dataset's meshes for every (camera_number, frame_number) of `pairs`: the
    model's z and alpha from ``render_depth_map``'s renderer (each frame's hull tightened by ``bake_occupancy_grid``
    once per frame when `bake`, as ``export_depth_sequence`` does), its mask alpha >= `mask_threshold`, against
    ``rasterize_mesh`` of ``reference_dir/reference_name.format(frame)`` (read once per frame, vertices times `scale`
    in world units) for ``loader.dataset.cameras[camera]``, scored by ``depth_scores``.  Cameras, frames and files are
    checked before any work; results are read back once, and a view with an out-of-range face index, a skipped face or
    a NaN score raises, naming it, before the tables are written.  Writes ``out_dir/depth.csv`` and
    ``out_dir/depth_averages.csv``; returns a ``DepthScore`` per pair."""
    from .learned_occupancy import bake_occupancy_grid

    pairs = [(_check_camera(loader, c), _check_frame(model, f)) for c, f in pairs]
    if not pairs:
        raise RuntimeError("no (camera, frame) pairs to evaluate")
    taus = _check_taus(taus)
    cameras = loader.dataset.cameras
    paths = {f: os.path.join(reference_dir, reference_name.format(f)) for _, f in pairs}
    missing = sorted({p for p in paths.values() if not os.path.isfile(p)})
    if missing:
        raise RuntimeError(f"missing reference meshes: {missing}")
    views = _Views(model, loader, render_step_size, rays_per_batch)
    dev = views.device
    vals = torch.empty((len(pairs), 4), dtype=torch.float64, device=dev)
    cnt = torch.empty((len(pairs), 5 + len(taus)), dtype=torch.int64, device=dev)
    err = torch.empty((len(pairs), 3), dtype=torch.int64, device=dev)    # raster error, skipped, score error
    last = _last_use([f for _, f in pairs])
    grids, meshes = {}, {}
    for k, (c, frame) in enumerate(pairs):
        if frame not in grids:
            grid = views.hull(frame)
            grids[frame] = bake_occupancy_grid(model, frame, grid, render_step_size) if bake else grid
            meshes[frame] = read_obj(paths[frame], device=dev)
        dm = views.render(c, frame, grids[frame])
        ref = rasterize_mesh(meshes[frame], cameras[c], scale, near, far)
        if ref.z.shape != dm.z.shape:
            raise RuntimeError(f"camera {c}: the dataset camera is {tuple(ref.z.shape)} pixels (height x width), the "
                               f"loader's {tuple(dm.z.shape)}")
        if last[frame] == k:
            del grids[frame], meshes[frame]
        _, counts, error = depth_scores(dm.z, dm.alpha >= mask_threshold, ref.z, ref.mask, taus, out=vals[k])
        cnt[k].copy_(counts)
        err[k, 0].copy_(ref.error[0])
        err[k, 1].copy_(ref.skipped[0])
        err[k, 2].copy_(error[0])
    v, n, e = vals.cpu().numpy(), cnt.cpu().numpy(), err.cpu().numpy()
    scores = [score_from(c, f, v[k], n[k], taus) for k, (c, f) in enumerate(pairs)]
    for k, s in enumerate(scores):
        view = f"camera {s.camera} frame {s.frame}"
        if e[k, 0]:
            raise RuntimeError(f"{view}: {paths[s.frame]} has face indices outside the vertex range")
        if e[k, 1]:
            raise RuntimeError(f"{view}: {e[k, 1]} faces of {paths[s.frame]} lie in front of the near plane ({near})")
        if any(math.isnan(x) for x in (s.bias, s.mae, s.rmse, s.absrel, s.iou, s.precision, s.recall)):
            why = "a depth that is not finite and positive" if e[k, 2] else "no pixel both masks cover"
            raise RuntimeError(f"{view}: no depth score ({why})")
    write_depth_tables(out_dir, scores)
    return scores
