"""Normal maps from the renderer itself, per camera and frame.

``render_normal_map`` renders one view through ``TileShardedRenderer.render_range_maps(normals=True)``: per pixel the
unit vector N / |N| with N = sum_i w_i n_i over the samples the colour is composited from, n_i = -grad sigma_i /
|grad sigma_i| the analytic density gradient of hrf_field_position_grad.  It is returned in world coordinates (the scene
normalisation is a uniform scale plus an offset, so normalised-scene normals are world normals) and in the dataset
camera's frame (x right, y down, z forward: the convention of the depth maps).  ``export_normal_sequence`` writes the
camera-frame maps beside the depth maps' layout.

Use them to inspect learned geometry view by view, to relight it, or to compare it with the dataset's meshes.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch

from .compact_model import require_trainable
from .depth_maps import _check_camera, _check_frame, _Views, camera_name, write_depth_exr


@dataclass
class NormalMap:
    """One rendered view on the device: alpha [H,W] (weights sum) and unit normals [H,W,3] in world and camera
    coordinates, 0 where the composited normal vanishes and outside the ray mask."""
    alpha: torch.Tensor
    world: torch.Tensor
    camera: torch.Tensor


def world_to_camera_rotation(camera) -> np.ndarray:
    """R_c2w^T (float64 [3,3]) of a dataset camera: maps world directions into its RDF frame."""
    from ..dataset.cameras import rotation_from_axisangle

    return rotation_from_axisangle(np.asarray(camera.rotation_axisangle, np.float64)).T


def _render(views: _Views, camera_number: int, frame: int, grid: torch.Tensor) -> NormalMap:
    tables = views.tables(camera_number, frame, grid)
    W, H = tables["width"], tables["height"]
    _, alpha, _, world = views.renderer.render_range_maps(tables, 0, W * H, 0.0, normals=True)
    R = torch.from_numpy(world_to_camera_rotation(views.loader.cameras[camera_number])).to(world.device)
    camera = (world.double() @ R.T).float()
    return NormalMap(alpha.view(H, W), world.view(H, W, 3), camera.view(H, W, 3))


@torch.no_grad()
def render_normal_map(model, loader, camera_number: int, frame_number: int, grid=None,
                      render_step_size: float = 4e-4, rays_per_batch: int = 262144) -> NormalMap:
    """Alpha and normal maps of `model` seen from `loader`'s camera `camera_number` at `frame_number` (the view and
    `grid` as for ``render_depth_map``: the frame's hull by default, or a given uint8 [G,G,G] grid)."""
    require_trainable(model, "normal maps (they need the density's position gradient)")
    frame = _check_frame(model, frame_number)
    c = _check_camera(loader, camera_number)
    views = _Views(model, loader, render_step_size, rays_per_batch)
    return _render(views, c, frame, views.hull(frame) if grid is None else grid)


def normal_path(out_dir, name: str, frame: int) -> str:
    return os.path.join(out_dir, "normals", name, f"{name}_normal{frame:06d}.exr")


def write_normal_exr(path, normals) -> None:
    """[H,W,3] camera-frame normals as a float32 OpenEXR with x, y, z in the R, G, B channels (OpenCV writes BGR)."""
    n = np.asarray(normals.detach().cpu() if isinstance(normals, torch.Tensor) else normals, dtype=np.float32)
    write_depth_exr(path, np.ascontiguousarray(n[..., ::-1]))


@torch.no_grad()
def export_normal_sequence(model, loader, pairs, out_dir, bake: bool = True, render_step_size: float = 4e-4,
                           rays_per_batch: int = 262144):
    """For every (camera_number, frame_number) of `pairs`, writes ``normals/<cam>/<cam>_normal%06d.exr`` under `out_dir`
    (<cam> = ``camera_name``): ``render_normal_map``'s camera-frame normals, float32, x, y, z in R, G, B, 0 on
    background.  With `bake`, each frame's hull is tightened by ``bake_occupancy_grid`` first (once per frame).
    Cameras and frames are checked before anything is written.  Returns the written paths."""
    require_trainable(model, "normal maps (they need the density's position gradient)")
    from .learned_occupancy import bake_occupancy_grid

    pairs = [(_check_camera(loader, c), _check_frame(model, f)) for c, f in pairs]
    views = _Views(model, loader, render_step_size, rays_per_batch)
    grids = {}
    paths = []
    for c, frame in pairs:
        if frame not in grids:
            grid = views.hull(frame)
            grids[frame] = bake_occupancy_grid(model, frame, grid, render_step_size) if bake else grid
        nm = _render(views, c, frame, grids[frame])
        path = normal_path(out_dir, camera_name(loader, c), frame)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        write_normal_exr(path, nm.camera)
        paths.append(path)
    return paths
