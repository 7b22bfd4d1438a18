"""Depth and opacity maps from the renderer itself, per camera and frame.

``render_depth_map`` renders one view through ``TileShardedRenderer.render_range_maps`` (the fused render kernel's depth
variant, include/humanrf_b200.h ``hrf_render_fused_depth``) and converts the expected ray distance into the camera-space
depth along the optical axis, in world units: the quantity the ActorsHQ toolbox's mesh renderer writes
(``depth = position_cam.z`` with an RDF camera, 0 on background).  ``export_depth_sequence`` writes those maps and the
thresholded opacity in that renderer's file layout.  ``toolbox/mesh_depth.py`` writes the dataset meshes' maps in the
same layout (``export_mesh_depth_sequence``) and scores the two against each other (``evaluate_depth``).

Unlike a mesh (``toolbox/mesh_extraction.py``) the depth needs no iso-level: it is the weight-averaged distance of what
the model renders, pixel for pixel aligned with its colour image.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch


@dataclass
class DepthMap:
    """One rendered view, [H,W] maps on the device: colour [H,W,3] (background 0), alpha (weights sum), distance along
    the ray and z (camera-space depth along the optical axis), both in world units and 0 where alpha is 0."""
    color: torch.Tensor
    alpha: torch.Tensor
    distance: torch.Tensor
    z: torch.Tensor


def pixel_ray_norms(inverse_kr: torch.Tensor, width: int, height: int) -> torch.Tensor:
    """|v| per pixel, float64 [height*width] in row-major pixel order, with v = M [px, py, 1], px = x + 0.5, py = y + 0.5
    and M = inv(world2pixel)[:3,:3]; `inverse_kr` is the loader's table (M transposed, float32 [3,3]), the one the
    sampler builds its ray directions from.  The camera-frame z of v is exactly 1, so a point at distance s along the
    normalised direction v / |v| has camera z = s / |v|."""
    T = inverse_kr.reshape(3, 3).to(torch.float64)
    dev = T.device
    px = torch.arange(width, dtype=torch.float64, device=dev) + 0.5
    py = torch.arange(height, dtype=torch.float64, device=dev) + 0.5
    v = px.view(1, -1, 1) * T[0] + py.view(-1, 1, 1) * T[1] + T[2]
    return torch.linalg.vector_norm(v, dim=-1).reshape(-1)


def camera_name(loader, camera_number: int) -> str:
    """The camera's `name`, or ``Cam%03d`` numbered from 1 (actorshq/evaluation's convention) when it has none."""
    name = getattr(loader.cameras[camera_number], "name", None)
    return str(name) if name else f"Cam{camera_number + 1:03d}"


def _check_frame(model, frame_number) -> int:
    frame = int(frame_number)
    if frame not in model.sorted_frame_numbers:
        raise RuntimeError(f"frame {frame} is not one of the model's frames")
    return frame


def _check_camera(loader, camera_number) -> int:
    c = int(camera_number)
    if not 0 <= c < len(loader.cameras):
        raise RuntimeError(f"camera {c} is not one of the loader's {len(loader.cameras)} cameras")
    return c


class _Views:
    """Sampler tables of a loader's cameras and one occupancy-grid slot, shared by the views of an export."""

    def __init__(self, model, loader, render_step_size: float, rays_per_batch: int):
        from ..parallel import TileShardedRenderer

        self.loader, self.device = loader, loader.aabb.device
        self.og, self.G = None, 0
        self.renderer = TileShardedRenderer(model, None, rays_per_batch=rays_per_batch, step=render_step_size)

    def hull(self, frame: int) -> torch.Tensor:
        return torch.from_numpy(np.ascontiguousarray(self.loader.dataset.get_occupancy_grid(frame_number=frame))).to(self.device)

    def tables(self, camera_number: int, frame: int, grid: torch.Tensor) -> dict:
        """The renderer's per-image tables of one view (``TileShardedRenderer.render_range``'s `cam`)."""
        from ..dataset.occupancy_grid_native import OccupanyGrid

        dl, dev = self.loader, self.device
        if (not isinstance(grid, torch.Tensor) or grid.dtype != torch.uint8 or grid.device != dev or grid.dim() != 3
                or not grid.shape[0] == grid.shape[1] == grid.shape[2]):
            raise RuntimeError(f"grid must be a cubic uint8 [G,G,G] tensor on {dev}")
        if self.og is None or self.G != grid.shape[0]:
            self.G = int(grid.shape[0])
            self.og = self.renderer.og = OccupanyGrid(self.G, 1)
        cam = dl.cameras[camera_number]
        W, H = int(cam.width), int(cam.height)
        tables = dict(frame_numbers=torch.tensor([frame], dtype=torch.int32, device=dev),
                      camera_numbers=torch.tensor([camera_number], dtype=torch.int32, device=dev),
                      grid_handles=torch.tensor([self.og.add_grid(grid.contiguous())], dtype=torch.int64, device=dev),
                      # the image's own width and height (the DataLoader's TEST mode does the same for portrait cameras)
                      landscape=torch.tensor([True], device=dev),
                      inverse_krs=dl.all_inverse_krs[camera_number:camera_number + 1].contiguous(),
                      camera_origins=dl.all_camera_origins[camera_number:camera_number + 1].contiguous(),
                      aabb=dl.aabb, G=self.G, width=W, height=H)
        return tables

    def render(self, camera_number: int, frame: int, grid: torch.Tensor) -> DepthMap:
        dl = self.loader
        tables = self.tables(camera_number, frame, grid)
        W, H = tables["width"], tables["height"]
        color, alpha, dist = self.renderer.render_range_maps(tables, 0, W * H, 0.0)
        scale = float(dl.scene_scale)
        norms = pixel_ray_norms(dl.all_inverse_krs[camera_number], W, H)
        distance = (dist.double() / scale).float()
        z = (dist.double() / (norms * scale)).float()
        return DepthMap(color.view(H, W, 3), alpha.view(H, W), distance.view(H, W), z.view(H, W))


@torch.no_grad()
def render_depth_map(model, loader, camera_number: int, frame_number: int, grid=None,
                     render_step_size: float = 4e-4, rays_per_batch: int = 262144) -> DepthMap:
    """Colour, alpha, distance and z maps of `model` seen from `loader`'s camera `camera_number` at `frame_number`.
    `loader` is a DataLoader (its cameras, ``all_inverse_krs``, ``all_camera_origins``, ``aabb`` and ``scene_scale`` give
    the view); the sampler skips space outside `grid`, by default the frame's hull from
    ``loader.dataset.get_occupancy_grid``, or a given uint8 [G,G,G] grid such as ``bake_occupancy_grid``'s."""
    frame = _check_frame(model, frame_number)
    c = _check_camera(loader, camera_number)
    views = _Views(model, loader, render_step_size, rays_per_batch)
    return views.render(c, frame, views.hull(frame) if grid is None else grid)


def write_depth_exr(path, z) -> None:
    """Single-channel float32 OpenEXR through OpenCV, the writer the ActorsHQ renderer uses."""
    # OpenCV reads this switch once, at its first EXR call: it has to be set before that call
    os.environ.setdefault("OPENCV_IO_ENABLE_OPENEXR", "1")
    import cv2

    img = np.ascontiguousarray(np.asarray(z.detach().cpu() if isinstance(z, torch.Tensor) else z, dtype=np.float32))
    try:
        ok = cv2.imwrite(str(path), img, [cv2.IMWRITE_EXR_TYPE, cv2.IMWRITE_EXR_TYPE_FLOAT])
    except cv2.error as e:
        raise RuntimeError(f"writing {path} failed (is OpenCV's OpenEXR codec enabled?): {e}") from e
    if not ok:
        raise RuntimeError(f"writing {path} failed (is OpenCV's OpenEXR codec enabled?)")


def write_mask_png(path, mask) -> None:
    """Single-channel 8-bit PNG, 255 where `mask` is true."""
    import cv2

    m = np.asarray(mask.detach().cpu() if isinstance(mask, torch.Tensor) else mask, dtype=bool)
    if not cv2.imwrite(str(path), np.ascontiguousarray(m.astype(np.uint8) * 255)):
        raise RuntimeError(f"writing {path} failed")


def depth_path(out_dir, name: str, frame: int) -> str:
    return os.path.join(out_dir, "depths", name, f"{name}_depth{frame:06d}.exr")


def mask_path(out_dir, name: str, frame: int) -> str:
    return os.path.join(out_dir, "masks", name, f"{name}_mask{frame:06d}.png")


@torch.no_grad()
def export_depth_sequence(model, loader, pairs, out_dir, bake: bool = True, mask_threshold: float = 0.5,
                          render_step_size: float = 4e-4, rays_per_batch: int = 262144):
    """For every (camera_number, frame_number) of `pairs`, writes the ActorsHQ mesh renderer's layout under `out_dir`:
    ``depths/<cam>/<cam>_depth%06d.exr`` (``render_depth_map``'s z, float32, 0 on background) and
    ``masks/<cam>/<cam>_mask%06d.png`` (255 where alpha >= `mask_threshold`), <cam> = ``camera_name``.  With `bake`, each
    frame's hull is tightened by ``bake_occupancy_grid`` first (once per frame).  Cameras and frames are checked before
    anything is written.  Returns the written (depth, mask) paths."""
    from .learned_occupancy import bake_occupancy_grid

    pairs = [(_check_camera(loader, c), _check_frame(model, f)) for c, f in pairs]
    views = _Views(model, loader, render_step_size, rays_per_batch)
    grids = {}
    paths = []
    for c, frame in pairs:
        if frame not in grids:
            grid = views.hull(frame)
            grids[frame] = bake_occupancy_grid(model, frame, grid, render_step_size) if bake else grid
        dm = views.render(c, frame, grids[frame])
        name = camera_name(loader, c)
        dp, mp = depth_path(out_dir, name, frame), mask_path(out_dir, name, frame)
        os.makedirs(os.path.dirname(dp), exist_ok=True)
        os.makedirs(os.path.dirname(mp), exist_ok=True)
        write_depth_exr(dp, dm.z)
        write_mask_png(mp, dm.alpha >= mask_threshold)
        paths.append((dp, mp))
    return paths
