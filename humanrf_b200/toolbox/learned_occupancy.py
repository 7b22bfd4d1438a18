"""Occupancy grids baked from a trained model's density field, for rendering.

The sampler skips space through per-frame occupancy grids.  A dataset provides visual hulls carved from foreground masks
(``occupancy_grid_generation_native.generate_from_masks``): conservative volumes that include concavities, the space
between limbs and whatever the cameras cannot rule out.  ``bake_occupancy_grid`` evaluates the trained density inside
such a hull and keeps only the voxels where pruning could keep a sample (include/humanrf_b200.h,
``hrf_bake_occupancy``), so a render evaluates far fewer candidate samples for the same image.

A grid baked once is for inference: baked from a model in training it would cull space the model has not learned yet.
For training, ``toolbox.training_occupancy.TrainingOccupancy`` refreshes learned grids from the current field every few
steps (DESIGN.md §3.21).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib as L

ALPHA_THRE = 1e-4   # the alpha threshold prune_samples / hrf_prune applies


def _check_hull(hull) -> int:
    if not isinstance(hull, torch.Tensor):
        raise RuntimeError("hull must be a torch.Tensor")
    if hull.dtype != torch.uint8:
        raise RuntimeError(f"hull has dtype {hull.dtype}, expected torch.uint8")
    if hull.dim() != 3 or not (hull.shape[0] == hull.shape[1] == hull.shape[2]):
        raise RuntimeError(f"hull must be a cubic [G,G,G] grid, got shape {tuple(hull.shape)}")
    if hull.device.type != "cuda":
        raise RuntimeError("hull must be a CUDA tensor")
    if not hull.is_contiguous():
        raise RuntimeError("hull must be contiguous")
    return int(hull.shape[0])


@torch.no_grad()
def bake_occupancy_grid(model, frame_number: int, hull: torch.Tensor, render_step_size: float = 4e-4,
                        return_max_sigma: bool = False):
    """Occupancy grid of `frame_number` baked from `model`'s density inside `hull`.

    hull: uint8 [G,G,G] CUDA tensor indexed [z][y][x], non-zero (255) = occupied, as ``OccupanyGrid.add_grid`` takes it.
    Every hull voxel is sampled at 8 sub-sample positions; it is live when the largest of their densities passes the
    alpha test prune_samples applies at `render_step_size`.  Returns uint8 [G,G,G] on the hull's device: the live voxels
    dilated by one voxel (26-neighbourhood) and limited to the hull, values {0, 255}.  With `return_max_sigma` also the
    float32 [G,G,G] volume of the per-voxel maximum density (0 outside the hull), e.g. for mesh extraction.
    Nothing is read back to the host."""
    G = _check_hull(hull)
    frame = int(frame_number)
    if frame not in model.sorted_frame_numbers:
        raise RuntimeError(f"frame {frame} is not one of the model's frames")
    nat = model.native()
    if hull.device != model.device:
        raise RuntimeError("hull and model must be on the same CUDA device")
    lib = L.lib()
    ws = torch.empty(int(lib.hrf_bake_occupancy_workspace_bytes(G)), dtype=torch.uint8, device=hull.device)
    out = torch.empty_like(hull)
    max_sigma = torch.empty(hull.shape, dtype=torch.float32, device=hull.device) if return_max_sigma else None
    L.check(lib.hrf_bake_occupancy(C.byref(nat.field), frame, hull.data_ptr(), G, float(render_step_size), ALPHA_THRE,
                                   out.data_ptr(), L.ptr(max_sigma), ws.data_ptr(), L.stream()))
    return (out, max_sigma) if return_max_sigma else out


class LearnedOccupancyDataset:
    """A dataset whose occupancy grids are baked from `model` (``bake_occupancy_grid``) out of the wrapped dataset's hulls.

    Everything but ``get_occupancy_grid`` is delegated to `dataset`.  ``get_occupancy_grid(frame_number)`` returns the
    baked grid in the type and layout datasets return (numpy uint8 [G,G,G]), baked once per frame and cached.  Hand it
    to a VALIDATION or TEST ``DataLoader`` (and through it to ``Trainer.validate`` / ``Trainer.test``) to render with
    learned grids.  It is not meant for TRAINING loaders: a model in training has not learned the space yet, and a grid
    baked from it once would cull space that the hull keeps for a reason (``TrainingOccupancy`` refreshes its grids
    while training instead).  The cache is not refreshed when the model changes;
    build a new wrapper after further training."""

    def __init__(self, dataset, model, render_step_size: float = 4e-4):
        self.dataset = dataset
        self.model = model
        self.render_step_size = float(render_step_size)
        self._grids = {}

    def __getattr__(self, name):
        if name in ("dataset", "model", "render_step_size", "_grids"):   # not set yet (e.g. during unpickling)
            raise AttributeError(name)
        return getattr(self.dataset, name)

    def get_occupancy_grid(self, frame_number):
        frame = int(frame_number)
        grid = self._grids.get(frame)
        if grid is None:
            device = self.model.device
            hull = torch.from_numpy(np.ascontiguousarray(self.dataset.get_occupancy_grid(frame_number=frame))).to(device)
            grid = bake_occupancy_grid(self.model, frame, hull, self.render_step_size).cpu().numpy()
            self._grids[frame] = grid
        return grid
