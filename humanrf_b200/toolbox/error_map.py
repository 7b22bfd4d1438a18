"""Error map of the training pool: draw training rays where the loss is high (``ErrorMap``,
``training.FusedTrainer(error_map=...)``, DESIGN.md §3.20).

Uniform ray sampling spends most of a batch where the field has already converged (background, smooth regions of the
body).  The error map keeps, for every image in the loader's GPU pool, a running per-tile colour error: each fused train
step adds its rays' Huber errors into their pixels' tiles (hrf_error_map_accumulate) and folds the step's tile means into
an exponential moving average (hrf_error_map_update, which also rebuilds the integer CDF of the tile weights
max(ema, floor) * npix).  The loader then draws each batch's pool indices from that CDF (hrf_error_map_draw): a share
`uniform_fraction` of every batch stays uniform over the pool's pixels, the rest picks a tile by its weight and a pixel
uniformly inside it.  The loss is not reweighted (as in Instant-NGP): the error map shifts the loss towards hard pixels.

A newly loaded image starts at `prior` (1.0, above any Huber value) on every tile, so the pool starts out drawing
uniformly by pixel count and new images are explored first.  The reset writes the slot's EMA only; the next train
step's update rebuilds the CDF, so the draw in the same ``next()`` as the reload still sees the slot's previous image.
Everything lives on the device; no call reads it back.

With two batches in flight (the batch for step k + 1 drawn before step k is enqueued), a draw sees the map as of the last
update enqueued before it: one step behind what a serial loop sees.  There, ``next()`` for batch k + 1 may also reload a
slot that step k's rays were drawn from; step k then adds the previous image's errors into the new image's reset tiles.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _lib as L


class ErrorMap:
    """Per-tile error map over the pool of a TRAINING `loader`; installs itself as the loader's ray source.

    tile: tile edge T in pixels (1..4096).  uniform_fraction: share of every batch drawn uniformly (floor(f R) rays).
    beta: EMA weight of a step's tile mean.  floor: least EMA a tile's weight uses (>= 2^-24, so every tile can be drawn).
    prior: EMA of the tiles of a newly loaded image.  seed, rank: the draws hash (seed + rank, draw counter, ray); every
    data-parallel rank owns its loader, pool and map, and no collective is involved."""

    def __init__(self, loader, tile: int = 16, uniform_fraction: float = 0.25, beta: float = 0.5, floor: float = 1e-5,
                 prior: float = 1.0, seed: int = 0, rank: int = 0):
        from ..dataset.data_loader import DataLoader

        if loader.mode != DataLoader.Mode.TRAINING:
            raise ValueError(f"an error map needs a TRAINING loader, got {loader.mode}")
        if int(tile) != tile or not 1 <= int(tile) <= 4096:
            raise ValueError(f"tile must be an integer in [1, 4096], got {tile}")
        if not 0.0 <= float(uniform_fraction) <= 1.0:
            raise ValueError(f"uniform_fraction must lie in [0, 1], got {uniform_fraction}")
        if not 0.0 < float(beta) <= 1.0:
            raise ValueError(f"beta must lie in (0, 1], got {beta}")
        if not (math.isfinite(float(floor)) and float(floor) >= 2.0 ** -24):
            raise ValueError(f"floor must be finite and at least 2^-24, got {floor}")
        if not (math.isfinite(float(prior)) and float(prior) >= 0.0):
            raise ValueError(f"prior must be finite and non-negative, got {prior}")
        if int(rank) < 0:
            raise ValueError(f"rank must be non-negative, got {rank}")
        self.loader = loader
        self.tile, self.uniform_fraction = int(tile), float(uniform_fraction)
        self.beta, self.floor, self.prior = float(beta), float(floor), float(prior)
        self.seed, self.rank, self.counter = int(seed) & (2 ** 64 - 1), int(rank), 0
        self.device = loader.pixel_colors.device
        width, height = loader.resolution
        g = L.ErrorMapGeometry()
        g.landscape_modes = loader.landscape_mode_cuda.data_ptr()
        g.num_slots, g.image_width, g.image_height, g.tile = loader.buffer_size, width, height, self.tile
        self._geometry = g
        lib = L.lib()
        n = int(lib.hrf_error_map_num_tiles(C.byref(g), max(self.prior, self.floor)))
        if n < 1:
            raise ValueError(f"a pool of {loader.buffer_size} x {width}x{height} pixels in {self.tile}-pixel tiles could "
                             "overflow the 64-bit tile weights")
        self.num_tiles = n
        self.tiles_per_slot = n // loader.buffer_size
        dev = self.device
        self.ema = torch.full((n,), self.prior, dtype=torch.float32, device=dev)
        self.tile_sum = torch.zeros(n, dtype=torch.int64, device=dev)     # uint64 in the kernels
        self.tile_count = torch.zeros(n, dtype=torch.int32, device=dev)   # uint32 in the kernels
        self.cdf = torch.empty(n, dtype=torch.int64, device=dev)          # uint64 in the kernels
        self.error = torch.zeros(1, dtype=torch.int32, device=dev)
        self.workspace = torch.empty(int(lib.hrf_error_map_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        self.update()
        loader.ray_source = self

    # ---------------------------------------------------------------------------------------------- geometry
    @property
    def geometry(self) -> dict:
        g = self._geometry
        return {"num_slots": int(g.num_slots), "image_width": int(g.image_width), "image_height": int(g.image_height),
                "tile": int(g.tile)}

    # ---------------------------------------------------------------------------------------------- train step
    def accumulate(self, color, weights_sum, rgba, background, pixels, num_rays: int, huber_delta: float,
                   response_table=None, cameras=None) -> int:
        """Enqueues hrf_error_map_accumulate on the step's [R] buffers (`pixels` int64, the batch's pool indices).
        `response_table` (and `cameras`): the camera responses the loss went through.  Returns the launch count."""
        num_cameras = 0 if response_table is None else int(response_table.shape[0])
        L.check(L.lib().hrf_error_map_accumulate(
            L.ptr(color), L.ptr(weights_sum), L.ptr(rgba), L.ptr(background), L.ptr(pixels), int(num_rays),
            L.ptr(response_table), L.ptr(cameras), num_cameras, float(huber_delta), C.byref(self._geometry),
            self.tile_sum.data_ptr(), self.tile_count.data_ptr(), self.error.data_ptr(), L.stream()))
        return 1 if num_rays > 0 else 0

    def update(self) -> int:
        """Enqueues hrf_error_map_update: the accumulated tile means into the EMA, and the CDF rebuilt."""
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_error_map_update(C.byref(self._geometry), self.ema.data_ptr(), self.tile_sum.data_ptr(),
                                                 self.tile_count.data_ptr(), self.beta, self.floor, self.cdf.data_ptr(),
                                                 self.workspace.data_ptr(), L.stream()))
        return 3

    # ---------------------------------------------------------------------------------------------- loader hooks
    def draw(self, batch_size: int) -> torch.Tensor:
        """The next batch's pool indices, int64 [batch_size] on the device (hrf_error_map_draw); no host read."""
        out = torch.empty(int(batch_size), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_error_map_draw(self.cdf.data_ptr(), C.byref(self._geometry),
                                               (self.seed + self.rank) & (2 ** 64 - 1), self.counter, int(batch_size),
                                               self.uniform_fraction, out.data_ptr(), L.stream()))
        self.counter += 1
        return out

    def reset_slot(self, slot: int) -> None:
        """The loader reloaded pool slot `slot`: its tiles restart at `prior` (one launch over the slot's tiles).  The
        CDF is rebuilt by the next train step's update, so the draw made right after the reload still weighs the slot by
        its previous image's errors."""
        if not 0 <= int(slot) < int(self._geometry.num_slots):
            raise ValueError(f"slot {slot} outside the pool's [0, {int(self._geometry.num_slots)})")
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_error_map_reset_slots(C.byref(self._geometry), int(slot), 1, self.prior,
                                                      self.ema.data_ptr(), L.stream()))

    # ---------------------------------------------------------------------------------------------- inspection
    def check(self) -> None:
        """Raises ``RuntimeError`` when a train step passed a pool index outside the pool (reads the device)."""
        if int(self.error.cpu()[0]) != 0:
            raise RuntimeError("a train step passed a pixel index outside the pool to the error map: those rays were "
                               "skipped")

    def tile_errors(self) -> torch.Tensor:
        """The running tile errors, float32 [slots, tiles_per_slot] (row-major tiles in each slot's orientation)."""
        return self.ema.view(-1, self.tiles_per_slot).clone()

    def sampling_density(self) -> torch.Tensor:
        """Probability that one ray of a batch lands in each tile, float64 [slots, tiles_per_slot]: uniform_fraction
        times the tile's pixel share plus the rest times its CDF weight share (the uniform share is floor(f R) of R rays,
        so this is exact for batches where f R is an integer)."""
        cdf = self.cdf.cpu().numpy().view("uint64").astype("float64")
        w = torch.from_numpy(cdf.copy())
        w[1:] -= torch.from_numpy(cdf[:-1].copy())
        g = self.geometry
        W, H, T = g["image_width"], g["image_height"], g["tile"]
        shapes = {True: tile_pixel_counts(W, H, T), False: tile_pixel_counts(H, W, T)}
        npix = torch.from_numpy(np.concatenate([shapes[bool(ls)] for ls in self.loader.landscape_mode_cuda.cpu()]))
        share = npix.double() / (g["num_slots"] * W * H)
        f = self.uniform_fraction
        return (f * share + (1 - f) * w / float(cdf[-1])).view(-1, self.tiles_per_slot)

    # ---------------------------------------------------------------------------------------------- state
    def state_dict(self) -> dict:
        self.check()
        return {"ema": self.ema.cpu(), "counter": int(self.counter), "seed": int(self.seed), "geometry": self.geometry}

    def load_state_dict(self, state: dict) -> None:
        """Restores the tile errors, the draw counter and the seed, and rebuilds the CDF.  Raises ``ValueError`` for a
        state of another pool geometry or with tile errors that are not finite or outside [0, max(prior, 1)]."""
        if not isinstance(state, dict) or any(k not in state for k in ("ema", "counter", "seed", "geometry")):
            raise ValueError("error map state must be a dict with ema, counter, seed and geometry")
        if not isinstance(state["geometry"], dict) or dict(state["geometry"]) != self.geometry:
            raise ValueError(f"error map state of geometry {state.get('geometry')}, this map has {self.geometry}")
        ema = state["ema"]
        if not isinstance(ema, torch.Tensor) or ema.dtype != torch.float32 or tuple(ema.shape) != (self.num_tiles,):
            raise ValueError(f"error map state: ema must be float32 [{self.num_tiles}]")
        top = max(float(np.float32(self.prior)), 1.0)
        if not bool(torch.isfinite(ema).all()) or float(ema.min()) < 0.0 or float(ema.max()) > top:
            raise ValueError(f"error map state: tile errors must be finite and in [0, {top}]")
        counter, seed = state["counter"], state["seed"]
        if not all(isinstance(v, int) and not isinstance(v, bool) and 0 <= v < 2 ** 64 for v in (counter, seed)):
            raise ValueError("error map state: counter and seed must lie in [0, 2^64)")
        with torch.no_grad():
            self.ema.copy_(ema)
            self.tile_sum.zero_()
            self.tile_count.zero_()
        self.counter, self.seed = counter, seed
        self.update()


def tile_pixel_counts(width: int, height: int, tile: int):
    """npix of every tile of a slot `width` pixels wide and `height` high, in the kernels' row-major tile order: int64
    [ceil(height / tile) * ceil(width / tile)].  A portrait slot of a W x H pool is H wide and W high."""
    cw = np.minimum(tile, width - np.arange(0, width, tile))
    ch = np.minimum(tile, height - np.arange(0, height, tile))
    return (ch[:, None] * cw[None, :]).reshape(-1).astype(np.int64)
