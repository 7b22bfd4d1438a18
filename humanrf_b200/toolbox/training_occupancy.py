"""Occupancy grids of the training sampler learned from the density field while it trains (``TrainingOccupancy``,
``training.FusedTrainer(training_occupancy=...)``, include/humanrf_b200.h, DESIGN.md §3.21).

A training loader marches every ray through its frame's visual hull, and every candidate inside the hull pays for the
density pass before pruning drops the ones whose alpha is below 1e-4.  ``TrainingOccupancy`` keeps a density bound for
every hull voxel of every frame the loader has loaded and, every `interval` steps from step `warmup` on, refreshes it
from the current field at one hashed point per voxel (bound = max(decay * bound, sigma)).  The grid hull AND
dilate(live), live being the bake's alpha test on the bound, is then written in place into the frame's occupancy ring
slot, where the sampler reads it.  A refreshed, dilated grid is a cached and conservative copy of the prune decision:
the candidates it culls are ones pruning would drop, up to the density gained since the last refresh and what the
hashed points and the dilation miss.

Schedule:
* before step `warmup` nothing is evaluated and every slot holds its hull: the loader's batches are those of a loader
  without a source;
* ``update(t)`` (called by FusedTrainer after step t's Adam, t = completed steps) refreshes every frame resident in the
  loader's ring when t >= warmup and (t - warmup) % interval == 0;
* after the first refresh, a frame entering the ring (``grid_added``, called by the loader) is evaluated and packed at
  once, so a frame that comes back never samples through a bound older than its entry.
Two resident frames that share one ring slot are skipped by a refresh (their slot is left as it is) and listed in
``skipped``.

Everything is enqueued on the current stream.  The one host read is the hull's voxel count, once per newly seen frame
(it sizes the frame's id list and bounds).  With two batches in flight (the batch for step k + 1 drawn before step k is
enqueued), a draw sees the grids one refresh late, as the error map's draw sees its map one step late.
"""
from __future__ import annotations

import ctypes as C
import math
import warnings

import numpy as np
import torch

from .. import _lib as L
from .learned_occupancy import ALPHA_THRE


class _FrameState:
    __slots__ = ("ids", "count", "n", "bound", "evaluations")

    def __init__(self, ids, count, n, bound, evaluations=0):
        self.ids, self.count, self.n, self.bound, self.evaluations = ids, count, n, bound, evaluations


class TrainingOccupancy:
    """Learned occupancy grids for the TRAINING `loader` (OCCUPANCY_GRID pruning) of `model`; installs itself as the
    loader's occupancy source and registers the frames already resident.

    interval: steps between refreshes (>= 1).  warmup: the first refresh's step (>= 0).  decay: weight of the old bound,
    in (0, 1].  render_step_size: the step of the alpha test (the trainer's).  seed: the points' hash seed.  rank: the
    data-parallel rank of the trainer it serves (every rank builds its own over its own loader)."""

    def __init__(self, loader, model, interval: int = 16, warmup: int = 256, decay: float = 0.95,
                 render_step_size: float = 4e-4, seed: int = 0, rank: int = 0):
        from ..dataset.data_loader import DataLoader
        from .compact_model import CompactHumanRF

        if loader.mode != DataLoader.Mode.TRAINING:
            raise ValueError(f"loader: training occupancy needs a TRAINING loader, got {loader.mode}")
        if loader.space_pruning_mode != DataLoader.SpacePruningMode.OCCUPANCY_GRID:
            raise ValueError(f"loader: training occupancy needs OCCUPANCY_GRID pruning, got {loader.space_pruning_mode}")
        if isinstance(model, CompactHumanRF):
            raise ValueError("model: a CompactHumanRF holds 8-bit tables for rendering only; training occupancy needs "
                             "the trained HumanRF")
        missing = sorted(set(int(f) for f in loader.frame_numbers) - set(int(f) for f in model.sorted_frame_numbers))
        if missing:
            raise ValueError(f"loader: frames {missing} are not frames of the model")
        G = int(loader.occupancy_grid_resolution)
        if not 1 <= G <= 1024:
            raise ValueError(f"loader: grid resolution {G} outside [1, 1024]")
        if isinstance(interval, bool) or int(interval) != interval or int(interval) < 1:
            raise ValueError(f"interval must be an integer >= 1, got {interval}")
        if isinstance(warmup, bool) or int(warmup) != warmup or int(warmup) < 0:
            raise ValueError(f"warmup must be an integer >= 0, got {warmup}")
        if not 0.0 < float(decay) <= 1.0:
            raise ValueError(f"decay must lie in (0, 1], got {decay}")
        if not (math.isfinite(float(render_step_size)) and float(render_step_size) > 0.0):
            raise ValueError(f"render_step_size must be positive and finite, got {render_step_size}")
        if int(rank) < 0:
            raise ValueError(f"rank must be non-negative, got {rank}")
        self.loader, self.model = loader, model
        self.G = G
        self.interval, self.warmup, self.decay = int(interval), int(warmup), float(decay)
        self.step = float(render_step_size)
        self.seed, self.rank = int(seed) & (2 ** 64 - 1), int(rank)
        self.device = loader.pixel_colors.device
        self.t = 0                      # the last step update() saw
        self.refreshes = 0
        self.skipped = []               # frames a refresh skipped (they shared a ring slot with another resident frame)
        self.frames = {}                # frame -> _FrameState
        self.words = (G ** 3 + 31) // 32
        self.workspace = torch.empty(int(L.lib().hrf_training_occupancy_workspace_bytes(G)), dtype=torch.uint8,
                                     device=self.device)
        for f in list(loader.frame_to_grid_texture):
            self._register(f, self._hull(f))
        loader.occupancy_source = self

    # ---------------------------------------------------------------------------------------------- frames
    @property
    def active(self) -> bool:
        """True once the first refresh ran: from then on the slots hold learned grids."""
        return self.refreshes > 0

    def _hull(self, frame: int) -> torch.Tensor:
        return torch.from_numpy(np.ascontiguousarray(self.loader.dataset.get_occupancy_grid(frame))).to(self.device)

    def _register(self, frame: int, hull: torch.Tensor) -> _FrameState:
        frame = int(frame)
        st = self.frames.get(frame)
        if st is not None:
            return st
        hull = L.require_cuda(hull, "hull", torch.uint8)
        if tuple(hull.shape) != (self.G,) * 3:
            raise ValueError(f"hull of frame {frame} has shape {tuple(hull.shape)}, expected {(self.G,) * 3}")
        lib = L.lib()
        count = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), self.G, None, count.data_ptr(),
                                                       self.workspace.data_ptr(), L.stream()))
            n = int(count.item())       # the feature's one host read: sizes the frame's ids and bounds
            ids = torch.empty(n, dtype=torch.int32, device=self.device)
            L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), self.G, L.ptr(ids), count.data_ptr(),
                                                       self.workspace.data_ptr(), L.stream()))
        st = _FrameState(ids, count, n, torch.full((n,), math.inf, dtype=torch.float32, device=self.device))
        self.frames[frame] = st
        return st

    def evaluate(self, frame: int, points: torch.Tensor = None) -> int:
        """Refreshes `frame`'s bounds from the current field (one launch); `points` (float32 [n, 3]) receives the
        evaluated points.  Returns the launch count."""
        st = self.frames[int(frame)]
        nat = self.model.native()
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_training_occupancy_update(
                C.byref(nat.field), int(frame), self.G, L.ptr(st.ids), st.count.data_ptr(), st.n, self.seed,
                st.evaluations, self.decay, L.ptr(st.bound), L.ptr(points), L.stream()))
        st.evaluations += 1
        return 1 if st.n > 0 else 0

    def _pack(self, frame: int, bits_ptr: int, counts=None, bound=None) -> int:
        st = self.frames[int(frame)]
        bound = st.bound if bound is None else bound
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_training_occupancy_pack(L.ptr(st.ids), L.ptr(bound), st.n, self.G, self.step,
                                                        ALPHA_THRE, int(bits_ptr), L.ptr(counts),
                                                        self.workspace.data_ptr(), L.stream()))
        return 3 if st.n > 0 else 2

    # ---------------------------------------------------------------------------------------------- schedule
    def grid_added(self, frame: int, hull: torch.Tensor, handle: int) -> int:
        """Loader hook: `frame` entered the ring at slot `handle` with `hull` (already packed there).  Registers the
        frame; after the first refresh also evaluates it and packs its learned grid into the slot.  Returns the launch
        count."""
        self._register(frame, hull)
        if not self.active:
            return 0
        return self.evaluate(frame) + self._pack(frame, handle)

    def update(self, t: int) -> int:
        """Called after step `t`'s optimiser update (t = steps completed).  Refreshes the resident frames when
        t >= warmup and (t - warmup) % interval == 0.  Returns the launch count."""
        self.t = int(t)
        if self.t < self.warmup or (self.t - self.warmup) % self.interval != 0:
            return 0
        return self.refresh()

    def resident(self) -> dict:
        """The loader's resident frames and their ring slots (frame -> handle), without the frames that share a slot."""
        res = {int(f): int(h) for f, h in self.loader.frame_to_grid_texture.items()}
        by_handle = {}
        for f, h in res.items():
            by_handle.setdefault(h, []).append(f)
        shared = sorted(f for fs in by_handle.values() if len(fs) > 1 for f in fs)
        if shared:
            warnings.warn(f"training occupancy: frames {shared} share a ring slot; the refresh skips them")
            self.skipped.extend(shared)
        return {f: h for f, h in res.items() if f not in shared}

    def refresh(self) -> int:
        """Evaluates and packs every resident frame now."""
        launches = 0
        for f, h in sorted(self.resident().items()):
            if f not in self.frames:
                self._register(f, self._hull(f))
            launches += self.evaluate(f) + self._pack(f, h)
        self.refreshes += 1
        return launches

    # ---------------------------------------------------------------------------------------------- inspection
    def _packed(self, frame: int, counts=None, bound=None) -> torch.Tensor:
        bits = torch.empty(self.words, dtype=torch.int32, device=self.device)
        self._pack(frame, bits.data_ptr(), counts, bound)
        return bits

    def grid(self, frame: int) -> torch.Tensor:
        """`frame`'s grid from its current bounds: uint8 [G,G,G] ([z][y][x], {0, 255}), what its slot holds after a
        pack (the hull before the frame's first evaluation)."""
        bits = self._packed(int(frame))
        shifts = torch.arange(32, dtype=torch.int32, device=self.device)
        flat = ((bits.view(-1, 1) >> shifts) & 1).view(-1)[: self.G ** 3]
        return (flat.to(torch.uint8) * 255).view(self.G, self.G, self.G)

    def stats(self) -> dict:
        """frame -> int64 [3] on the device: (live voxels, voxels of the dilated grid, hull voxels)."""
        out = {}
        for f, st in sorted(self.frames.items()):
            counts = torch.empty(2, dtype=torch.int64, device=self.device)
            self._packed(f, counts)
            out[f] = torch.cat((counts, st.count.to(torch.int64)))
        return out

    # ---------------------------------------------------------------------------------------------- state
    def state_dict(self) -> dict:
        return {"G": self.G, "seed": int(self.seed), "t": int(self.t), "refreshes": int(self.refreshes),
                "frames": {f: {"ids": st.ids.cpu(), "bound": st.bound.cpu(), "evaluations": int(st.evaluations)}
                           for f, st in sorted(self.frames.items())}}

    def load_state_dict(self, state: dict) -> None:
        """Restores every frame's ids, bounds and evaluation counter, the step and the refresh count, then rewrites the
        resident frames' slots from the restored bounds (their hulls before the first refresh).  Raises ``ValueError``
        for a state of another grid resolution, a frame the model does not have, or malformed ids or bounds."""
        if not isinstance(state, dict) or any(k not in state for k in ("G", "seed", "t", "refreshes", "frames")):
            raise ValueError("training occupancy state must be a dict with G, seed, t, refreshes and frames")
        if state["G"] != self.G:
            raise ValueError(f"training occupancy state of grid resolution {state['G']}, this one has {self.G}")
        for k in ("seed", "t", "refreshes"):
            v = state[k]
            if not (isinstance(v, int) and not isinstance(v, bool) and 0 <= v < 2 ** 64):
                raise ValueError(f"training occupancy state: {k} must be an integer in [0, 2^64)")
        model_frames = set(int(f) for f in self.model.sorted_frame_numbers)
        frames = {}
        for f, fs in dict(state["frames"]).items():
            if int(f) not in model_frames:
                raise ValueError(f"training occupancy state: frame {f} is not a frame of the model")
            ids, bound, ev = fs.get("ids"), fs.get("bound"), fs.get("evaluations")
            if not (isinstance(ids, torch.Tensor) and ids.dtype == torch.int32 and ids.dim() == 1):
                raise ValueError(f"training occupancy state: ids of frame {f} must be int32 [n]")
            if not (isinstance(bound, torch.Tensor) and bound.dtype == torch.float32 and bound.shape == ids.shape):
                raise ValueError(f"training occupancy state: bound of frame {f} must be float32 [{ids.numel()}]")
            if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= self.G ** 3
                                or bool((ids[1:] <= ids[:-1]).any())):
                raise ValueError(f"training occupancy state: ids of frame {f} must be ascending voxel indices")
            if bool(torch.isnan(bound).any()) or (bound.numel() and float(bound.min()) < 0.0):
                raise ValueError(f"training occupancy state: bound of frame {f} must be non-negative, not NaN")
            if not (isinstance(ev, int) and not isinstance(ev, bool) and ev >= 0):
                raise ValueError(f"training occupancy state: evaluations of frame {f} must be a non-negative integer")
            known = self.frames.get(int(f))
            if known is not None and not torch.equal(known.ids.cpu(), ids):
                raise ValueError(f"training occupancy state: frame {f}'s hull differs from the loader's")
            frames[int(f)] = (ids, bound, ev)
        for f, (ids, bound, ev) in frames.items():
            n = int(ids.numel())
            self.frames[f] = _FrameState(ids.to(self.device), torch.tensor([n], dtype=torch.int32, device=self.device),
                                         n, bound.to(self.device), ev)
        self.seed, self.t, self.refreshes = state["seed"], state["t"], state["refreshes"]
        for f, h in self.resident().items():
            if f not in self.frames:
                self._register(f, self._hull(f))
            st = self.frames[f]
            hull_bound = None if self.active else torch.full_like(st.bound, math.inf)
            self._pack(f, h, bound=hull_bound)
