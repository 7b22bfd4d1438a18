"""Per-camera colour response (gain and offset per channel) learnt with the field in the fused train step
(``CameraResponses``, ``training.FusedTrainer(camera_responses=...)``, DESIGN.md §3.17).

Multi-camera captures differ in exposure and white balance.  Without a model of that, the field bakes every camera's
colour differences into its radiance as view-dependent colour.  Camera c gets a per-channel log gain gamma_c and offset
b_c; the field learns one canonical radiance, and the response explains how camera c recorded it.  With the render's
colour `color`, opacity w (weights_sum) and the trainer's random background bg (never seen by a camera), the response
acts on the foreground fg = color - (1 - w) bg only:

    pred = e^gamma fg + w b + (1 - w) bg  =  color + expm1(gamma) fg + w b
    dpred/dcolor = e^gamma,  dpred/dw = expm1(gamma) bg + b,  dpred/dgamma = e^gamma fg,  dpred/db = w

The Huber term of the loss is taken on pred - gt, the mask's BCE term is unchanged (hrf_train_loss_response).  At
gamma = b = 0 the loss kernel writes hrf_train_loss's bytes.  After the field's Adam, hrf_camera_response_step runs
Adam (float64) on every camera that had rays and is not fixed.  The response exports as 6 numbers per camera
(``gains()``, ``offsets()``, ``write_response_csv``) and can be applied to a render afterwards (``apply``).

Cameras that were never trained (held-out test cameras) get their response from a closed-form least-squares fit
against the frozen model on frames the evaluation does not score (``held_out_fit_pairs``,
``CameraResponses.fit_held_out``, DESIGN.md §3.18).
"""
from __future__ import annotations

import csv
import ctypes as C
import hashlib
import math
from dataclasses import dataclass
from typing import Iterable, Optional, Sequence

import numpy as np
import torch

from .. import _lib as L

RESPONSE_COLUMNS = ("name", "gain_r", "gain_g", "gain_b", "offset_r", "offset_g", "offset_b")
FIT_COLUMNS = ("name", "fit_views", "n", "gain_r", "gain_g", "gain_b", "offset_r", "offset_g", "offset_b",
               "psnr_before", "psnr_after")
FIT_ROW = 17            # moments per camera: n, S_aa, per channel S_ff, S_fa, S_fy, S_ay, S_yy
FIT_STATUS = {1: "fewer fit pixels than min_pixels", 2: "the fit is not finite (gain and offset cannot be told apart)",
              3: "the fitted gain is not positive", 4: "camera outside the responses' cameras"}


@dataclass
class ResponseFit:
    """One held-out camera's fit: its fit frames, the number of fit pixels, the gain and offset per channel, and the
    masked PSNR (dB) of the float render against the dataset's colour over the fit pixels, before and after the fit."""
    camera: int
    frames: tuple
    n: int
    gain: tuple
    offset: tuple
    psnr_before: float
    psnr_after: float


def held_out_fit_pairs(score_pairs, frame_numbers, per_camera: int = 8) -> list:
    """(camera, frame) pairs to fit held-out responses on: for each camera of `score_pairs` (in order of first
    appearance), `per_camera` of `frame_numbers` spread evenly (``np.round(np.linspace(0, n - 1, per_camera))``, the
    rounding of the ActorsHQ presets' ``get_spaced_elements``) over the frames that camera is NOT scored on, or all of
    them when there are fewer.  No returned pair is a scored pair."""
    if per_camera < 1:
        raise ValueError(f"per_camera must be at least 1, got {per_camera}")
    scored, order = {}, []
    for c, f in score_pairs:
        c = int(c)
        if c not in scored:
            scored[c] = set()
            order.append(c)
        scored[c].add(int(f))
    frames = list(dict.fromkeys(int(f) for f in frame_numbers))
    out = []
    for c in order:
        spare = [f for f in frames if f not in scored[c]]
        if len(spare) <= per_camera:
            picked = spare
        else:
            idx = np.round(np.linspace(0, len(spare) - 1, per_camera)).astype(int)
            picked = [spare[i] for i in dict.fromkeys(idx.tolist())]
        out.extend((c, f) for f in picked)
    return out


def _masked_psnr(sse: float, n: int) -> float:
    mse = sse / (3 * n)
    return math.inf if mse <= 0 else -10.0 * math.log10(mse)


class CameraResponses:
    """Per-camera colour responses (gamma_c, b_c) of every camera of `loader` (``loader.all_inverse_krs`` gives the camera
    count), learnt jointly with the field by ``FusedTrainer(camera_responses=...)``.  Everything lives on the device:
    the parameters and Adam's moments (float64 [C,6]: gamma rgb, b rgb), one Adam step counter per camera, and the
    table the loss kernel reads (float32 [C,6]: expm1(gamma), b).

    Each train step from `start_step` on computes the loss through the response of each ray's camera and reduces the
    response gradient per camera; after the field's Adam, every camera that had rays and is not fixed takes one Adam step.
    The learning rate decays exponentially from `lr` at `start_step` to `lr * final_lr_ratio` `max_steps` steps later;
    the default lr is the one the recovery test converges with (DESIGN.md §3.17).

    `fixed_cameras` keep the identity.  Scaling every camera's gain and the field's radiance inversely changes no
    prediction, so the problem has no unique solution without an anchor; by default the loader's first training camera
    holds the gauge.  A camera number outside [0, C) in a batch stops every later response update and makes ``check()``
    and ``state_dict()`` raise.

    Data-parallel training: build one per rank with the trainer's `world_size` and `process_group`; construction checks,
    as a collective, that every rank has the same cameras and settings (``ValueError`` on every rank otherwise).  The
    ranks exchange their gradient records (``record``; ``response_grad``, ``ray_count`` and ``error`` are views of it)
    and every rank takes the same step (hrf_camera_response_step_ranks), so the replicas stay bit-identical."""

    def __init__(self, loader, lr: float = 5e-3, final_lr_ratio: float = 1e-2, max_steps: int = 50001,
                 start_step: int = 0, fixed_cameras: Optional[Iterable[int]] = None, betas=(0.9, 0.99),
                 eps: float = 1e-15, world_size: int = 1, process_group=None):
        self.loader = loader
        self.world_size, self.process_group = int(world_size), process_group
        if not 1 <= self.world_size <= L.DP_MAX_WORLD:
            raise ValueError(f"world_size {world_size} outside [1, {L.DP_MAX_WORLD}]")
        self.lr, self.final_lr_ratio, self.max_steps, self.start_step = float(lr), float(final_lr_ratio), int(max_steps), int(start_step)
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        n = int(loader.all_inverse_krs.shape[0])
        if not 1 <= n <= 1024:
            raise RuntimeError(f"{n} cameras: the colour response handles 1 to 1024")
        dev = loader.all_inverse_krs.device
        self.device, self.num_cameras = dev, n
        f64 = dict(dtype=torch.float64, device=dev)
        self.params = torch.zeros((n, 6), **f64)
        self.exp_avg = torch.zeros((n, 6), **f64)
        self.exp_avg_sq = torch.zeros((n, 6), **f64)
        self.steps = torch.zeros(n, dtype=torch.int32, device=dev)
        self.table = torch.zeros((n, 6), dtype=torch.float32, device=dev)
        if fixed_cameras is None:
            fixed_cameras = (int(loader.camera_numbers[0]),)
        fixed = sorted({int(c) for c in fixed_cameras})
        if any(c < 0 or c >= n for c in fixed):
            raise RuntimeError(f"fixed cameras {fixed} outside [0, {n})")
        self.fixed_cameras = tuple(fixed)
        self.fixed = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.fixed[list(fixed)] = 1
        lib = L.lib()
        self.record = torch.zeros(int(lib.hrf_camera_response_record_bytes(n)), dtype=torch.uint8, device=dev)
        self._bind_record()
        self.workspace = torch.empty(int(lib.hrf_train_loss_response_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        p = L.CameraResponses()
        p.params, p.exp_avg, p.exp_avg_sq = (t.data_ptr() for t in (self.params, self.exp_avg, self.exp_avg_sq))
        p.step, p.fixed, p.table, p.num_cameras = self.steps.data_ptr(), self.fixed.data_ptr(), self.table.data_ptr(), n
        self._desc = p
        self.fits = {}          # camera -> ResponseFit of fit_held_out; not part of state_dict
        self.rank = 0
        if self.world_size > 1:
            import torch.distributed as dist

            self.rank = dist.get_rank(process_group)
            self._check_replicas_agree()

    def _bind_record(self) -> None:
        n, words = self.num_cameras, self.record.view(torch.int32)
        self.response_grad = words[:6 * n].view(torch.float32).view(n, 6)   # the last step's, before Adam
        self.ray_count = words[6 * n:7 * n]
        self.error = words[7 * n:]      # sticky: bit 0, a bad camera number; bit 1, one in another rank's batch

    def _adopt_record(self, buffer: torch.Tensor) -> None:
        """Moves the gradient record into `buffer` (uint8, the record's size: peer-visible memory the other ranks read)."""
        with torch.no_grad():
            buffer.copy_(self.record)
        self.record = buffer
        self._bind_record()

    def _replica_config(self) -> dict:
        """What every rank must agree on: the cameras (the loader's camera tables and training cameras), the fixed
        cameras and the settings."""
        digest = lambda t: hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()   # noqa: E731
        return {"num_cameras": self.num_cameras, "cameras": digest(self.loader.all_inverse_krs),
                "training_cameras": tuple(int(c) for c in self.loader.camera_numbers),
                "fixed_cameras": self.fixed_cameras,
                "lr": self.lr, "final_lr_ratio": self.final_lr_ratio, "max_steps": self.max_steps,
                "start_step": self.start_step, "betas": self.betas, "eps": self.eps}

    def _check_replicas_agree(self) -> None:
        """Collective over `process_group`: every rank gathers every rank's configuration and takes the same decision,
        so either all ranks go on or all raise ``ValueError`` naming the first field that differs."""
        import torch.distributed as dist

        mine = self._replica_config()
        configs = [None] * self.world_size
        dist.all_gather_object(configs, mine, group=self.process_group)
        for name in mine:
            values = [cfg[name] for cfg in configs]
            if any(v != values[0] for v in values):
                raise ValueError(f"CameraResponses differ between the ranks in {name}: every rank needs the same cameras "
                                 "and settings")

    # ---------------------------------------------------------------------------------------------- train step
    def active(self, t: int) -> bool:
        """Whether the train step after `t` completed steps uses and refines the responses."""
        return t >= self.start_step

    def current_lr(self, t: int) -> float:
        return self.lr * self.final_lr_ratio ** min(max(t - self.start_step, 0) / max(self.max_steps, 1), 1.0)

    def loss(self, color, weights_sum, rgba, background, cameras, num_rays: int, huber_delta: float, bce_weight: float,
             loss_scale, d_color, d_weights_sum, loss_out) -> int:
        """Enqueues hrf_train_loss_response into the given [R] buffers and this object's gradient record; no host read.
        Returns the launch count."""
        L.check(L.lib().hrf_train_loss_response(
            L.ptr(color), L.ptr(weights_sum), L.ptr(rgba), L.ptr(background), L.ptr(cameras), int(num_rays),
            self.table.data_ptr(), self.num_cameras, float(huber_delta), float(bce_weight), L.ptr(loss_scale),
            L.ptr(d_color), L.ptr(d_weights_sum), L.ptr(loss_out), self.response_grad.data_ptr(),
            self.ray_count.data_ptr(), self.error.data_ptr(), self.workspace.data_ptr(), L.stream()))
        return 2 if num_rays > 0 else 1

    def step(self, t: int, records: Optional[Sequence[int]] = None) -> int:
        """Enqueues hrf_camera_response_step at the learning rate of step `t`; no host read.  `records`: with
        world_size > 1, the device addresses of every rank's gradient record in rank order; the step then reduces them
        (hrf_camera_response_step_ranks).  Returns the launch count."""
        b1, b2 = self.betas
        if records is not None:
            if len(records) != self.world_size:
                raise ValueError(f"{len(records)} gradient records for world_size {self.world_size}")
            rec = L.CameraGradRecords()
            for r, a in enumerate(records):
                rec.record[r] = a
            rec.world, rec.rank = self.world_size, self.rank
            L.check(L.lib().hrf_camera_response_step_ranks(C.byref(self._desc), C.byref(rec), self.error.data_ptr(),
                                                           self.current_lr(t), b1, b2, self.eps, L.stream()))
            return 1
        L.check(L.lib().hrf_camera_response_step(C.byref(self._desc), self.response_grad.data_ptr(),
                                                 self.ray_count.data_ptr(), self.error.data_ptr(), self.current_lr(t),
                                                 b1, b2, self.eps, L.stream()))
        return 1

    def check(self) -> None:
        """Raises ``RuntimeError`` when a batch held a camera number outside the loader's cameras (reads the device)."""
        err = int(self.error.cpu()[0])
        if err & 1:
            raise RuntimeError(f"a train batch held a camera number outside [0, {self.num_cameras}): the colour "
                               "responses stopped updating at that step")
        if err:
            raise RuntimeError(f"another rank's train batch held a camera number outside [0, {self.num_cameras}): the "
                               "colour responses stopped updating at that step on every rank")

    # ---------------------------------------------------------------------------------------------- read out
    def gains(self) -> torch.Tensor:
        """e^gamma per camera and channel, float64 [C,3] (1 at identity)."""
        return torch.exp(self.params[:, :3])

    def offsets(self) -> torch.Tensor:
        """b per camera and channel, float64 [C,3] (in the image's [0,1] units, weighted by the render's opacity)."""
        return self.params[:, 3:].clone()

    def learned(self) -> torch.Tensor:
        """bool [C]: the cameras whose response differs from the identity."""
        return (self.table != 0).any(dim=1)

    def apply(self, color: torch.Tensor, alpha: torch.Tensor, camera: int, background=None) -> torch.Tensor:
        """Applies camera `camera`'s response to a rendered image in place and returns it: `color` float32 [..., 3]
        composited on `background` (3 floats, default black) with opacity `alpha` float32 [...]
        (hrf_camera_response_apply).  A camera at identity leaves the bytes unchanged."""
        L.require_cuda(color, "color", torch.float32)
        L.require_cuda(alpha, "alpha", torch.float32)
        P = alpha.numel()
        if color.numel() != 3 * P or color.shape[-1] != 3:
            raise RuntimeError(f"color must be [..., 3] with one alpha per pixel, got {tuple(color.shape)} and "
                               f"{tuple(alpha.shape)}")
        if not 0 <= int(camera) < self.num_cameras:
            raise RuntimeError(f"camera {camera} outside [0, {self.num_cameras})")
        bg = torch.zeros(3, dtype=torch.float32, device=color.device) if background is None else \
            torch.as_tensor(background, dtype=torch.float32).reshape(3).to(color.device).contiguous()
        with torch.cuda.device(color.device):
            L.check(L.lib().hrf_camera_response_apply(color.data_ptr(), alpha.data_ptr(), P, self.table.data_ptr(),
                                                      int(camera), self.num_cameras, bg.data_ptr(), L.stream()))
        return color

    # ---------------------------------------------------------------------------------------------- held-out fit
    @property
    def fitted_pairs(self) -> dict:
        """camera -> the (camera, frame) pairs its held-out response was fitted on (``fit_held_out``)."""
        return {c: [(c, f) for f in fit.frames] for c, fit in self.fits.items()}

    def accumulate_fit(self, color, alpha, gt_u8, mask, camera: int, moments, error, workspace=None) -> None:
        """Enqueues hrf_response_fit_accumulate: adds one view's sums (pixels where `mask` != 0) to row `camera` of
        `moments` (float64 [C,17]).  `color` float32 [...,3], `alpha` float32 [...], `gt_u8` uint8 [...,3], `mask` uint8
        or bool [...], all contiguous on the responses' device; `error` int32 [1]."""
        if isinstance(mask, torch.Tensor) and mask.dtype == torch.bool:
            mask = mask.view(torch.uint8)
        for t, name, dt in ((color, "color", torch.float32), (alpha, "alpha", torch.float32), (gt_u8, "gt", torch.uint8),
                            (mask, "mask", torch.uint8), (moments, "moments", torch.float64), (error, "error", torch.int32)):
            L.require_cuda(t, name, dt)
        P = alpha.numel()
        if color.numel() != 3 * P or gt_u8.numel() != 3 * P or mask.numel() != P:
            raise RuntimeError(f"color {tuple(color.shape)}, gt {tuple(gt_u8.shape)} and mask {tuple(mask.shape)} do not "
                               f"match {P} pixels")
        if tuple(moments.shape) != (self.num_cameras, FIT_ROW):
            raise RuntimeError(f"moments must be [{self.num_cameras}, {FIT_ROW}], got {tuple(moments.shape)}")
        lib = L.lib()
        if workspace is None:
            workspace = torch.empty(int(lib.hrf_response_fit_workspace_bytes(P)), dtype=torch.uint8, device=color.device)
        with torch.cuda.device(color.device):
            L.check(lib.hrf_response_fit_accumulate(color.data_ptr(), alpha.data_ptr(), gt_u8.data_ptr(),
                                                    mask.data_ptr(), P, int(camera), self.num_cameras,
                                                    moments.data_ptr(), error.data_ptr(), workspace.data_ptr(),
                                                    L.stream()))

    def solve_fit(self, moments, cameras, ridge: float = 1e-6, min_pixels: int = 1024):
        """Enqueues hrf_response_fit_solve for `cameras` and returns (report float64 [K,8], status int32 [K]) on the
        device: report rows (n, SSE at the identity rgb, SSE at the fit rgb, status).  Writes the listed cameras' params
        and table rows only when every one of them succeeds."""
        L.require_cuda(moments, "moments", torch.float64)
        if tuple(moments.shape) != (self.num_cameras, FIT_ROW):
            raise RuntimeError(f"moments must be [{self.num_cameras}, {FIT_ROW}], got {tuple(moments.shape)}")
        cams = torch.as_tensor(list(cameras), dtype=torch.int32).to(self.device)
        K = int(cams.numel())
        report = torch.zeros((K, 8), dtype=torch.float64, device=self.device)
        status = torch.zeros(K, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_response_fit_solve(C.byref(self._desc), moments.data_ptr(), cams.data_ptr(), K,
                                                   float(ridge), float(min_pixels), report.data_ptr(),
                                                   status.data_ptr(), L.stream()))
        return report, status

    @torch.no_grad()
    def fit_held_out(self, model, loader, pairs, *, ridge: float = 1e-6, min_pixels: int = 1024, bake: bool = False,
                     render_step_size: float = 4e-4, rays_per_batch: int = 262144) -> list:
        """Fits the response of every camera of `pairs` (camera, frame) against the frozen `model` (DESIGN.md §3.18).
        Each pair is rendered as ``evaluate_sequence`` renders it (``_Views``, background 0, the frame's hull, or with
        `bake` the hull baked once per frame) and its pixels inside the dataset's mask are added to the camera's moments;
        one solve then gives, per channel, the gain g and offset b minimising sum (g f + a b - y)^2 +
        ridge n ((g - 1)^2 + b^2) (f the render, a its alpha, y = gt / 255), written as gamma = log g and b.

        Raises ``ValueError`` before any work for a fixed camera, a camera with a trained response (step counter > 0), a
        frame that is not one of the model's or a loader whose camera count differs, and after the solve, naming the
        camera and the reason, when a camera cannot be fitted (fewer than `min_pixels` pixels, a singular system, a gain
        <= 0); nothing has been written then.  Fitting a camera again replaces its earlier fit.  Returns a
        ``ResponseFit`` per camera, in camera order; ``fits`` and ``fitted_pairs`` keep them."""
        from .compact_model import require_trainable

        require_trainable(model, "fit_held_out")
        from .depth_maps import _Views
        from .evaluation import ground_truth
        from .learned_occupancy import bake_occupancy_grid

        n_loader = int(loader.all_inverse_krs.shape[0])
        if n_loader != self.num_cameras:
            raise ValueError(f"the loader has {n_loader} cameras, the responses {self.num_cameras}")
        pairs = [(int(c), int(f)) for c, f in pairs]
        if not pairs:
            raise ValueError("no (camera, frame) pairs to fit on")
        steps = self.steps.cpu().numpy()
        for c, f in pairs:
            if not 0 <= c < self.num_cameras:
                raise ValueError(f"camera {c} outside [0, {self.num_cameras})")
            if c in self.fixed_cameras:
                raise ValueError(f"camera {c} is fixed: it holds the gauge and keeps the identity")
            if steps[c] > 0:
                raise ValueError(f"camera {c} has a trained response ({int(steps[c])} steps): a held-out fit would "
                                 "replace it")
            if f not in model.sorted_frame_numbers:
                raise ValueError(f"frame {f} is not one of the model's frames")
        cameras = sorted({c for c, _ in pairs})
        dev = self.device
        moments = torch.zeros((self.num_cameras, FIT_ROW), dtype=torch.float64, device=dev)
        error = torch.zeros(1, dtype=torch.int32, device=dev)
        views = _Views(model, loader, render_step_size, rays_per_batch)
        grids = {}
        for c, frame in pairs:
            if frame not in grids:
                grid = views.hull(frame)
                grids[frame] = bake_occupancy_grid(model, frame, grid, render_step_size) if bake else grid
            view = views.render(c, frame, grids[frame])
            gt, mask = ground_truth(loader, c, frame)
            self.accumulate_fit(view.color.contiguous(), view.alpha.contiguous(), torch.from_numpy(gt).to(dev),
                                torch.from_numpy(mask).to(dev), c, moments, error)
            del view
        report, status = self.solve_fit(moments, cameras, ridge, min_pixels)
        report, status = report.cpu().numpy(), status.cpu().numpy()
        if int(error.cpu()[0]) != 0:
            raise RuntimeError("hrf_response_fit_accumulate saw a camera outside the responses' cameras")
        bad = [(c, int(s)) for c, s in zip(cameras, status) if s != 0]
        if bad:
            raise ValueError("held-out response fit refused, nothing written: " + "; ".join(
                f"camera {c}: {FIT_STATUS.get(s, f'status {s}')} ({int(report[cameras.index(c), 0])} pixels)"
                for c, s in bad))
        params = self.params.cpu().numpy()
        fits = []
        for k, c in enumerate(cameras):
            n = int(report[k, 0])
            fit = ResponseFit(camera=c, frames=tuple(f for cc, f in pairs if cc == c), n=n,
                              gain=tuple(float(x) for x in np.exp(params[c, :3])),
                              offset=tuple(float(x) for x in params[c, 3:]),
                              psnr_before=_masked_psnr(float(report[k, 1:4].sum()), n),
                              psnr_after=_masked_psnr(float(report[k, 4:7].sum()), n))
            self.fits[c] = fit
            fits.append(fit)
        return fits

    def write_fit_csv(self, path, loader=None) -> None:
        """One row per camera with a held-out fit (``fits``), in camera order: name (from `loader`'s cameras, by
        default the responses' loader), fit views, fit pixels, gains, offsets, and the masked PSNR of the float render
        over the fit pixels before and after the fit."""
        from .camera_refinement import _camera_name

        cams = getattr(self.loader if loader is None else loader, "cameras", None)
        with open(path, "w", newline="") as fh:
            w = csv.writer(fh)
            w.writerow(FIT_COLUMNS)
            for c in sorted(self.fits):
                fit = self.fits[c]
                name = _camera_name(cams[c], c) if cams is not None and c < len(cams) else f"Cam{c + 1:03d}"
                w.writerow([name, len(fit.frames), fit.n] + [repr(float(x)) for x in (*fit.gain, *fit.offset)]
                           + [repr(fit.psnr_before), repr(fit.psnr_after)])

    # ---------------------------------------------------------------------------------------------- state
    def _write_table(self) -> None:
        """Rebuilds the table from the parameters on the device, with the step kernels' expression
        (hrf_camera_response_write_table), so a reloaded table is the one the step would have written."""
        with torch.cuda.device(self.device):
            L.check(L.lib().hrf_camera_response_write_table(C.byref(self._desc), L.stream()))

    def state_dict(self) -> dict:
        self.check()
        return {"params": self.params.cpu(), "exp_avg": self.exp_avg.cpu(), "exp_avg_sq": self.exp_avg_sq.cpu(),
                "steps": self.steps.cpu(), "fixed_cameras": list(self.fixed_cameras)}

    def load_state_dict(self, state: dict) -> None:
        """Restores parameters, moments, step counters and fixed cameras in place and rewrites the table."""
        if tuple(state["params"].shape) != (self.num_cameras, 6):
            raise RuntimeError(f"state_dict holds {state['params'].shape[0]} cameras, not {self.num_cameras}")
        with torch.no_grad():
            for name in ("params", "exp_avg", "exp_avg_sq", "steps"):
                getattr(self, name).copy_(state[name])
            fixed = sorted(int(c) for c in state["fixed_cameras"])
            self.fixed.zero_()
            self.fixed[fixed] = 1
            self.fixed_cameras = tuple(fixed)
        self.fits = {}          # the loaded parameters replace any held-out fit
        self._write_table()

    def write_response_csv(self, path) -> None:
        """One row per camera: name, gain_r, gain_g, gain_b, offset_r, offset_g, offset_b."""
        from .camera_refinement import _camera_name

        gains, offsets = self.gains().cpu().numpy(), self.offsets().cpu().numpy()
        cams = getattr(self.loader, "cameras", None)
        with open(path, "w", newline="") as fh:
            w = csv.writer(fh)
            w.writerow(RESPONSE_COLUMNS)
            for c in range(self.num_cameras):
                name = _camera_name(cams[c], c) if cams is not None and c < len(cams) else f"Cam{c + 1:03d}"
                w.writerow([name] + [repr(float(x)) for x in (*gains[c], *offsets[c])])
