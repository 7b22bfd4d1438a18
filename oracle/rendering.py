"""Oracle: transmittance / visibility / compositing / loss on the CPU.

TEST INFRASTRUCTURE ONLY.  Follows humanrf/volume_rendering.py:42-150 and
humanrf/trainer.py:205-255, humanrf/utils/loss.py:4-10.  The first-party glue (positions,
jitter, alpha, t_ends = t + step, mask application, background blend) is PINNED: the
reference's own prune_samples / render run on the CPU and agree bit for bit
(tests/test_reference_live_cpu.py).  PARITY UNPINNED for the nerfacc==0.3.1 pieces
(requirements.txt:3, not part of the reference checkout): restated from its published semantics
(nerfacc/vol_rendering.py: render_visibility, render_weight_from_density,
accumulate_along_rays).
"""
from __future__ import annotations

import numpy as np
import torch

STEP = 4e-4  # volume_rendering.py:47,92 ; data_loader.py:573


def _exclusive_by_ray(vals: torch.Tensor, ray_indices: torch.Tensor, op: str) -> torch.Tensor:
    """Exclusive cumsum / cumprod restarting at every ray (ray_indices sorted ascending)."""
    n = vals.shape[0]
    if n == 0:
        return vals.clone()
    ri = ray_indices.reshape(-1)
    start = torch.ones(n, dtype=torch.bool)
    start[1:] = ri[1:] != ri[:-1]
    seg_id = torch.cumsum(start.long(), 0) - 1
    first = torch.nonzero(start).reshape(-1)
    if op == "sum":
        inc = torch.cumsum(vals, 0)
        exc = inc - vals
        return exc - exc[first][seg_id]
    # product: do it per ray sequentially in log-free form (exact left-to-right product)
    out = torch.empty_like(vals)
    v = vals.detach().numpy()
    o = np.empty_like(v)
    bounds = list(first.numpy()) + [n]
    for a, b in zip(bounds[:-1], bounds[1:]):
        t = v.dtype.type(1.0)
        for i in range(a, b):
            o[i] = t
            t = t * v[i]
    out.copy_(torch.from_numpy(o))
    return out


def render_visibility(alphas: torch.Tensor, ray_indices: torch.Tensor, early_stop_eps=1e-4, alpha_thre=1e-4):
    """nerfacc 0.3.1: T_i = prod_{j<i}(1-alpha_j) over the ray; keep = (T>=eps) & (alpha>=thre)."""
    a = alphas.reshape(-1)
    T = _exclusive_by_ray(1.0 - a, ray_indices, "prod")
    return (T >= early_stop_eps) & (a >= alpha_thre)


def prune_mask(sigma: torch.Tensor, ray_indices: torch.Tensor, step: float = STEP) -> torch.Tensor:
    """volume_rendering.py:75-81 : alphas = 1 - exp(-density*step)."""
    alphas = 1.0 - torch.exp(-sigma.reshape(-1) * step)
    return render_visibility(alphas, ray_indices)


def weights_from_density(t: torch.Tensor, sigma: torch.Tensor, ray_indices: torch.Tensor, step: float = STEP):
    """volume_rendering.py:123-129 + nerfacc 0.3.1 render_weight_from_density:
    dt = (t+step) - t (fp32, as computed by the caller); T = exp(-excl_sum(sigma*dt)); w = T*(1-exp(-sigma*dt))."""
    t = t.reshape(-1)
    dt = (t + step) - t
    sdt = sigma.reshape(-1) * dt
    T = torch.exp(-_exclusive_by_ray(sdt, ray_indices, "sum"))
    return T * (1.0 - torch.exp(-sdt))


def accumulate(weights: torch.Tensor, ray_indices: torch.Tensor, values, n_rays: int) -> torch.Tensor:
    """nerfacc accumulate_along_rays: scatter-add of w (or w*values) per ray."""
    w = weights.reshape(-1, 1)
    src = w if values is None else w * values
    out = torch.zeros((n_rays, src.shape[1]), dtype=src.dtype)
    return out.index_add(0, ray_indices.reshape(-1).long(), src)


def render(t, sigma, rgb, ray_indices, n_rays, background=None, step: float = STEP):
    """volume_rendering.py:123-150.  Returns color [R,3], weights_sum [R,1]."""
    w = weights_from_density(t, sigma, ray_indices, step)
    color = accumulate(w, ray_indices, rgb, n_rays)
    wsum = accumulate(w, ray_indices, None, n_rays)
    if background is not None:
        color = color + background * (1.0 - wsum)
    return color, wsum


def bce_loss(pred, target):
    """utils/loss.py:4-10."""
    p = torch.clamp(pred, min=0, max=1)
    return -(target * torch.log(p + 1e-10) + (1 - target) * torch.log(1 - p + 1e-10))


def training_loss(color, wsum, rgba, background, bce_weight=1e-3, huber_delta=0.01):
    """trainer.py:205-215,229-238 : Huber(delta=.01, mean) + w * mean(BCE(wsum, mask))."""
    gt_mask = rgba[:, 3:4]
    gt = rgba[:, :3] * gt_mask + background * (1 - gt_mask)
    photo = torch.nn.functional.huber_loss(color, gt, delta=huber_delta, reduction="mean")
    mask = bce_loss(wsum, gt_mask).mean() * bce_weight
    return photo + mask, gt
