"""Volume renderer on the fused sm_90a kernels.

Drop-in for humanrf/volume_rendering.py:14-150: ``RenderOutput``, ``prune_samples`` (in-place,
returns None) and ``render`` with the reference signatures.  Differences by design:

* positions / directions / frame numbers are never materialised per sample: the field kernel
  reads ``sample_distances`` + ``ray_indices`` and the per-ray arrays directly (the reference
  builds three [N,3] gathers per call, volume_rendering.py:66-72,110-119);
* nerfacc's scan-by-key / scatter-add are replaced by one warp-per-ray kernel
  (csrc/composite.cu); pruning compacts on the device and reads back one counter;
* without gradients ``render`` is ONE field kernel with the compositing as its epilogue (hrf_render_fused): per-sample
  sigma / rgb never reach HBM;
* ``prune_samples`` keeps the composed features of the candidates it encoded (64 B/sample) on the batch object; a
  following ``render`` of the same (unchanged) batch runs the two MLPs on them instead of encoding the survivors again.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List

import torch

from . import _lib as L
from .dataset.input_batch import InputBatch
from .scene_representation.humanrf import HumanRF


@dataclass
class RenderOutput:
    # (#rays x 3): [torch.float]
    color: torch.Tensor = None
    # (#rays x 1): [torch.float]
    weights_sum: torch.Tensor = None

    @classmethod
    @torch.no_grad()
    def merge_render_outputs(cls, render_outputs: List["RenderOutput"]) -> "RenderOutput":
        out = RenderOutput()
        for key, val in vars(render_outputs[0]).items():
            if isinstance(val, torch.Tensor):
                setattr(out, key, torch.cat([getattr(r, key) for r in render_outputs], dim=0))
            else:   # as the reference (volume_rendering.py:30-37): every field has to be a tensor, None included
                raise RuntimeError("Unknown data type in the input_batches!")
        return out


def _ray_arrays(ib: InputBatch):
    o = L.require_cuda(ib.ray_origins.detach().float().contiguous(), "ray_origins")
    d = L.require_cuda(ib.ray_directions.detach().float().contiguous(), "ray_directions")
    fr = L.require_cuda(ib.frame_numbers.detach().reshape(-1).to(torch.int32).contiguous(), "frame_numbers")
    t = L.require_cuda(ib.sample_distances.detach().reshape(-1).float().contiguous(), "sample_distances")
    ri = L.require_cuda(ib.ray_indices.detach().reshape(-1).to(torch.int64).contiguous(), "ray_indices")
    return o, d, fr, t, ri


def ray_offsets(ray_indices: torch.Tensor, num_rays: int) -> torch.Tensor:
    off = torch.empty(num_rays + 1, dtype=torch.int32, device=ray_indices.device)
    L.check(L.lib().hrf_ray_offsets(ray_indices.data_ptr(), ray_indices.shape[0], num_rays, off.data_ptr(), L.stream()))
    return off


@torch.no_grad()
def prune_samples(input_batch: InputBatch, scene_representation: HumanRF, is_training: bool,
                  render_step_size: float = 4e-4) -> None:
    """volume_rendering.py:42-84.  Density-only pass + visibility mask (T>=1e-4 & alpha>=1e-4), in place."""
    ib = input_batch
    if is_training:
        ib.sample_distances += torch.rand_like(ib.sample_distances) * render_step_size  # :63-64
    nat = scene_representation.native()
    o, d, fr, t, ri = _ray_arrays(ib)
    n, num_rays = t.shape[0], ib.num_rays
    dev = t.device
    off = ray_offsets(ri, num_rays)
    # density-only pass; chunks of a ray behind an already opaque prefix are provably pruned and are not evaluated
    sigma, saved = nat.density_early_stop(nat.samples_rays(o, d, fr, t, ri), off, num_rays, render_step_size, save="feat")
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    kept_off = torch.empty(num_rays + 1, dtype=torch.int32, device=dev)
    out_t = torch.empty(n, dtype=torch.float32, device=dev)
    out_ri = torch.empty(n, dtype=torch.int64, device=dev)
    src = torch.empty(n, dtype=torch.int32, device=dev)
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    L.check(L.lib().hrf_prune(sigma.data_ptr(), t.data_ptr(), ri.data_ptr(), off.data_ptr(), num_rays,
                              float(render_step_size), 1e-4, 1e-4, keep.data_ptr(), kept_off.data_ptr(),
                              out_t.data_ptr(), out_ri.data_ptr(), src.data_ptr(), counter.data_ptr(), L.stream()))
    kept = int(counter.item())      # the reference's API hands out exactly-sized tensors (merge_input_batches concatenates them)
    ib.sample_distances = out_t[:kept].view(-1, 1)
    ib.ray_indices = out_ri[:kept]
    # what a render() of this very batch can reuse: composed features of the candidates, the survivors' rows in them, the
    # survivors' ray-offset table.  Kept beside the batch (the reference's merge_input_batches walks vars(batch) and
    # rejects anything that is not a tensor, input.py:17-22) and tied to the identity of the two tensors above: any edit
    # of the batch drops it.
    _remember(ib, (saved, src[:kept], kept_off, ib.sample_distances, ib.ray_indices, id(scene_representation)))


_REUSE = {}      # id(batch) -> (weakref to the batch, payload); entries die with their batch


def _remember(ib: InputBatch, payload) -> None:
    import weakref

    key = id(ib)
    _REUSE[key] = (weakref.ref(ib, lambda _r, k=key: _REUSE.pop(k, None)), payload)


def _reusable_features(ib: InputBatch, model: HumanRF):
    e = _REUSE.get(id(ib))
    if e is None or e[0]() is not ib:
        return None
    r = e[1]
    if r[3] is not ib.sample_distances or r[4] is not ib.ray_indices or r[5] != id(model):
        return None
    return r[0], r[1], r[2]


class _RenderFunction(torch.autograd.Function):
    """field forward (ray-batch form) + compositing; backward = composite bwd + fused field bwd."""

    @staticmethod
    def forward(ctx, model: HumanRF, o, d, fr, t, ri, num_rays, background, step, cams, needs_grad, active, reuse, *params):
        nat = model.native()
        dev = t.device
        samples = nat.samples_rays(o, d, fr, t, ri, cams)
        src = None
        if reuse is not None:       # composed features of the prune pass: MLPs only, and the scatter re-gathers the tables
            feat, src, off = reuse
            sigma, rgb = nat.forward_from_features(samples, feat, src)
        else:
            sigma, _, rgb, feat = nat.forward(samples, 1, want_geo=False, want_feat=needs_grad)
            off = ray_offsets(ri, num_rays)
        color = torch.empty((num_rays, 3), dtype=torch.float32, device=dev)
        wsum = torch.empty((num_rays, 1), dtype=torch.float32, device=dev)
        bg = _background_rows(background, num_rays, dev)
        L.check(L.lib().hrf_composite_forward(sigma.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(), num_rays,
                                              float(step), L.ptr(bg), color.data_ptr(), wsum.data_ptr(), None,
                                              L.stream()))
        ctx.model, ctx.num_rays, ctx.step, ctx.active = model, num_rays, float(step), active
        ctx.bg = bg
        ctx.save_for_backward(o, d, fr, t, ri, sigma, rgb, off, feat if feat is not None else t,
                              cams if cams is not None else fr, src if src is not None else fr)
        ctx.has_cams, ctx.has_src = cams is not None, src is not None
        return color, wsum

    @staticmethod
    def backward(ctx, d_color, d_wsum):
        model = ctx.model
        o, d, fr, t, ri, sigma, rgb, off, feat, cams, src = ctx.saved_tensors
        nat = model.native()
        dev = t.device
        n = t.shape[0]
        dc = d_color.detach().float().contiguous() if d_color is not None else torch.zeros((ctx.num_rays, 3), device=dev)
        dw = d_wsum.detach().float().reshape(-1).contiguous() if d_wsum is not None else None
        d_sigma = torch.empty(n, dtype=torch.float32, device=dev)
        d_rgb = torch.empty((n, 3), dtype=torch.float32, device=dev)
        L.check(L.lib().hrf_composite_backward(sigma.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(),
                                               ctx.num_rays, ctx.step, L.ptr(ctx.bg), dc.data_ptr(), L.ptr(dw),
                                               d_sigma.data_ptr(), d_rgb.data_ptr(), L.stream()))
        params = model.hot_parameters()
        grads = [torch.zeros_like(p) for p in params]
        nat.backward(nat.samples_rays(o, d, fr, t, ri, cams if ctx.has_cams else None), d_sigma, d_rgb, feat, grads,
                     feat_index=src if ctx.has_src else None)
        if ctx.active is not None:      # segments the batch did not touch get no gradient at all (None), as in the reference
            from .parallel import mask_inactive_segment_grads

            grads = mask_inactive_segment_grads(grads, ctx.active)
        return (None,) * 13 + tuple(grads)


def render(input_batch: InputBatch, scene_representation: HumanRF, background_rgb: torch.Tensor, is_training: bool,
           render_step_size: float = 4e-4) -> RenderOutput:
    """volume_rendering.py:87-150.  color = sum w*rgb + background*(1 - sum w); weights_sum = sum w."""
    ib = input_batch
    o, d, fr, t, ri = _ray_arrays(ib)
    cams = None
    if scene_representation.camera_embedding_dim > 0 and is_training:   # humanrf.py:194-204 (zeros at evaluation)
        cams = L.require_cuda(ib.camera_numbers.detach().reshape(-1).to(torch.int32).contiguous(), "camera_numbers")
    params = scene_representation.hot_parameters()
    # (ctx.needs_input_grad ignores torch.no_grad(): decide here whether the backward buffers are worth saving)
    needs_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    reuse = _reusable_features(ib, scene_representation)
    if not needs_grad:
        color, wsum = render_fused(scene_representation, o, d, fr, t, ri, ib.num_rays, background_rgb, render_step_size, cams,
                                   reuse=reuse)
        return RenderOutput(color=color, weights_sum=wsum)
    # humanrf.py:162-179: only the segments of this batch's frames are run (and receive gradients)
    active = scene_representation.active_segment_list(fr, ib.unique_frame_numbers)
    color, wsum = _RenderFunction.apply(scene_representation, o, d, fr, t, ri, ib.num_rays, background_rgb,
                                        render_step_size, cams, needs_grad, active, reuse, *params)
    return RenderOutput(color=color, weights_sum=wsum)


def _background_rows(background, num_rays: int, dev) -> "torch.Tensor | None":
    if background is None:
        return None
    bg = torch.as_tensor(background, dtype=torch.float32, device=dev)
    return bg.expand(num_rays, 3).contiguous() if bg.dim() < 2 or bg.shape[0] != num_rays else bg.contiguous()


@torch.no_grad()
def render_fused(model: HumanRF, o, d, fr, t, ri, num_rays: int, background, step: float = 4e-4, cams=None, reuse=None,
                 count_dev=None, ray_offsets_dev=None):
    """Inference render of a ray batch in one field kernel (hrf_render_fused): encode -> MLPs -> compositing, nothing per
    sample written to HBM.  reuse = (features [M,32] bf16, row index per sample, ray-offset table) from a pruning pass:
    no encode at all.  count_dev: live sample count on the device (t / ri are then capacity-sized).
    Returns (color [R,3], weights_sum [R,1])."""
    nat = model.native()
    dev = t.device
    lib = L.lib()
    samples = nat.samples_rays(o, d, fr, t, ri, cams, count_dev=count_dev)
    feat = src = None
    if reuse is not None:
        feat, src, off = reuse
    else:
        off = ray_offsets_dev if ray_offsets_dev is not None else ray_offsets(ri, num_rays)
    color = torch.empty((num_rays, 3), dtype=torch.float32, device=dev)
    wsum = torch.empty((num_rays, 1), dtype=torch.float32, device=dev)
    bg = _background_rows(background, num_rays, dev)
    ws = torch.empty(int(lib.hrf_render_fused_workspace_bytes(t.shape[0])), dtype=torch.uint8, device=dev)
    L.check(lib.hrf_render_fused(C.byref(nat.field), C.byref(samples), off.data_ptr(), num_rays, float(step), L.ptr(bg),
                                 L.ptr(feat), L.ptr(src), color.data_ptr(), wsum.data_ptr(), ws.data_ptr(), L.stream()))
    return color, wsum
