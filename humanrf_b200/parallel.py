"""Multi-GPU plumbing for the hot path (new work: the reference is single-process, single-GPU, SURVEY 2.4).

Training shards ray batches data-parallel, one process per GPU (torch.distributed / NCCL over NVLink):
every rank holds a full replica, samples its own rays, and the only exchange step is ONE all-reduce (sum) of
the flat gradient bucket the fused backward kernel wrote (humanrf_b200.training.FusedTrainer).  Ranks may
keep different numbers of rays after masking, so each rank weights its loss by
``world * R_local / R_total`` -- the sum over ranks then equals the gradient of the mean loss over the UNION
batch (HuberLoss(reduction="mean"), trainer.py:89).

Inference shards image tiles (contiguous pixel ranges, exactly the ranges DataLoader.__next__ walks,
data_loader.py:578-580) or whole (camera, frame) pairs round-robin; no collective on the data path.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [start, end) share of n items; shares differ by at most one item."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard_bounds(n: int, rank: int, world: int, align: int = 4096) -> Tuple[int, int]:
    """[begin, end) of rank's slice of an n-element tensor under data-parallel sharding of the optimiser
    (FusedTrainer exchange="p2p"): equal slices rounded up to `align` elements (the Adam kernel's block), the last
    ranks' slices may be short or empty.  Every element belongs to exactly one rank."""
    per = -(-n // world)
    per = -(-per // align) * align
    begin = min(rank * per, n)
    return begin, min(begin + per, n)


def deal_round_robin(items: Sequence, rank: int, world: int) -> List:
    """(camera, frame) pairs of a render sequence dealt round-robin to ranks (SURVEY 8e)."""
    return [x for i, x in enumerate(items) if i % world == rank]


def grid_major_bucket_layout(sizes: Sequence[int], num_segments: int):
    """Layout of the flat gradient bucket for parameters given in hot_parameters() order (per segment: grid 0..3,
    vectors; then the MLPs and, if any, the camera embeddings).  Returns (slices, regions, order):
    slices[i] = (start, end) of parameter i inside the bucket; regions = 5 contiguous (start, end) spans -- grid k of
    every segment for k = 0..3, then everything else; order = parameter indices in bucket order.  Region k is complete
    once the scatter launch of grid k has run, which is what lets its all-reduce overlap the next launch."""
    S = num_segments
    order = [5 * s + k for k in range(4) for s in range(S)] + [5 * s + 4 for s in range(S)] + list(range(5 * S, len(sizes)))
    slices: List = [None] * len(sizes)
    starts, pos = [], 0
    for j, i in enumerate(order):
        if j % S == 0 and j <= 4 * S:
            starts.append(pos)
        slices[i] = (pos, pos + int(sizes[i]))
        pos = slices[i][1]
    regions = list(zip(starts, starts[1:] + [pos]))
    return slices, regions, order


def active_segments(frame_to_segment: torch.Tensor, frame_numbers: torch.Tensor, num_segments: int) -> torch.Tensor:
    """bool [num_segments], on frame_numbers' device: the temporal segments the batch's frames fall into
    (humanrf.py:162-163).  Only these take part in a training step: the reference never calls the other segments'
    encodings, their .grad stays None (trainer.py:174 zero_grad(set_to_none=True)) and torch.optim.Adam leaves their
    parameters, moments and per-parameter step counters untouched."""
    lut = frame_to_segment.to(frame_numbers.device)
    f = frame_numbers.reshape(-1).long()
    ok = (f >= 0) & (f < lut.numel())
    seg = torch.where(ok, lut[f.clamp(0, lut.numel() - 1)].long(), torch.full_like(f, -1))
    used = torch.zeros(num_segments + 1, dtype=torch.bool, device=f.device)
    used[(seg + 1).clamp(0, num_segments)] = True          # slot 0 collects frames without a segment
    return used[1:]


def mask_inactive_segment_grads(grads: List, active: Sequence[bool]) -> List:
    """grads in hot_parameters() order (per segment: 4 grids + vectors, then the rest): None for the five tensors of
    every segment that is not active, as autograd gives the reference for segments it did not call."""
    out = list(grads)
    for s, a in enumerate(active):
        if not a:
            out[5 * s:5 * s + 5] = [None] * 5
    return out


def _merge_spans(spans):
    out = []
    for a, b in sorted(spans):
        if out and out[-1][1] == a:
            out[-1] = (out[-1][0], b)
        elif b > a:
            out.append((a, b))
    return out


def allreduce_spans(slices, regions, num_segments: int, active=None):
    """What has to cross NVLink in one step: for each of the 5 bucket regions (grid 0..3 of every segment, then the tail)
    the contiguous spans holding gradients of ACTIVE segments (SURVEY 8e: a batch touches <= 8 frames, i.e. typically one
    or two segments); the MLP / embedding block at the end of the tail always takes part.  With active=None every
    region is one span (single-segment models, or a batch touching every segment)."""
    S = num_segments
    on = [True] * S if active is None else list(active)
    out = [_merge_spans([slices[5 * s + k] for s in range(S) if on[s]]) for k in range(4)]
    out.append(_merge_spans([slices[5 * s + 4] for s in range(S) if on[s]] + [(slices[5 * S][0], regions[4][1])]))
    return out


def union_batch_loss_scale(num_rays_local: int, device, group=None):
    """world * R_local / R_total, so that summing rank gradients and dividing by world gives the gradient of the
    mean loss over the union of all ranks' rays.  One 8-byte all-reduce; the result stays ON THE DEVICE (a 0-dim
    tensor to multiply the loss with), so the step keeps running without a host sync."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 1.0
    t = torch.full((1,), float(num_rays_local), dtype=torch.float32, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return (dist.get_world_size(group) * float(num_rays_local)) / t.clamp(min=1.0)[0]


def allreduce_bucket_(flat: torch.Tensor, group=None, async_op: bool = False):
    """In-place sum of (a region of) the flat gradient bucket over the ranks (mean is folded into Adam's grad_scale).
    With async_op the NCCL work handle is returned (None when there is nothing to reduce): the collective runs on
    NCCL's stream behind everything already queued on the current stream, and .wait() orders later kernels after it."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        work = dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        return work if async_op else flat
    return None if async_op else flat


def broadcast_parameters_(params, src: int = 0, group=None, model=None) -> None:
    """Make every replica start from rank `src`'s parameters.  The parameter itself is broadcast into (under no_grad),
    not `p.data`: an in-place write through `.data` does not bump `p._version`, and the native view decides from the
    versions whether the bf16 shadow tables / the packed MLP blob have to be refreshed.  Pass `model` to also drop its
    native view explicitly (for callers that wrote through raw pointers)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        with torch.no_grad():
            for p in params:
                dist.broadcast(p, src=src, group=group)
    if model is not None and hasattr(model, "invalidate_native"):
        model.invalidate_native()


class TileShardedRenderer:
    """Full-image rendering with the image's pixels split into contiguous ranges over the ranks
    (Trainer.test / validate, trainer.py:258-526, without the per-batch D2H and the CPU scatter: the image is
    assembled on the device, SURVEY 8f-3).

    Per batch of `rays_per_batch` pixels: sampler -> density pass with the exact early stop (keeps the composed features of
    every candidate it evaluates) -> visibility compaction -> ONE fused kernel for the survivors (MLPs on the kept
    features + compositing, hrf_render_fused) -> colours placed by the ray mask.  The only host read is the sampler's
    pair of counters that sizes the candidate arrays: the survivor count stays on the device, the placement is a
    cumulative-sum gather (no nonzero())."""

    def __init__(self, model, occupancy_grid, rays_per_batch: int = 262144, step: float = 4e-4):
        self.model, self.og, self.rays_per_batch, self.step = model, occupancy_grid, rays_per_batch, step
        self.last_stats = {}

    @torch.no_grad()
    def render_range(self, cam: dict, start: int, end: int, background: float = 0.0) -> torch.Tensor:
        """cam: dict of the per-image sampler tables for ONE image (frame_numbers, camera_numbers, grid handle,
        landscape, inverse_krs, camera_origins, aabb, G, width, height).  Returns float32 [end-start, 3]."""
        return self._render(cam, start, end, background, False)

    @torch.no_grad()
    def render_range_maps(self, cam: dict, start: int, end: int, background: float = 0.0, normals: bool = False):
        """``render_range`` plus opacity and distance maps (hrf_render_fused_depth): returns (color [P,3], alpha [P],
        distance [P]), P = end - start.  alpha is the weights sum; distance = sum w * t_mid / alpha, the expected
        distance along the ray in the loader's normalised scene units, where alpha > 0, and 0 elsewhere.  Pixels outside
        the ray mask get alpha = distance = 0.  The colours are bit-identical to ``render_range``'s.

        With `normals`, a fourth output [P,3]: unit normals in normalised scene coordinates, N / |N| with
        N = sum_i w_i n_i over the same samples and weights, n_i = -grad sigma_i / |grad sigma_i| (0 where the gradient
        vanishes; hrf_field_position_grad).  0 where |N| = 0 and outside the ray mask.  Colour, alpha and distance are
        bit-identical to the call without normals."""
        return self._render(cam, start, end, background, True, normals)

    def _render(self, cam: dict, start: int, end: int, background: float, maps: bool, normals: bool = False):
        import ctypes as C

        from . import _lib as L
        from .dataset import ray_sampler_native as rs
        from .volume_rendering import ray_offsets, render_fused

        dev = cam["aabb"].device
        lib, nat, step = L.lib(), self.model.native(), self.step
        parts, alphas, dists, norms, nwsums = [], [], [], [], []
        empty_rgba = torch.zeros((0, 4), dtype=torch.uint8, device=dev)
        empty_mask = torch.zeros(0, dtype=torch.bool, device=dev)
        candidates = 0
        for s in range(start, end, self.rays_per_batch):
            e = min(s + self.rays_per_batch, end)
            idx = torch.arange(s, e, dtype=torch.int64, device=dev)
            (o, d, _, fn, cn, mm, mask, dist_, rel) = rs.get_samples_occupancy_minmax(
                empty_rgba, empty_mask, cam["frame_numbers"], cam["camera_numbers"], cam["grid_handles"],
                cam["landscape"], idx, cam["inverse_krs"], cam["camera_origins"], cam["aabb"], cam["G"], cam["width"],
                cam["height"], step, False)
            nr, n = o.shape[0], dist_.shape[0]
            candidates += n
            if nr == 0:
                parts.append(torch.full((e - s, 3), float(background), dtype=torch.float32, device=dev))
                if maps:
                    alphas.append(torch.zeros(e - s, dtype=torch.float32, device=dev))
                    dists.append(torch.zeros(e - s, dtype=torch.float32, device=dev))
                if normals:
                    norms.append(torch.zeros((e - s, 3), dtype=torch.float32, device=dev))
                    nwsums.append(torch.zeros(e - s, dtype=torch.float32, device=dev))
                continue
            ri = rel.long()
            off0 = ray_offsets(ri, nr)
            samples = nat.samples_rays(o, d, fn, dist_, ri)
            sigma, saved = nat.density_early_stop(samples, off0, nr, step, save="feat")
            keep = torch.empty(n, dtype=torch.uint8, device=dev)
            kept_off = torch.empty(nr + 1, dtype=torch.int32, device=dev)
            t2 = torch.empty(n, dtype=torch.float32, device=dev)
            ri2 = torch.empty(n, dtype=torch.int64, device=dev)
            src = torch.empty(n, dtype=torch.int32, device=dev)
            count = torch.zeros(1, dtype=torch.int64, device=dev)
            L.check(lib.hrf_prune(sigma.data_ptr(), dist_.data_ptr(), ri.data_ptr(), off0.data_ptr(), nr, step, 1e-4, 1e-4,
                                  keep.data_ptr(), kept_off.data_ptr(), t2.data_ptr(), ri2.data_ptr(), src.data_ptr(),
                                  count.data_ptr(), L.stream()))
            out = render_fused(self.model, o, d, fn, t2, ri2, nr, float(background), step, reuse=(saved, src, kept_off),
                               count_dev=count, want_depth=maps)
            color = out[0]
            # combine_rays_to_image (volume_rendering.py:26-39) on the device, without nonzero(): ray j of the compacted
            # batch is the (j+1)-th set bit of the mask
            pos = (torch.cumsum(mask.view(-1).long(), 0) - 1).clamp_(min=0)
            parts.append(torch.where(mask.view(-1, 1), color[pos], torch.full((1, 3), float(background), device=dev)))
            if maps:
                alpha, wm = out[1].view(-1), out[2].view(-1)
                dist = torch.where(alpha > 0, wm / alpha, torch.zeros_like(alpha))
                m = mask.view(-1)
                alphas.append(torch.where(m, alpha[pos], torch.zeros((), device=dev)))
                dists.append(torch.where(m, dist[pos], torch.zeros((), device=dev)))
            if normals:
                nrm, nws = self._normals(nat, o, d, fn, t2, ri2, count, saved, src, kept_off, nr)
                norms.append(torch.where(mask.view(-1, 1), nrm[pos], torch.zeros((), device=dev)))
                nwsums.append(torch.where(mask.view(-1), nws[pos], torch.zeros((), device=dev)))
        self.last_stats = {"candidate_samples": candidates}
        cat = lambda xs: xs[0] if len(xs) == 1 else torch.cat(xs, 0)
        if normals:
            # the weights sum of the normals' compositing pass, per pixel: a check that it composited what the render did
            self.last_stats["normal_weights_sum"] = cat(nwsums)
            return cat(parts), cat(alphas), cat(dists), cat(norms)
        return (cat(parts), cat(alphas), cat(dists)) if maps else cat(parts)

    def _normals(self, nat, o, d, fn, t2, ri2, count, saved, src, kept_off, nr):
        """Unit normal per compacted ray of one batch, from the survivors of its prune pass.  The survivor buffers are
        capacity-sized and only the first `count` (a device scalar) rows are live: every step below honours the live
        count or reads through `kept_off`, nothing indexes them on the host side.  Returns (normals [R,3], weights sum [R])."""
        import ctypes as C

        from . import _lib as L

        lib, dev, n = L.lib(), t2.device, t2.shape[0]
        samples = nat.samples_rays(o, d, fn, t2, ri2, count_dev=count)
        sigma, _ = nat.forward_from_features(samples, saved, src)
        ws = torch.empty(n * 40, dtype=torch.float32, device=dev)     # 160 B / sample, hrf_field_backward_mlp's layout
        ones = torch.ones(n, dtype=torch.float32, device=dev)
        L.check(lib.hrf_field_backward_mlp(C.byref(nat.field), C.byref(samples), ones.data_ptr(), None, None, saved.data_ptr(),
                                           src.data_ptr(), None, None, ws.data_ptr(), L.stream()))
        grad = torch.zeros((n, 3), dtype=torch.float32, device=dev)
        L.check(lib.hrf_field_position_grad(C.byref(nat.field), C.byref(samples), ws.data_ptr(), grad.data_ptr(), L.stream()))
        gn = torch.linalg.vector_norm(grad, dim=1, keepdim=True)
        n_i = torch.where(gn > 0, -grad / torch.where(gn > 0, gn, torch.ones_like(gn)), torch.zeros_like(grad))
        acc = torch.empty((nr, 3), dtype=torch.float32, device=dev)
        wsum = torch.empty(nr, dtype=torch.float32, device=dev)
        # sum_i w_i n_i with the render's weights: the compositing kernel with the normals in place of the colours and no
        # background term
        L.check(lib.hrf_composite_forward(sigma.data_ptr(), n_i.data_ptr(), t2.data_ptr(), kept_off.data_ptr(), nr, self.step,
                                          None, acc.data_ptr(), wsum.data_ptr(), None, L.stream()))
        an = torch.linalg.vector_norm(acc, dim=1, keepdim=True)
        return torch.where(an > 0, acc / torch.where(an > 0, an, torch.ones_like(an)), torch.zeros_like(acc)), wsum

    def render_image_sharded(self, cam: dict, rank: int, world: int, background: float = 0.0):
        """This rank's tile of the image: returns (start, end, colours)."""
        start, end = shard_range(cam["width"] * cam["height"], rank, world)
        return start, end, self.render_range(cam, start, end, background)
