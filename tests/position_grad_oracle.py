"""Float64 reference of hrf_field_position_grad: d_positions = sum over levels and grids of J^T . dF, where J is the
derivative of the composed features (4 hash grids x 16 levels, composed with the vector lerps) with respect to the
sample position.

The trilinear weights are computed here in float64 torch, so autograd reaches them (oracle/hashgrid.py computes them in
float32 numpy).  The cells, corner indices and vector taps are decided as field_common.cuh decides them.  Two modes:
* ``exact32=True``: every fractional offset (grid cells and vector taps) has the float32 value the kernel computes
  (pos = fma(scale, u, 0.5), frac = pos - floor(pos)); the derivative of the offset is still scale (resp. vec_res).
  This is the mode to compare the kernel with: what remains is the kernel's fp32 accumulation.
* ``exact32=False``: a pure float64 function of u (frac = scale * u + 0.5 - floor), whose derivative central finite
  differences can check.

``bound_terms`` returns S_d = sum of |every product term| of d_positions[:, d] (the Jacobian terms in absolute value,
contracted with |dF|): a sum of m terms in fp32, in any order, is within m * 2^-23 * S of its exact value.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import numpy as np
import torch

PRIME_Y = np.uint32(2654435761)
PRIME_Z = np.uint32(805459861)
GRID_DIMS = ((0, 1, 2), (0, 1, 3), (1, 2, 3), (0, 2, 3))    # xyz, xyt, yzt, xzt over (x, y, z, t)
PAIRED_AXIS = (3, 2, 0, 1)                                    # F = xyz V_t + xyt V_z + yzt V_x + xzt V_y


@dataclass
class Segment:
    scale: np.ndarray            # float32 [16]
    res: np.ndarray              # uint32 [16]
    offset: np.ndarray           # uint32 [16]
    size: np.ndarray             # uint32 [16]
    hashed: np.ndarray           # bool [16]
    tables: List[torch.Tensor]   # 4 x float64 [entries, 2] (the bf16 values the kernels read)
    vectors: torch.Tensor        # float64 [4, VR, 32]


def segments_of(model) -> List[Segment]:
    """The segments of a HumanRF module, with its tables rounded to bf16 as the shadow copies are."""
    out = []
    for fg in model.feature_grids:
        lay = fg.layout
        hashed = np.array([(lay.hashed_mask >> l) & 1 for l in range(16)], bool)
        tabs = [g.detach().cpu().to(torch.bfloat16).to(torch.float64).view(-1, 2) for g in fg.grids()]
        out.append(Segment(lay.scale.copy(), lay.res.copy(), lay.offset.copy(), lay.size.copy(), hashed, tabs,
                           fg.vectors.detach().cpu().to(torch.float64)))
    return out


def frame_tables(model):
    return (model.frame_numbers_to_segment_numbers.cpu().numpy(),
            model.frame_numbers_to_normalized_local_frame_numbers.cpu().numpy())


def _fma32(a, b, c) -> np.ndarray:
    return (np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
            + np.float64(c)).astype(np.float32)


def _cell(u: torch.Tensor, scale: np.float32, exact32: bool):
    """(uint32 cell [N], frac [N] float64 with d frac / d u = scale)."""
    s64 = float(scale)
    if exact32:
        pos = _fma32(u.detach().numpy().astype(np.float32), scale, 0.5)
        fl = np.floor(pos)
        frac0 = torch.from_numpy((pos - fl).astype(np.float64))
        frac = frac0 + s64 * (u - u.detach())
    else:
        p = s64 * u + 0.5
        fl = np.floor(p.detach().numpy())
        frac = p - torch.from_numpy(fl)
    return fl.astype(np.int64).astype(np.uint32), frac


def _indices(g, hashed: bool, res: int, size: int):
    """[N,8] entry indices, corner bit d <-> +1 along dimension d (corner_indices)."""
    idx = []
    for c in range(8):
        gl = [g[d] + np.uint32((c >> d) & 1) for d in range(3)]
        with np.errstate(over="ignore"):
            if hashed:
                h = gl[0] ^ (gl[1] * PRIME_Y) ^ (gl[2] * PRIME_Z)
            else:
                h = gl[0] + gl[1] * np.uint32(res) + gl[2] * np.uint32(res * res)
        idx.append((h % np.uint32(size)).astype(np.int64))
    return np.stack(idx, 1)


def _tap(coord: torch.Tensor, vr: int, exact32: bool):
    """make_row_tap2: (i0, i1, frac with d frac / d coord = vr)."""
    if exact32:
        c = _fma32(coord.detach().numpy().astype(np.float32), np.float32(vr), -0.5)
        fl = np.floor(c)
        frac = torch.from_numpy((c - fl).astype(np.float64)) + float(vr) * (coord - coord.detach())
    else:
        c = coord * float(vr) - 0.5
        fl = np.floor(c.detach().numpy())
        frac = c - torch.from_numpy(fl)
    i0 = np.clip(np.maximum(fl, 0.0).astype(np.int64), 0, vr - 1)
    i1 = np.clip(np.minimum(fl + 1.0, vr - 1).astype(np.int64), 0, vr - 1)
    return i0, i1, frac


def _level(seg: Segment, l: int, u: torch.Tensor, exact32: bool):
    """Per grid k: (corner values [N,8,2], corner weight factors [N,8,3] as differentiable tensors); per axis a: the tap
    (v0, v1 [N,2], frac [N])."""
    cells = [_cell(u[:, d], seg.scale[l], exact32) for d in range(4)]
    grids = []
    for k, dims in enumerate(GRID_DIMS):
        g = [cells[d][0] for d in dims]
        idx = _indices(g, bool(seg.hashed[l]), int(seg.res[l]), int(seg.size[l])) + int(seg.offset[l])
        vals = seg.tables[k][torch.from_numpy(idx.reshape(-1))].view(-1, 8, 2)
        fr = [cells[d][1] for d in dims]
        fac = torch.stack([torch.stack([fr[d] if (c >> d) & 1 else 1 - fr[d] for d in range(3)], 1) for c in range(8)], 1)
        grids.append((vals, fac))
    vr = seg.vectors.shape[1]
    taps = []
    for a in range(4):
        i0, i1, fr = _tap(u[:, a], vr, exact32)
        v = seg.vectors[a][:, 2 * l:2 * l + 2]
        taps.append((v[torch.from_numpy(i0)], v[torch.from_numpy(i1)], fr))
    return grids, taps


def _features_seg(seg: Segment, u: torch.Tensor, exact32: bool) -> torch.Tensor:
    out = []
    for l in range(16):
        grids, taps = _level(seg, l, u, exact32)
        e = [(vals * fac.prod(2, keepdim=True)).sum(1) for vals, fac in grids]
        V = [v0 + fr.unsqueeze(1) * (v1 - v0) for v0, v1, fr in taps]
        out.append(sum(e[k] * V[PAIRED_AXIS[k]] for k in range(4)))
    return torch.cat(out, 1)


def _normalised(positions: np.ndarray, frames: np.ndarray, f2s, f2t):
    """(u float32 [N,4] as the kernels build it: p + 0.5 in fp32, local time; segment [N], -1 = none)."""
    p = np.asarray(positions, np.float32)
    fr = np.asarray(frames, np.int64)
    ok = (fr >= 0) & (fr < len(f2s))
    seg = np.where(ok, f2s[np.clip(fr, 0, len(f2s) - 1)], -1)
    t = np.where(ok, f2t[np.clip(fr, 0, len(f2t) - 1)], 0).astype(np.float32)
    u = np.concatenate([(p + np.float32(0.5)).astype(np.float32), t[:, None]], 1)
    return u, seg


def features(segs, f2s, f2t, positions, frames, exact32=True) -> torch.Tensor:
    """Composed features [N,32] float64 (no bf16 rounding of the result); 0 for samples without a segment."""
    u32, seg = _normalised(positions, frames, f2s, f2t)
    u = torch.from_numpy(u32.astype(np.float64))
    out = torch.zeros((u.shape[0], 32), dtype=torch.float64)
    for s, sd in enumerate(segs):
        m = np.nonzero(seg == s)[0]
        if len(m):
            out[torch.from_numpy(m)] = _features_seg(sd, u[torch.from_numpy(m)], exact32)
    return out


def position_grad(segs, f2s, f2t, positions, frames, dF, exact32=True, u_override=None) -> torch.Tensor:
    """d_positions [N,3] float64 = J^T dF through autograd, dF [N,32] (level-major pairs).  `u_override`: float64 [N,4]
    normalised coordinates to use instead of p + 0.5 (the finite-difference check moves them)."""
    u32, seg = _normalised(positions, frames, f2s, f2t)
    u = torch.from_numpy(u32.astype(np.float64)) if u_override is None else u_override.detach().clone()
    dF = torch.as_tensor(dF, dtype=torch.float64)
    out = torch.zeros((u.shape[0], 3), dtype=torch.float64)
    for s, sd in enumerate(segs):
        m = torch.from_numpy(np.nonzero(seg == s)[0])
        if len(m) == 0:
            continue
        um = u[m].clone().requires_grad_(True)
        F = _features_seg(sd, um, exact32)
        (g,) = torch.autograd.grad((F * dF[m]).sum(), um)
        out[m] = g[:, :3]
    return out


def bound_terms(segs, f2s, f2t, positions, frames, dF) -> torch.Tensor:
    """S [N,3]: sum over levels, features, grids and corners of |dF| * |each product term| of the kernel's sum."""
    u32, seg = _normalised(positions, frames, f2s, f2t)
    u = torch.from_numpy(u32.astype(np.float64))
    adF = torch.as_tensor(dF, dtype=torch.float64).abs()
    out = torch.zeros((u.shape[0], 3), dtype=torch.float64)
    for s, sd in enumerate(segs):
        m = torch.from_numpy(np.nonzero(seg == s)[0])
        if len(m) == 0:
            continue
        um = u[m]
        vr = float(sd.vectors.shape[1])
        acc = torch.zeros((len(m), 3), dtype=torch.float64)
        for l in range(16):
            with torch.no_grad():
                grids, taps = _level(sd, l, um, True)
            scale = float(sd.scale[l])
            Vabs = [v0.abs() + v1.abs() for v0, v1, _ in taps]
            dVabs = [vr * (v0.abs() + v1.abs()) for v0, v1, _ in taps]
            for k, (vals, fac) in enumerate(grids):
                av = vals.abs()
                eabs = (av * fac.prod(2, keepdim=True).abs()).sum(1)
                for j, d in enumerate(GRID_DIMS[k]):
                    others = [i for i in range(3) if i != j]
                    dw = (fac[:, :, others[0]] * fac[:, :, others[1]]).abs().unsqueeze(2)
                    if d < 3:   # grid term along a spatial axis
                        acc[:, d] += (adF[m, 2 * l:2 * l + 2] * scale * (av * dw).sum(1) * Vabs[PAIRED_AXIS[k]]).sum(1)
                a = PAIRED_AXIS[k]
                if a < 3:       # vector term along the paired axis
                    acc[:, a] += (adF[m, 2 * l:2 * l + 2] * eabs * dVabs[a]).sum(1)
        out[m] = acc
    return out


def face_distance(positions, frames, f2s, f2t, segs) -> np.ndarray:
    """Smallest distance (in u units) from each sample to a cell face of any level or a vector-tap kink, over the three
    spatial axes (the time coordinate is not moved)."""
    u32, seg = _normalised(positions, frames, f2s, f2t)
    u = u32.astype(np.float64)[:, :3]
    dmin = np.full(len(u), np.inf)
    sd = segs[0]
    for l in range(16):
        p = float(sd.scale[l]) * u + 0.5
        dmin = np.minimum(dmin, (np.abs(p - np.round(p)) / float(sd.scale[l])).min(1))
    vr = float(sd.vectors.shape[1])
    c = u * vr - 0.5
    return np.minimum(dmin, (np.abs(c - np.round(c)) / vr).min(1))
