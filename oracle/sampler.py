"""Oracle: ray generation, AABB slab test, occupancy march and sample generation on the CPU.

TEST INFRASTRUCTURE ONLY.  Follows actorshq/dataset/native/ray_sampler.cu:11-194,196-325 and
the texture set-up of actorshq/dataset/native/occupancy_grid.cu:28-38 (clamp addressing,
linear filter, normalised coordinates, normalised-float read mode).

Canonical arithmetic (what "bit-exact" means for this path): every float op is an IEEE
round-to-nearest float32 op; a*b+c patterns that nvcc contracts are single-rounded FMAs
(``fma32``); 1/x and sqrt are correctly rounded.  The reference's own build uses
--use_fast_math (approximate rcp/rsqrt), which cannot be emulated bit-for-bit on a CPU; the
mismatch rate against a real build of the reference is measured on the GPU box
(tests/test_ref_parity_gpu.py).

Hardware trilinear filtering is emulated with the documented 1.8 fixed-point weights
(CUDA Programming Guide, "Linear Filtering"): xB = x*G - 0.5, q = floor(xB*256 + 0.5),
i = q >> 8, alpha = (q & 255)/256, plus the 8-bit result precision measured on real hardware
texture unit (see tex_occupied).  Pinned against a real tex3D on the GPU box
(tests/test_texture_probe_gpu.py), exact except at .5 rounding ties.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def fma32(a, b, c):
    """Correctly rounded float32 fma(a,b,c) (round-to-odd in float64, then one rounding)."""
    a = np.asarray(a, f32).astype(np.float64)
    b = np.asarray(b, f32).astype(np.float64)
    c = np.asarray(c, f32).astype(np.float64)
    p = a * b                                    # exact: 24+24 bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)              # TwoSum residual (exact)
    s = np.array(s, np.float64, copy=True, ndmin=1)
    err = np.broadcast_to(err, s.shape)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even & np.isfinite(s)
    s[fix] = np.nextafter(s[fix], np.where(err[fix] > 0, np.inf, -np.inf))
    return s.astype(f32).reshape(np.broadcast(a, b, c).shape)


def _gmin(a, b):  # glm::min(a,b) = (b < a) ? b : a
    return np.where(b < a, b, a)


def _gmax(a, b):  # glm::max(a,b) = (a < b) ? b : a
    return np.where(a < b, b, a)


def tex_occupied(grid: np.ndarray, p: np.ndarray) -> np.ndarray:
    """grid: uint8 [G,G,G] indexed [z][y][x]; p: [N,3] float32 normalised coords (x,y,z).
    Emulates tex3D<float>(...) > 0 for the reference's texture descriptor.

    Model fitted to a real texture unit (scripts/probe_texture.py; tests/test_texture_probe_gpu.py re-checks it): per-axis alpha in 1.8 fixed point,
    rounded half-up; the filter result itself has 8 fractional bits; each corner weight is
    W = (((wx*wz + 128) >> 8) * wy + 128) >> 8 with w = 256-alpha / alpha, and the result is > 0 iff an
    occupied corner has W >= 1.  Residual disagreement with the hardware is confined to exact .5 ties of
    those roundings (measured < 2e-4 on adversarial points, tests/test_texture_probe_gpu.py)."""
    G = grid.shape[0]
    q = np.floor(((p.astype(f32) * f32(G)).astype(f32) - f32(0.5)).astype(f32) * f32(256.0) + f32(0.5))
    q = q.astype(np.int64)
    i0 = q >> 8
    a = q & 255
    occ = np.zeros(p.shape[0], bool)
    gb = grid > 0
    for dz in (0, 1):
        wz = a[:, 2] if dz else 256 - a[:, 2]
        iz = np.clip(i0[:, 2] + dz, 0, G - 1)
        for dy in (0, 1):
            wy = a[:, 1] if dy else 256 - a[:, 1]
            iy = np.clip(i0[:, 1] + dy, 0, G - 1)
            for dx in (0, 1):
                wx = a[:, 0] if dx else 256 - a[:, 0]
                ix = np.clip(i0[:, 0] + dx, 0, G - 1)
                w = ((((wx * wz + 128) >> 8) * wy) + 128) >> 8
                occ |= (w > 0) & gb[iz, iy, ix]
    return occ


def ray_directions(inverse_krs, camera_origins, landscape, ray_idx, width, height):
    """ray_sampler.cu:96-119.  inverse_krs [B,3,3] f32 stored transposed (column-major for GLM)."""
    idx = np.asarray(ray_idx, np.int64)
    img = idx // (width * height)
    ls = np.asarray(landscape, bool)[img]
    w = np.where(ls, width, height)
    h = np.where(ls, height, width)
    px = (idx % w).astype(f32) + f32(0.5)
    py = ((idx // w) % h).astype(f32) + f32(0.5)
    T = np.asarray(inverse_krs, f32)[img]                # T[i][k] = GLM column i, component k
    v = []
    for k in range(3):
        r = (T[:, 0, k] * px).astype(f32)
        r = fma32(T[:, 1, k], py, r)
        r = fma32(T[:, 2, k], np.ones_like(px), r)
        v.append(r)
    dot = fma32(v[2], v[2], fma32(v[1], v[1], (v[0] * v[0]).astype(f32)))
    inv = (f32(1.0) / np.sqrt(dot, dtype=f32)).astype(f32)
    d = np.stack([(c * inv).astype(f32) for c in v], 1)
    o = np.asarray(camera_origins, f32)[img]
    return o, d, img


def aabb_minmax(o, d, aabb):
    """ray_sampler.cu:11-26."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (f32(1.0) / d).astype(f32)
        t0 = ((aabb[0][None, :] - o).astype(f32) * inv).astype(f32)
        t1 = ((aabb[1][None, :] - o).astype(f32) * inv).astype(f32)
    mn, mx = _gmin(t0, t1), _gmax(t0, t1)
    tmin = _gmax(mn[:, 0], _gmax(mn[:, 1], mn[:, 2]))
    tmax = _gmin(mx[:, 0], _gmin(mx[:, 1], mx[:, 2]))
    return tmin.astype(f32), tmax.astype(f32)


def _point(o, d, t):
    """ray_origin + ray_direction * t + 0.5f  (fma, then add)."""
    return (fma32(d, t[:, None], o) + f32(0.5)).astype(f32)


def occupancy_minmax(o, d, aabb, grids, img, G):
    """ray_sampler.cu:28-78.  grids: list/array of uint8 [G,G,G], one per image slot."""
    tmin, tmax_aabb = aabb_minmax(o, d, aabb)
    step = f32(0.5) / f32(G)
    n = o.shape[0]

    def occ(mask, t):
        out = np.zeros(n, bool)
        ids = np.nonzero(mask)[0]
        if ids.size:
            p = _point(o[ids], d[ids], t[ids])
            for g in np.unique(img[ids]):
                sel = img[ids] == g
                out[ids[sel]] = tex_occupied(grids[g], p[sel])
        return out

    tmin = tmin.copy()
    active = tmin < tmax_aabb
    while active.any():
        hit = occ(active, tmin)
        active &= ~hit
        tmin[active] = (tmin[active] + step).astype(f32)
        active &= tmin < tmax_aabb
    found = tmin < tmax_aabb
    refine = np.full(n, -step * f32(0.5), f32)
    for _ in range(5):
        tmin[found] = (tmin[found] + refine[found]).astype(f32)
        hit = occ(found, tmin)
        mag = (np.abs(refine) * f32(0.5)).astype(f32)
        refine = np.where(hit, -mag, mag).astype(f32)
    tmax = tmax_aabb.copy()
    active = tmax > tmin
    while active.any():
        hit = occ(active, tmax)
        active &= ~hit
        tmax[active] = (tmax[active] - step).astype(f32)
        active &= tmax > tmin
    return tmin, tmax


def get_data(rgba_u8, light_mask, frame_numbers, camera_numbers, grids, landscape, all_ray_idx,
             inverse_krs, camera_origins, aabb, G, width, height, step, filter_light_bloom,
             occupancy=True, samples=True):
    """ray_sampler.cu:196-325 (get_{rays,samples}_{aabb,occupancy}_minmax).  Returns the 9 outputs as numpy."""
    aabb = np.asarray(aabb, f32)
    o_all, d_all, img_all = ray_directions(inverse_krs, camera_origins, landscape, all_ray_idx, width, height)
    if occupancy:
        tmin, tmax = occupancy_minmax(o_all, d_all, aabb, grids, img_all, G)
    else:
        tmin, tmax = aabb_minmax(o_all, d_all, aabb)
    mask = tmin < tmax
    idx = np.asarray(all_ray_idx, np.int64)
    if filter_light_bloom:
        mask = mask & ~np.asarray(light_mask, bool)[idx]
    sel = np.nonzero(mask)[0]
    ridx = idx[sel]
    d = d_all[sel]
    mm = np.stack((tmin[sel], tmax[sel]), 1)
    rgba = (np.asarray(rgba_u8)[ridx].astype(f32) / f32(255.0)).astype(f32)
    img = ridx // (width * height)
    o = np.asarray(camera_origins, f32)[img]
    fn = np.asarray(frame_numbers, np.int32)[img]
    cn = np.asarray(camera_numbers, np.int32)[img]
    if not samples:
        return o, d, rgba, fn, cn, mm, mask, np.zeros(0, f32), np.zeros(0, np.int32)
    # torch's CUDA div-by-scalar multiplies by the float32 reciprocal (BinaryDivTrueKernel.cu)
    inv_step = f32(1.0) / f32(step)
    counts = ((mm[:, 1] - mm[:, 0]).astype(f32) * inv_step).astype(f32).astype(np.int32)
    counts = np.maximum(counts, 0)
    rel = np.repeat(np.arange(sel.size, dtype=np.int32), counts)
    ends = np.cumsum(counts)
    starts = ends - counts
    k = (np.arange(rel.size, dtype=np.int64) - starts[rel]).astype(f32)
    t = fma32(k, np.full_like(k, f32(step)), mm[rel, 0])
    if occupancy and rel.size:
        p = _point(o[rel], d[rel], t)
        keep = np.zeros(rel.size, bool)
        simg = img[rel]
        for g in np.unique(simg):
            s = simg == g
            keep[s] = tex_occupied(grids[g], p[s])
    else:
        keep = np.ones(rel.size, bool)
    return o, d, rgba, fn, cn, mm, mask, t[keep], rel[keep]
