"""numpy restatement of the error map (humanrf_b200/csrc/error_map.cu, DESIGN.md §3.20), bit for bit: the tile mapping
in both orientations, the per-ray error and its fixed point, the EMA, the integer weights and scan, the SplitMix64 hash
and the draw.  `mutant` names a deliberate defect for the checks to reject (test_error_map_cpu.py):
  "orientation"   portrait slots mapped as landscape;
  "npix"          every tile counted as T x T pixels, border tiles included;
  "lower_bound"   the first tile whose CDF reaches the target instead of exceeding it;
  "ema_unsampled" tiles without rays take the EMA towards 0 as well;
  "uniform_ceil"  the uniform share rounded up.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.sampler import fma32

F32, U64 = np.float32, np.uint64
M32 = U64(0xFFFFFFFF)
GOLDEN = U64(0x9E3779B97F4A7C15)


class Geometry:
    def __init__(self, landscape, width: int, height: int, tile: int):
        self.landscape = np.asarray(landscape, bool)
        self.B, self.W, self.H, self.T = len(self.landscape), int(width), int(height), int(tile)
        self.P = self.W * self.H
        self.tiles_w, self.tiles_h = -(-self.W // self.T), -(-self.H // self.T)
        self.nt = self.tiles_w * self.tiles_h
        self.num_tiles = self.B * self.nt

    def slot_shape(self, slot, mutant=None):
        ls = self.landscape[slot] | (mutant == "orientation")
        return np.where(ls, self.W, self.H), np.where(ls, self.H, self.W), np.where(ls, self.tiles_w, self.tiles_h)

    def tile_of_pixel(self, idx, mutant=None):
        idx = np.asarray(idx, np.int64)
        slot, p = idx // self.P, idx % self.P
        w, _, rt = self.slot_shape(slot, mutant)
        x, y = p % w, p // w
        return slot * self.nt + (y // self.T) * rt + x // self.T

    def tile_extent(self, t, mutant=None):
        """(slot, x0, y0, cw, ch, w) of tiles t."""
        t = np.asarray(t, np.int64)
        slot, l = t // self.nt, t % self.nt
        w, h, rt = self.slot_shape(slot, mutant)
        x0, y0 = (l % rt) * self.T, (l // rt) * self.T
        cw, ch = np.minimum(self.T, w - x0), np.minimum(self.T, h - y0)
        if mutant == "npix":
            cw, ch = np.full_like(cw, self.T), np.full_like(ch, self.T)
        return slot, x0, y0, cw, ch, w

    def npix(self, mutant=None):
        _, _, _, cw, ch, _ = self.tile_extent(np.arange(self.num_tiles), mutant)
        return (cw * ch).astype(np.int64)

    def max_total(self, max_ema: float) -> float:
        """The bound hrf_error_map_num_tiles checks against 2^63."""
        return self.B * self.P * max(max_ema, 1.0) * 2.0 ** 24 + self.num_tiles


def sampler_pixel_xy(geo: Geometry, idx):
    """The sampler's pixel coordinates (sampler.cu ray_minmax_kernel): (slot, x, y)."""
    idx = np.asarray(idx, np.int64)
    slot = idx // geo.P
    w = np.where(geo.landscape[slot], geo.W, geo.H)
    h = np.where(geo.landscape[slot], geo.H, geo.W)
    return slot, idx % w, (idx // w) % h


# ------------------------------------------------------------------------------------------------ accumulate
def respond(color, w, bg, em, b):
    """camera_common.cuh respond(): color + em fg + w b with fg = fma(-(1 - w), bg, color), zero em / b not added."""
    fg = fma32(-(F32(1) - w).astype(F32), bg, color)
    pred = np.where(em != 0, fma32(em, fg, color), color).astype(F32)
    return np.where(b != 0, fma32(w, b, pred), pred).astype(F32)


def target(m, rgb, bg, response: bool):
    """gt = rgb m + bg (1 - m) rounded as the loss kernel in use is compiled: hrf_train_loss fma(m, rgb, (1 - m) bg),
    hrf_train_loss_response fma(1 - m, bg, m rgb)."""
    m, rgb, bg = (np.asarray(a, F32) for a in (m, rgb, bg))
    om = (F32(1) - m).astype(F32)
    return fma32(om, bg, (m * rgb).astype(F32)) if response else fma32(m, rgb, (om * bg).astype(F32))


def ray_error(color, wsum, rgba, bg, delta, table=None, cams=None):
    color, rgba, bg = (np.asarray(a, F32) for a in (color, rgba, bg))
    delta = F32(delta)
    m = rgba[:, 3]
    e = None
    if table is not None:
        table = np.asarray(table, F32)
        cams = np.asarray(cams, np.int64)
        ok = (cams >= 0) & (cams < table.shape[0])
        row = np.where(ok[:, None], table[np.where(ok, cams, 0)], F32(0))
        w = np.asarray(wsum, F32).reshape(-1)
    for k in range(3):
        c = color[:, k]
        if table is not None:
            c = respond(c, w, bg[:, k], row[:, k], row[:, 3 + k])
        gt = target(m, rgba[:, k], bg[:, k], table is not None)
        x = (c - gt).astype(F32)
        ax = np.abs(x)
        h = np.where(ax < delta, ((x * F32(0.5)).astype(F32) * x).astype(F32),
                     (fma32(np.full_like(ax, delta), F32(-0.5), ax) * delta).astype(F32))
        e = h if e is None else (e + h).astype(F32)
    return e


def quantise(e):
    s = (np.asarray(e, F32) * F32(2.0 ** 32)).astype(F32)
    with np.errstate(invalid="ignore"):
        ok = s < F32(2.0 ** 32)
        q = np.where(ok, np.rint(np.where(ok, s, 0)).astype(np.float64), 0).astype(U64)
    return np.where(ok, q, M32)


def accumulate(geo: Geometry, pixels, e, sums=None, counts=None):
    """(sum uint64 [tiles], count uint32 [tiles], error bit) after adding the rays' fixed-point errors."""
    sums = np.zeros(geo.num_tiles, U64) if sums is None else sums.copy()
    counts = np.zeros(geo.num_tiles, np.uint32) if counts is None else counts.copy()
    pixels = np.asarray(pixels, np.int64)
    ok = (pixels >= 0) & (pixels < geo.B * geo.P)
    t = geo.tile_of_pixel(pixels[ok])
    np.add.at(sums, t, quantise(e)[ok])
    np.add.at(counts, t, np.uint32(1))
    return sums, counts, int(not ok.all())


# ------------------------------------------------------------------------------------------------ update
def update(geo: Geometry, ema, sums, counts, beta, floor, mutant=None):
    """(new ema float32 [tiles], cdf uint64 [tiles]); the sums and counts are cleared by the kernel."""
    ema = np.asarray(ema, F32).copy()
    c = np.asarray(counts, np.uint32)
    hit = c > 0 if mutant != "ema_unsampled" else np.ones(c.shape, bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        m = (np.asarray(sums, U64).astype(np.float64) / np.maximum(c, 1).astype(np.float64) * 2.0 ** -32).astype(F32)
    new = fma32(np.full_like(ema, F32(beta)), (m - ema).astype(F32), ema)
    ema = np.where(hit, new, ema).astype(F32)
    return ema, cdf_of(geo, ema, floor, mutant)


def weights(geo: Geometry, ema, floor, mutant=None):
    v = np.maximum(np.asarray(ema, F32), F32(floor)).astype(np.float64) * geo.npix(mutant).astype(np.float64) * 2.0 ** 24
    return np.rint(v).astype(U64)


def cdf_of(geo: Geometry, ema, floor, mutant=None):
    return np.cumsum(weights(geo, ema, floor, mutant), dtype=U64)


# ------------------------------------------------------------------------------------------------ draw
def splitmix64(x):
    with np.errstate(over="ignore"):
        z = np.asarray(x, U64) + GOLDEN
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
        return z ^ (z >> U64(31))


def umulhi(a, b):
    """High 64 bits of the 128-bit product (CUDA __umul64hi)."""
    a, b = np.broadcast_arrays(np.asarray(a, U64), np.asarray(b, U64))
    al, ah, bl, bh = a & M32, a >> U64(32), b & M32, b >> U64(32)
    ll, lh, hl, hh = al * bl, al * bh, ah * bl, ah * bh
    mid = (ll >> U64(32)) + (lh & M32) + (hl & M32)
    return hh + (lh >> U64(32)) + (hl >> U64(32)) + (mid >> U64(32))


def hashes(seed: int, counter: int, rays, stream: int):
    with np.errstate(over="ignore"):
        key = splitmix64(splitmix64(U64(seed)) ^ U64(counter))
        return splitmix64(key ^ (U64(4) * np.asarray(rays, U64) + U64(stream)))


def num_uniform(f: float, R: int, mutant=None) -> int:
    return math.ceil(f * R) if mutant == "uniform_ceil" else math.floor(f * R)


def pick_tile(cdf, targets, mutant=None):
    return np.searchsorted(np.asarray(cdf, U64), np.asarray(targets, U64),
                           side="left" if mutant == "lower_bound" else "right").astype(np.int64)


def draw(geo: Geometry, cdf, seed: int, counter: int, R: int, f: float, mutant=None):
    """(pool indices int64 [R], the tile of every importance ray or -1 for a uniform ray)."""
    r = np.arange(R, dtype=np.int64)
    h0 = hashes(seed, counter, r, 0)
    nu = num_uniform(f, R, mutant)
    out = umulhi(h0, U64(geo.B * geo.P)).astype(np.int64)
    tiles = np.full(R, -1, np.int64)
    imp = r >= nu
    t = pick_tile(cdf, umulhi(h0[imp], np.asarray(cdf, U64)[-1]), mutant)
    slot, x0, y0, cw, ch, w = geo.tile_extent(t, mutant)
    k = umulhi(hashes(seed, counter, r[imp], 1), (cw * ch).astype(U64)).astype(np.int64)
    out[imp] = slot * geo.P + (y0 + k // cw) * w + x0 + k % cw
    tiles[imp] = t
    return out, tiles


def target_probabilities(geo: Geometry, cdf, f: float, R: int):
    """Probability of each tile for one ray of an R-ray batch: its pixel share on the uniform rays, its CDF weight share
    on the others."""
    cdf = np.asarray(cdf, U64)
    w = np.diff(np.concatenate(([0], cdf.astype(object)))).astype(np.float64)
    nu = math.floor(f * R)
    return (nu * geo.npix() / (geo.B * geo.P) + (R - nu) * w / float(cdf[-1])) / R
