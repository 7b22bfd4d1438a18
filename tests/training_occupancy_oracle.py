"""numpy restatement of the training occupancy (include/humanrf_b200.h, hrf_training_occupancy_*; DESIGN.md §3.21):
the hull's voxel list, the hashed points, the bound update, the alpha test, the dilation inside the hull and the slot's
bit layout, bit for bit in float32 and uint64.

Every step takes a `mutant` naming a deliberately wrong variant; tests/test_training_occupancy_cpu.py shows that its
checks reject each of them:
  "decay_after_max" : bound = decay * max(bound, sigma)
  "six"             : a 6-neighbourhood dilation
  "leave_hull"      : a dilation that is not limited to the hull
  "no_counter"      : the points' hash without the refresh counter
  "gt"              : live <=> alpha > alpha_thre
  "inf_dead"        : a +inf bound (never evaluated) is dead"""
from __future__ import annotations

import numpy as np

U64, F32 = np.uint64, np.float32
GOLDEN = U64(0x9E3779B97F4A7C15)
MUTANTS = ("decay_after_max", "six", "leave_hull", "no_counter", "gt", "inf_dead")
STEP, ALPHA_THRE = 4e-4, 1e-4


def splitmix64(x):
    with np.errstate(over="ignore"):
        z = np.asarray(x, U64) + GOLDEN
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
        return z ^ (z >> U64(31))


# ------------------------------------------------------------------------------------------------ 1. voxel list
def compact(hull) -> np.ndarray:
    """The hull's voxel indices z G^2 + y G + x, int32, ascending: each occupied voxel goes to the place the running
    count of occupied voxels before it gives."""
    occ = np.asarray(hull).reshape(-1) != 0
    place = np.cumsum(occ) - 1
    ids = np.empty(int(occ.sum()), np.int32)
    ids[place[occ]] = np.arange(occ.size, dtype=np.int64)[occ]
    return ids


# ------------------------------------------------------------------------------------------------ 3. points
def key(seed: int, frame: int, counter: int, mutant=None) -> np.uint64:
    """S(S(S(seed) ^ frame) ^ counter); the frame enters as its uint32 bits."""
    k = splitmix64(splitmix64(U64(seed & (2 ** 64 - 1))) ^ U64(frame & 0xFFFFFFFF))
    return k if mutant == "no_counter" else splitmix64(k ^ U64(counter))


def fractions(ids, k):
    """u_x, u_y, u_z: exact 24-bit fractions (float32) of h = S(key ^ id) and g = S(h)."""
    h = splitmix64(U64(k) ^ np.asarray(ids, np.uint32).astype(U64))
    g = splitmix64(h)
    scale = F32(2.0 ** -24)
    ux = (h >> U64(40)).astype(F32) * scale
    uy = ((h >> U64(16)) & U64(0xFFFFFF)).astype(F32) * scale
    uz = (g >> U64(40)).astype(F32) * scale
    return ux, uy, uz


def points(ids, G: int, seed: int, frame: int, counter: int, mutant=None) -> np.ndarray:
    """float32 [n, 3]: p = fl(fl(fl(i + u) / G) - 0.5) per axis (round to nearest even at every step)."""
    ids = np.asarray(ids, np.int64)
    x, y, z = ids % G, (ids // G) % G, ids // (G * G)
    us = fractions(ids, key(seed, frame, counter, mutant))
    out = [((i.astype(F32) + u) / F32(G)).astype(F32) - F32(0.5) for i, u in zip((x, y, z), us)]
    return np.stack(out, -1).astype(F32)


# ------------------------------------------------------------------------------------------------ 3. bound update
def update(bound, sigma, decay: float, mutant=None) -> np.ndarray:
    bound, sigma = np.asarray(bound, F32), np.asarray(sigma, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        if mutant == "decay_after_max":
            kept = (F32(decay) * np.maximum(bound, sigma)).astype(F32)
        else:
            kept = np.maximum((F32(decay) * bound).astype(F32), sigma)
    out = np.where(np.isinf(bound), sigma, kept)
    return np.where(np.isfinite(sigma), out, F32(np.inf)).astype(F32)


# ------------------------------------------------------------------------------------------------ 4. pack
def live(bound, step: float = STEP, alpha_thre: float = ALPHA_THRE, mutant=None) -> np.ndarray:
    """1.f - expf(-bound * step) >= alpha_thre in float32."""
    bound = np.asarray(bound, F32)
    with np.errstate(over="ignore", invalid="ignore"):
        alpha = F32(1.0) - np.exp((-bound * F32(step)).astype(F32)).astype(F32)
    out = alpha > F32(alpha_thre) if mutant == "gt" else alpha >= F32(alpha_thre)
    if mutant == "inf_dead":
        out = out & np.isfinite(bound)
    return out


def dilate(live_grid, hull, mutant=None) -> np.ndarray:
    """hull AND (some voxel of the 3x3x3 neighbourhood is live), bool [G,G,G]."""
    lv = np.pad(np.asarray(live_grid, bool), 1)
    G = lv.shape[0] - 2
    out = np.zeros((G, G, G), bool)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                if mutant == "six" and abs(dz) + abs(dy) + abs(dx) > 1:
                    continue
                out |= lv[1 + dz:1 + dz + G, 1 + dy:1 + dy + G, 1 + dx:1 + dx + G]
    return out if mutant == "leave_hull" else out & (np.asarray(hull) != 0)


def grid(ids, bound, G: int, step: float = STEP, alpha_thre: float = ALPHA_THRE, mutant=None) -> np.ndarray:
    """uint8 [G,G,G] {0, 255}: hull (rebuilt from ids) AND dilate(live)."""
    hull = np.zeros(G ** 3, bool)
    hull[np.asarray(ids, np.int64)] = True
    lv = np.zeros(G ** 3, bool)
    lv[np.asarray(ids, np.int64)] = live(bound, step, alpha_thre, mutant)
    out = dilate(lv.reshape(G, G, G), hull.reshape(G, G, G), mutant)
    return np.where(out, 255, 0).astype(np.uint8)


def pack_bits(grid_u8) -> np.ndarray:
    """The slot's words (hrf_occgrid_add): voxel i is bit i & 31 of word i >> 5, bits past the last voxel 0."""
    flat = np.asarray(grid_u8).reshape(-1) != 0
    n = flat.size
    padded = np.zeros(((n + 31) // 32) * 32, bool)
    padded[:n] = flat
    w = padded.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)
    return w.sum(1).astype(np.uint32)
