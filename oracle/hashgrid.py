"""Oracle: tiny-cuda-nn multi-resolution hash grid (3-D inputs), restated on the CPU.

TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED: tiny-cuda-nn is an un-vendored, un-pinned
dependency of the reference (README.md:19); this restates its published algorithm
(include/tiny-cuda-nn/encodings/grid.h: grid_scale, grid_resolution, pos_fract, grid_index,
coherent_prime_hash, kernel_grid) as called from
humanrf/scene_representation/decomposition4d.py:79-122,126-129.
"""
from __future__ import annotations

import numpy as np
import torch

from .sampler import fma32

PRIME_Y = np.uint32(2654435761)
PRIME_Z = np.uint32(805459861)


def per_level_scale(coarsest: int = 32, finest: int = 2048, n_levels: int = 16) -> float:
    """decomposition4d.py:73 (computed in float64 by numpy, handed to tcnn as JSON)."""
    return float(np.exp(np.log(finest / coarsest) / (n_levels - 1)))


def level_table(log2_hashmap_size: int, n_levels: int = 16, base_resolution: int = 32,
                pls: float | None = None):
    """Per-level (scale f32, resolution u32, offset u32, size u32, hashed bool).

    grid.h: scale_l = exp2f(l * log2f(pls)) * base - 1 ; res_l = ceil(scale_l) + 1 ;
    params_in_level = min(roundup8(res^3), 2^log2T) ; offsets are running sums (entries).
    All float arithmetic in float32, as tcnn does on the host.
    """
    if pls is None:
        pls = per_level_scale(base_resolution, 2048, n_levels)
    pls32 = np.float32(pls)
    log2_pls = np.log2(pls32, dtype=np.float32)
    scales, ress, offs, sizes, hashed = [], [], [], [], []
    off = 0
    for l in range(n_levels):
        scale = np.float32(np.exp2(np.float32(l) * log2_pls, dtype=np.float32) * np.float32(base_resolution)
                           - np.float32(1.0))
        res = int(np.ceil(scale)) + 1
        dense = res ** 3
        n = min((dense + 7) // 8 * 8, 1 << log2_hashmap_size) if dense < 2 ** 31 else (1 << log2_hashmap_size)
        # grid_index: hashed iff the dense stride product exceeds the level's size
        scales.append(scale); ress.append(res); offs.append(off); sizes.append(n)
        hashed.append(dense > n)
        off += n
    return (np.array(scales, np.float32), np.array(ress, np.uint32), np.array(offs, np.uint32),
            np.array(sizes, np.uint32), np.array(hashed, bool), off)


def _fma32(a: np.ndarray, b: np.ndarray, c) -> np.ndarray:
    """float32 fused multiply-add, rounded once (a float64 sum rounded again to float32 would round twice when it lands
    on an fp32 midpoint, and that moves the cell of a position whose scale * x + 0.5 sits next to an integer)."""
    return fma32(a, b, np.float32(c))


def corner_indices_and_weights(x: np.ndarray, scale: np.float32, res: int, size: int, hashed: bool):
    """x: [N,3] float32 in [0,1].  Returns idx [N,8] int64 (entry index inside the level) and
    w [N,8] float32, corner order idx bit d <-> +1 along dim d (grid.h kernel_grid)."""
    pos = _fma32(x, np.broadcast_to(np.float32(scale), x.shape), 0.5)          # pos_fract: fmaf(scale,x,0.5)
    fl = np.floor(pos)
    g = fl.astype(np.int64).astype(np.uint32)                                   # (uint32_t)(int)floorf
    fr = (pos - fl).astype(np.float32)
    n = x.shape[0]
    idx = np.empty((n, 8), np.int64)
    w = np.empty((n, 8), np.float32)
    for c in range(8):
        wc = np.ones(n, np.float32)
        gl = []
        for d in range(3):
            if (c >> d) & 1:
                wc = wc * fr[:, d]
                gl.append(g[:, d] + np.uint32(1))
            else:
                wc = wc * (np.float32(1.0) - fr[:, d])
                gl.append(g[:, d])
        if hashed:
            h = gl[0] ^ (gl[1] * PRIME_Y) ^ (gl[2] * PRIME_Z)                    # uint32 wrap-around
        else:
            h = gl[0] + gl[1] * np.uint32(res) + gl[2] * np.uint32(res * res)   # uint32 wrap-around
        idx[:, c] = (h % np.uint32(size)).astype(np.int64)
        w[:, c] = wc
    return idx, w


def encode(table: torch.Tensor, x: torch.Tensor, log2_hashmap_size: int, sparse_grad: bool = False) -> torch.Tensor:
    """table: [entries, 2] float (any grad-enabled leaf); x: [N,3] float32 in [0,1].
    Returns [N, 32] float32, level-major feature pairs; fp32 blend (fma accumulate order 0..7).
    sparse_grad: gather through an embedding lookup whose gradient is a sparse tensor (same values; the CPU training
    baseline uses it so that 64 gathers per grid do not each allocate a dense zero gradient of the whole table)."""
    scales, ress, offs, sizes, hashed, total = level_table(log2_hashmap_size)
    assert table.shape[0] == total, (table.shape, total)
    xn = x.detach().cpu().numpy().astype(np.float32)
    outs = []
    for l in range(16):
        idx, w = corner_indices_and_weights(xn, scales[l], int(ress[l]), int(sizes[l]), bool(hashed[l]))
        idx_t = torch.from_numpy(idx + int(offs[l]))
        w_t = torch.from_numpy(w).to(table.dtype)
        if sparse_grad:
            vals = torch.nn.functional.embedding(idx_t.reshape(-1), table, sparse=True).reshape(-1, 8, 2)
        else:
            vals = table[idx_t.reshape(-1)].reshape(-1, 8, 2)
        acc = torch.zeros((xn.shape[0], 2), dtype=table.dtype)
        for c in range(8):
            acc = acc + w_t[:, c:c + 1] * vals[:, c]
        outs.append(acc)
    return torch.cat(outs, dim=1)
