"""Host-side layout of the multi-resolution hash grids and the packed MLP weight blob.

Level table: tiny-cuda-nn's GridEncoding constructor (grid.h: grid_scale / grid_resolution /
offset table) as configured by humanrf/scene_representation/decomposition4d.py:73-122 and
humanrf.py:106-109.  All float math in float32, like tcnn on the host.
"""
from __future__ import annotations

import numpy as np

PREDEFINED_SEGMENT_SIZES = (6, 12, 25, 50, 100)  # humanrf/adaptive_temporal_partitioning.py:8
N_LEVELS = 16
N_FEATURES_PER_LEVEL = 2


def segment_log2_hashmap_size(segment_size: int, log2_hashmap_size: int) -> int:
    """humanrf.py:106-109."""
    return int(np.round(np.log2(segment_size / max(PREDEFINED_SEGMENT_SIZES) * (2 ** log2_hashmap_size))))


class GridLayout:
    def __init__(self, log2_hashmap_size: int, n_levels: int = N_LEVELS, base_resolution: int = 32,
                 finest_resolution: int = 2048):
        pls = np.float32(np.exp(np.log(finest_resolution / base_resolution) / (n_levels - 1)))  # decomposition4d.py:73
        log2_pls = np.log2(pls, dtype=np.float32)
        self.log2_hashmap_size = log2_hashmap_size
        self.scale = np.zeros(n_levels, np.float32)
        self.res = np.zeros(n_levels, np.uint32)
        self.offset = np.zeros(n_levels, np.uint32)
        self.size = np.zeros(n_levels, np.uint32)
        self.hashed_mask = 0
        off = 0
        for l in range(n_levels):
            s = np.float32(np.exp2(np.float32(l) * log2_pls, dtype=np.float32) * np.float32(base_resolution)
                           - np.float32(1.0))
            r = int(np.ceil(s)) + 1
            dense = r ** 3
            n = min((dense + 7) // 8 * 8, 1 << log2_hashmap_size) if dense < 2 ** 31 else (1 << log2_hashmap_size)
            self.scale[l], self.res[l], self.offset[l], self.size[l] = s, r, off, n
            if dense > n:
                self.hashed_mask |= 1 << l
                assert n == 1 << log2_hashmap_size
            off += n
        self.n_entries = off

    @property
    def n_params(self) -> int:
        return self.n_entries * N_FEATURES_PER_LEVEL


# ---- packed bf16 MLP blob (wgmma K-major no-swizzle core-matrix layout, csrc/field_common.cuh) ----
MLP_SIGMA_PARAMS = 64 * 32 + 16 * 64          # 3072  (tcnn FullyFusedMLP, output padded to 16)
MLP_BLOB_ELEMS = 22528 // 2


def blob_offsets(camera_embedding_dim: int = 0):
    """Byte offsets of the five weight matrices inside the blob (kWSig1.., w_col2/w_col3 in csrc/field_common.cuh)."""
    k = color_in_width(camera_embedding_dim)
    return (0, 4096, 6144, 6144 + 128 * k, 6144 + 128 * k + 8192)


def color_in_width(camera_embedding_dim: int) -> int:
    """tcnn Composite[SH(16) | Identity(15 + E)] padded to a multiple of 16 with 1.0 (humanrf.py:135-156)."""
    return 32 if camera_embedding_dim == 0 else 48


def mlp_layers(camera_embedding_dim: int = 0):
    k = color_in_width(camera_embedding_dim)
    return ((64, 32), (16, 64), (64, k), (64, 64), (16, 64))


def mlp_color_params(camera_embedding_dim: int = 0) -> int:
    return sum(o * i for o, i in mlp_layers(camera_embedding_dim)[2:])


MLP_COLOR_PARAMS = mlp_color_params(0)  # 7168


def mlp_blob_permutation(camera_embedding_dim: int = 0):
    """(dst, src): blob_elems[dst] = cat(sigma_params, color_params)[src]; untouched blob elements stay 0."""
    dst, src = [], []
    s0 = 0
    for (n_out, n_in), off in zip(mlp_layers(camera_embedding_dim), blob_offsets(camera_embedding_dim)):
        n, k = np.meshgrid(np.arange(n_out), np.arange(n_in), indexing="ij")
        d = off // 2 + ((k // 8) * (n_out // 8) + n // 8) * 64 + (n % 8) * 8 + (k % 8)
        dst.append(d.reshape(-1))
        src.append(s0 + (n * n_in + k).reshape(-1))
        s0 += n_out * n_in
    return np.concatenate(dst).astype(np.int64), np.concatenate(src).astype(np.int64)
