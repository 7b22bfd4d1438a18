"""The 8-bit table format of the compact model (csrc/quantize.cu, DESIGN.md §3.19) restated in numpy, rounding exactly
where the kernels round, and the int8 encode built on tests/encode_oracle.py.

TEST INFRASTRUCTURE ONLY.  Per slice (grid, level, feature) of a segment's fp32 master tables:
  s_c = (c * absmax) / 127                      two fp32 roundings, c from CLIP_RATIOS (fp32)
  q_c = 0 if s_c == 0 else clamp(rint(x / s_c), -127, 127)      fp32 division, round half to even
  err_c = sum (x - s_c q_c)^2                   float64
and the chosen c is the least err_c, ties to the larger c (the earlier in the list).  The kernels sum err_c in another
order than numpy does, so a chosen c is only determined where its two best candidates differ by more than the float64
sum's rounding; `decided` says where.  Scales, codes and folded vectors are bit-exact.

The int8 encode: codes are integers in [-127, 127], which bf16 represents exactly, so encode_oracle.encode over bf16
tables holding the codes and over the folded vectors is the int8 kernels' encode: the gather's fma chain reads the same
floats, the composition the same operands.

MUTANTS (deliberately wrong formats that the CPU tests must reject): "wrong_axis" (the scales of grid k folded into
vector axis k), "half_away" (round half away from zero), "allow_m128" (clamp to -128), "not_folded" (vectors without
the scales), "ties_smaller" (a tie goes to the smaller c).
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np

import encode_oracle as E

F32, F64 = np.float32, np.float64
CLIP_RATIOS = np.array([1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3], F32)
GRID_OF_AXIS = (2, 3, 1, 0)     # axis x, y, z, t is composed with grid yzt, xzt, xyt, xyz (encode_oracle.VECTOR_OF_TERM)
MUTANTS = ("wrong_axis", "half_away", "allow_m128", "not_folded", "ties_smaller")


def scale_of(c, absmax) -> np.float32:
    return F32(F32(F32(c) * F32(absmax)) / F32(127))


def codes_of(x, s, mutant: Optional[str] = None) -> np.ndarray:
    x = np.asarray(x, F32)
    if F32(s) == 0:
        return np.zeros(x.shape, np.int8 if mutant != "allow_m128" else np.int16)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        r = x / F32(s)
    r = np.sign(r) * np.floor(np.abs(r) + F32(0.5)) if mutant == "half_away" else np.rint(r)
    lo = -128 if mutant == "allow_m128" else -127
    return np.clip(r, lo, 127).astype(np.int16 if mutant == "allow_m128" else np.int8)


def slice_errors(x) -> tuple:
    """(absmax, scales [8], errors [8]) of one slice."""
    x = np.asarray(x, F32)
    absmax = F32(np.max(np.abs(x))) if x.size else F32(0)
    scales = np.array([scale_of(c, absmax) for c in CLIP_RATIOS], F32)
    errs = np.array([np.sum((x.astype(F64) - F64(s) * codes_of(x, s).astype(F64)) ** 2) for s in scales], F64)
    return absmax, scales, errs


def choose(errs, mutant: Optional[str] = None) -> int:
    best = np.min(errs)
    hits = np.nonzero(errs == best)[0]
    return int(hits[-1] if mutant == "ties_smaller" else hits[0])


def decided(errs, rel: float = 1e-9) -> bool:
    """The choice does not hinge on the float64 sum's order: its two best candidates differ by more than `rel`."""
    e = np.sort(np.asarray(errs, F64))
    return bool(e[1] - e[0] > rel * max(e[1], 1e-300))


def quantize_grid(master, lt: E.LevelTable, mutant: Optional[str] = None):
    """One grid's fp32 master table (flat, tcnn layout) -> scale [16, 2], clip index [16, 2], errors [16, 2, 8],
    codes int8 [n_entries, 2]."""
    t = np.asarray(master, F32).reshape(-1, 2)
    scale = np.zeros((E.N_LEVELS, 2), F32)
    clip = np.zeros((E.N_LEVELS, 2), np.int32)
    errs = np.zeros((E.N_LEVELS, 2, len(CLIP_RATIOS)), F64)
    codes = np.zeros(t.shape, np.int16 if mutant == "allow_m128" else np.int8)
    for l in range(E.N_LEVELS):
        a, b = int(lt.offset[l]), int(lt.offset[l]) + int(lt.size[l])
        for f in range(2):
            _, sc, er = slice_errors(t[a:b, f])
            ci = choose(er, mutant)
            scale[l, f], clip[l, f], errs[l, f] = sc[ci], ci, er
            codes[a:b, f] = codes_of(t[a:b, f], sc[ci], mutant)
    return scale, clip, errs, codes


def fold_vectors(vectors, scales, mutant: Optional[str] = None) -> np.ndarray:
    """vectors f32 [4, VR, 32], scales f32 [4 grids, 16, 2] -> v'[a][row][2l+f] = s(grid(a), l, f) * v[a][row][2l+f]."""
    v = np.asarray(vectors, F32)
    if mutant == "not_folded":
        return v.copy()
    out = np.empty_like(v)
    for a in range(4):
        g = a if mutant == "wrong_axis" else GRID_OF_AXIS[a]
        out[a] = v[a] * np.asarray(scales[g], F32).reshape(1, 32)
    return out


def quantize_segment(grids: List[np.ndarray], vectors: np.ndarray, lt: E.LevelTable, mutant: Optional[str] = None):
    """A segment's four master grids and its vectors -> (scales [4,16,2], clip [4,16,2], errs [4,16,2,8],
    codes [4][n_entries, 2], folded vectors)."""
    out = [quantize_grid(g, lt, mutant) for g in grids]
    scales = np.stack([o[0] for o in out])
    return (scales, np.stack([o[1] for o in out]), np.stack([o[2] for o in out]), [o[3] for o in out],
            fold_vectors(vectors, scales, mutant))


def int8_field(codes: List[List[np.ndarray]], folded: List[np.ndarray], sorted_frame_numbers, segment_sizes,
               log2_hashmap_size: int = 19) -> E.FieldArrays:
    """The FieldArrays whose encode_oracle.encode is the int8 kernels' encode: bf16 tables holding the codes (exact)."""
    tabs = [[E.bf16_bits(np.asarray(c, F32)).reshape(-1, 2) for c in cs] for cs in codes]
    return E.FieldArrays(tabs, [np.ascontiguousarray(v, F32) for v in folded],
                         [E.segment_log2_hashmap_size(s, log2_hashmap_size) for s in segment_sizes],
                         sorted_frame_numbers, segment_sizes)


def dequantised_encode(codes, scales, vectors, lt: E.LevelTable, x, t, absolute: bool = False) -> np.ndarray:
    """float64 composed features [N, 32] of one segment from the dequantised tables s * q and the UNFOLDED vectors: what
    the int8 encode approximates up to fp32 rounding.  x: normalised positions [N, 3], t: local times [N].  absolute:
    the same sums over the absolute values of every term instead (the scale of the fp32 rounding error)."""
    coords = np.concatenate((np.asarray(x, F32), np.asarray(t, F32)[:, None]), axis=1)
    vr = vectors.shape[1]
    vl = []
    for a in range(4):
        i0, i1, fr = E.row_tap(coords[:, a], vr)
        v0, v1 = vectors[a][i0].astype(F64), vectors[a][i1].astype(F64)
        vl.append(v0 + fr.astype(F64)[:, None] * (v1 - v0))
    out = np.zeros((coords.shape[0], 32), F64)
    for l in range(E.N_LEVELS):
        cells = [E.to_cell(lt.scale[l], coords[:, a]) for a in range(4)]
        for k in range(4):
            ax = E.GRID_AXES[k]
            (ga, fa), (gb, fb), (gc, fc) = (cells[ax[0]], cells[ax[1]], cells[ax[2]])
            tab = codes[k][int(lt.offset[l]):int(lt.offset[l]) + int(lt.size[l])].astype(F64) * scales[k, l].astype(F64)
            tab = np.abs(tab) if absolute else tab
            wd = ((1 - fa.astype(F64), fa.astype(F64)), (1 - fb.astype(F64), fb.astype(F64)),
                  (1 - fc.astype(F64), fc.astype(F64)))
            e = np.zeros((coords.shape[0], 2), F64)
            for c in range(8):
                w = wd[0][c & 1] * wd[1][(c >> 1) & 1] * wd[2][(c >> 2) & 1]
                idx = E.corner_index(c, bool(lt.hashed[l]), int(lt.res[l]), int(lt.size[l]), ga, gb, gc)
                e += w[:, None] * tab[idx]
            v = vl[E.VECTOR_OF_TERM[k]][:, 2 * l:2 * l + 2]
            out[:, 2 * l:2 * l + 2] += e * (np.abs(v) if absolute else v)
    return out
