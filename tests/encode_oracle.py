"""The hash-grid encode of the field kernels (csrc/field_common.cuh: load_sample -> to_cell -> corner_indices /
corner_weights -> gather_level -> make_row_tap2 / lerp_row_tap -> the four-term composition) restated in numpy,
rounding exactly where the kernels round.

TEST INFRASTRUCTURE ONLY.  The kernels pin nearly all of their arithmetic: __fadd_rn / __fmul_rn in load_sample,
__fmaf_rn in to_cell, make_row_tap2 and the 8-step gather chain, products in corner_weights that cannot be contracted,
and no -ftz / -use_fast_math (denormals follow IEEE).  So the per-grid features e_k that the forward saves for the
backward (`egrid`) are determined to the bit, and `encode` returns them as the exact u32 words the kernel writes.

Two expressions are left to nvcc's default contraction (-fmad=true): the vector lerp v0 + frac * (v1 - v0) and the sum
e0*vt + e1*vz + e2*vx + e3*vy.  For each composed feature the reference enumerates every way they can be contracted
(VARIANTS: lerp fused or not; the first add as a plain add of two products or an fma over either product; the second
and third adds fused or not: 2 x 3 x 2 x 2 = 24) and the comparison accepts a kernel output iff one of them produces
its bf16 bits.  Outputs whose variants disagree are flagged as ambiguous; everywhere else the composed bits are
determined too.

Float arithmetic: numpy float32 add / sub / mul round to nearest even like the kernel's; `fma32` is an exactly rounded
fused multiply-add (the product is exact in float64, the sum is carried with its TwoSum tail, and the one case where
rounding the float64 sum to float32 would round twice -- the sum landed on an fp32 midpoint -- is decided by the tail).

Non-finite positions are unspecified (neither the kernels nor this reference promise anything for them).
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

F32, F64 = np.float32, np.float64
PRIME_Y = np.uint32(2654435761)   # tcnn coherent_prime_hash
PRIME_Z = np.uint32(805459861)
N_LEVELS = 16
PREDEFINED_SEGMENT_SIZES = (6, 12, 25, 50, 100)   # humanrf/adaptive_temporal_partitioning.py:8

# Contraction choices nvcc may make for the two expressions it is free to fuse: (lerp, first add, second add, third add).
# first add of  a*b + c*d:  "mul" = add of two rounded products, "fma_ab" = fma(a, b, c*d), "fma_cd" = fma(c, d, a*b).
VARIANTS = tuple(itertools.product(("fused", "unfused"), ("mul", "fma_ab", "fma_cd"), ("fused", "unfused"),
                                   ("fused", "unfused")))
MUTANTS = ("to_cell_unfused", "corners_reversed", "scale_ulp_up", "t_half_offset", "lerp_two_products", "bf16_truncate")
MUTANT_SCALE_LEVEL = 5   # the level whose scale "scale_ulp_up" moves


def variant_name(v) -> str:
    return f"lerp={v[0]} add1={v[1]} add2={v[2]} add3={v[3]}"


# ---------------------------------------------------------------------------------------------------- float helpers
def f32(x) -> np.ndarray:
    return np.asarray(x, dtype=F32)


def fadd(a, b):
    return f32(a) + f32(b)


def fsub(a, b):
    return f32(a) - f32(b)


def fmul(a, b):
    return f32(a) * f32(b)


def fma32(a, b, c) -> np.ndarray:
    """fp32 a * b + c rounded once, to nearest even (CUDA __fmaf_rn)."""
    a, b, c = np.broadcast_arrays(f32(a), f32(b), f32(c))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(F64) * b.astype(F64)          # exact: 24 + 24 significant bits fit in 53
        cd = c.astype(F64)
        s = p + cd
        bb = s - p
        tail = (p - (s - bb)) + (cd - bb)          # TwoSum: s + tail == p + c exactly
        r = s.astype(F32)
        # s sits on an fp32 midpoint only if it is not an fp32 value; its other fp32 neighbour is `o`
        o = np.nextafter(r, np.where(s > r.astype(F64), F32(np.inf), F32(-np.inf))).astype(F32)
        on_mid = (s != r.astype(F64)) & (s == (r.astype(F64) + o.astype(F64)) * 0.5)
        # the exact value lies on the tail's side of the midpoint: round towards o iff the tail points at it
        to_o = on_mid & (tail != 0) & ((tail > 0) == (o.astype(F64) > r.astype(F64)))
    return np.where(to_o, o, r).astype(F32)


def bf16_bits(x, truncate: bool = False) -> np.ndarray:
    """fp32 -> bf16 bits, round to nearest even (__float2bfloat16_rn); truncate=True drops the low half instead."""
    u = f32(x).view(np.uint32).astype(np.uint64)
    if truncate:
        out = u >> 16
    else:
        out = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    out = np.where(np.isnan(f32(x)), 0x7FFF, out)
    return out.astype(np.uint16)


def bf16_to_f32(bits) -> np.ndarray:
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(F32)


def pack_bf16x2(lo_bits, hi_bits) -> np.ndarray:
    return np.asarray(lo_bits, np.uint32) | (np.asarray(hi_bits, np.uint32) << 16)


# ---------------------------------------------------------------------------------------------------- model layout
def segment_log2_hashmap_size(segment_size: int, log2_hashmap_size: int = 19) -> int:
    """humanrf.py:106-109: the table of a segment scales with its share of the largest predefined segment."""
    return int(np.round(np.log2(segment_size / max(PREDEFINED_SEGMENT_SIZES) * 2.0 ** log2_hashmap_size)))


@dataclass
class LevelTable:
    scale: np.ndarray    # f32 [16]
    res: np.ndarray      # u32 [16]
    offset: np.ndarray   # u32 [16] first entry of the level
    size: np.ndarray     # u32 [16] entries of the level
    hashed: np.ndarray   # bool [16]
    n_entries: int


def level_table(log2T: int, base_resolution: int = 32, finest_resolution: int = 2048,
                n_levels: int = N_LEVELS) -> LevelTable:
    """tcnn grid.h as configured by decomposition4d.py:73 (per-level scale computed in float64, handed over as a float):
    scale_l = exp2f(l * log2f(pls)) * base - 1, res_l = ceil(scale_l) + 1, entries = min(next multiple of 8 of res^3,
    2^log2T); a level is hashed iff res^3 exceeds its entries.  Float math in float32, as tcnn does on the host."""
    pls = F32(np.exp(np.log(finest_resolution / base_resolution) / (n_levels - 1)))
    log2_pls = np.log2(pls, dtype=F32)
    scale = np.zeros(n_levels, F32)
    res = np.zeros(n_levels, np.uint32)
    offset = np.zeros(n_levels, np.uint32)
    size = np.zeros(n_levels, np.uint32)
    hashed = np.zeros(n_levels, bool)
    off = 0
    for l in range(n_levels):
        s = F32(np.exp2(F32(l) * log2_pls, dtype=F32) * F32(base_resolution) - F32(1.0))
        r = int(np.ceil(s)) + 1
        dense = r ** 3
        n = min(-(-dense // 8) * 8, 1 << log2T)
        scale[l], res[l], offset[l], size[l], hashed[l] = s, r, off, n, dense > n
        off += n
    return LevelTable(scale, res, offset, size, hashed, off)


def frame_luts(sorted_frame_numbers: Sequence[int], segment_sizes: Sequence[int], t_half_offset: bool = False):
    """humanrf.py:79-103: frame -> segment (-1: none) and frame -> local index / frames in the segment, the quotient
    taken in float64 and stored as float32.  t_half_offset: the wrong rule (local + 0.5) / n (a mutant)."""
    num = len(sorted_frame_numbers)
    end = np.cumsum(segment_sizes).astype(np.int64)
    end[-1] = min(end[-1], num)
    start = np.concatenate(([0], end[:-1]))
    f2s = np.full(sorted_frame_numbers[-1] + 1, -1, np.int32)
    f2t = np.full(sorted_frame_numbers[-1] + 1, -1, F32)
    for s in range(len(segment_sizes)):
        frames = [sorted_frame_numbers[j] for j in range(start[s], end[s])]
        for local, fr in enumerate(frames):
            f2s[fr] = s
            f2t[fr] = ((local + 0.5) if t_half_offset else local) / len(frames)
    return f2s, f2t


@dataclass
class FieldArrays:
    """What the encode reads: per segment four bf16 tables (u16 bits [entries, 2], level-major as tcnn), the fp32 vectors
    [4, VR, 32] and log2T; the frame LUTs; the layout of the grids."""
    tables: List[List[np.ndarray]]
    vectors: List[np.ndarray]
    log2T: List[int]
    sorted_frame_numbers: Sequence[int]
    segment_sizes: Sequence[int]
    levels: List[LevelTable] = field(default_factory=list)

    def __post_init__(self):
        self.levels = [level_table(l2) for l2 in self.log2T]
        for s, lt in enumerate(self.levels):
            assert all(t.shape == (lt.n_entries, 2) and t.dtype == np.uint16 for t in self.tables[s])
            assert self.vectors[s].dtype == F32 and self.vectors[s].shape[0] == 4 and self.vectors[s].shape[2] == 32

    @property
    def vec_res(self) -> int:
        return int(self.vectors[0].shape[1])


def field_from_fp32(grids: List[List[np.ndarray]], vectors: List[np.ndarray], sorted_frame_numbers, segment_sizes,
                    log2_hashmap_size: int = 19) -> FieldArrays:
    """From the fp32 master parameters (flat tcnn tables of 2 * entries values per grid): the bf16 shadows are their
    round-to-nearest-even copies."""
    tabs = [[bf16_bits(np.asarray(g, F32)).reshape(-1, 2) for g in gs] for gs in grids]
    return FieldArrays(tabs, [np.ascontiguousarray(v, F32) for v in vectors],
                       [segment_log2_hashmap_size(s, log2_hashmap_size) for s in segment_sizes], sorted_frame_numbers,
                       segment_sizes)


# ---------------------------------------------------------------------------------------------------- samples
def load_query(positions, frame_numbers):
    """Query form: x = positions + 0.5 per component (one fp32 add)."""
    p = f32(positions)
    return fadd(p, F32(0.5)), np.asarray(frame_numbers, np.int64)


def load_rays(ray_origins, ray_directions, ray_frames, distances, ray_indices):
    """Ray-batch form: p = o[r] + t * d[r] (an fp32 multiply, then an fp32 add), x = p + 0.5."""
    ri = np.asarray(ray_indices, np.int64)
    t = f32(distances)[:, None]
    p = fadd(f32(ray_origins)[ri], fmul(t, f32(ray_directions)[ri]))
    return fadd(p, F32(0.5)), np.asarray(ray_frames, np.int64)[ri]


def segment_and_time(fa: FieldArrays, frames, t_half_offset: bool = False):
    """load_sample's frame rule: a frame < 0, >= the LUT size, or mapped to no segment has no segment (-1)."""
    f2s, f2t = frame_luts(fa.sorted_frame_numbers, fa.segment_sizes, t_half_offset)
    fr = np.asarray(frames, np.int64)
    ok = (fr >= 0) & (fr < f2s.size)
    frc = np.where(ok, fr, 0)
    seg = np.where(ok, f2s[frc], -1)
    seg = np.where((seg >= 0) & (seg < len(fa.tables)), seg, -1)
    t = np.where(ok, f2t[frc], F32(0)).astype(F32)
    return seg.astype(np.int64), t


# ---------------------------------------------------------------------------------------------------- encode pieces
def to_cell(scale, v, fused: bool = True):
    """pos = fmaf(scale, x, 0.5); cell = (uint32)(int)floorf(pos); frac = pos - floor."""
    v = f32(v)
    p = fma32(scale, v, F32(0.5)) if fused else fadd(fmul(scale, v), F32(0.5))
    fl = np.floor(p)
    return fl.astype(np.int64).astype(np.uint32), fsub(p, fl)


def corner_index(k: int, hashed: bool, res: int, size: int, ga, gb, gc) -> np.ndarray:
    """Corner k (bit d set: +1 along dimension d) of a cell: the coherent prime hash masked to the power-of-two size, or
    the dense x + y res + z res^2 in uint32 arithmetic, modulo the size."""
    one = np.uint32(1)
    a = ga + one if k & 1 else ga
    b = gb + one if k & 2 else gb
    c = gc + one if k & 4 else gc
    if hashed:
        return (a ^ (b * PRIME_Y) ^ (c * PRIME_Z)) & np.uint32(size - 1)
    return (a + b * np.uint32(res) + c * np.uint32(res * res)) % np.uint32(size)


def gather_level(tab_level: np.ndarray, hashed: bool, res: int, size: int, ca, cb, cc, reverse: bool = False):
    """Trilinear blend of one level of one grid -> fp32 [N, 2]: weights multiplied in dimension order, then the fma chain
    acc = fma(w_k, table value, acc) over corners 0..7 (reverse=True: 7..0, a mutant)."""
    (ga, fa), (gb, fb), (gc, fc) = ca, cb, cc
    one = F32(1.0)
    wd = ((fsub(one, fa), fa), (fsub(one, fb), fb), (fsub(one, fc), fc))
    acc = np.zeros((ga.shape[0], 2), F32)
    for k in (range(7, -1, -1) if reverse else range(8)):
        w = fmul(fmul(wd[0][k & 1], wd[1][(k >> 1) & 1]), wd[2][(k >> 2) & 1])
        vals = bf16_to_f32(tab_level[corner_index(k, hashed, res, size, ga, gb, gc)])
        acc = fma32(w[:, None], vals, acc)
    return acc


def row_tap(coord, vec_res: int):
    """make_row_tap2: c = fmaf(coord, vec_res, -0.5); rows floor(c) and floor(c) + 1 clamped into [0, vec_res)."""
    c = fma32(coord, F32(vec_res), F32(-0.5))
    fl = np.floor(c)
    i0 = np.clip(np.maximum(fl, F32(0)).astype(np.int64), 0, vec_res - 1)
    i1 = np.clip(np.minimum(fadd(fl, F32(1)), F32(vec_res - 1)).astype(np.int64), 0, vec_res - 1)
    return i0, i1, fsub(c, fl)


def lerp(v0, v1, frac, how: str):
    if how == "fused":
        return fma32(frac, fsub(v1, v0), v0)
    if how == "unfused":
        return fadd(v0, fmul(frac, fsub(v1, v0)))
    if how == "two_products":                    # (1 - f) v0 + f v1: a mutant
        return fadd(fmul(fsub(F32(1), frac), v0), fmul(frac, v1))
    raise ValueError(how)


def compose(e, v, variant) -> np.ndarray:
    """e0*vt + e1*vz + e2*vx + e3*vy with one contraction variant; e[k], v[k] are the k-th term's factors."""
    (a, b), (c, d), (g, h), (i, j) = zip(e, v)
    first = {"mul": lambda: fadd(fmul(a, b), fmul(c, d)), "fma_ab": lambda: fma32(a, b, fmul(c, d)),
             "fma_cd": lambda: fma32(c, d, fmul(a, b))}[variant[1]]()
    second = fma32(g, h, first) if variant[2] == "fused" else fadd(first, fmul(g, h))
    return fma32(i, j, second) if variant[3] == "fused" else fadd(second, fmul(i, j))


# ---------------------------------------------------------------------------------------------------- the encode
GRID_AXES = ((0, 1, 2), (0, 1, 3), (1, 2, 3), (0, 2, 3))   # decomposition4d.py:126-129: xyz, xyt, yzt, xzt
VECTOR_OF_TERM = (3, 2, 0, 1)                                # tensor_composition.cu:49-52: xyz*v_t + xyt*v_z + yzt*v_x + xzt*v_y


@dataclass
class Encoding:
    seg: np.ndarray          # int [N], -1: no segment
    egrid: np.ndarray        # u32 [64, N]: bf16x2 of e_k at row 4 l + k; 0 in rows without a segment (unwritten by contract)
    feat: np.ndarray         # u16 [N, 32]: composed features of variant VARIANTS[0]; 0 in rows without a segment
    ambiguous: np.ndarray    # bool [N, 32]: the contraction variants disagree on these bits
    check: Optional[dict] = None   # comparison with kernel output (encode(..., feat_gpu=...))


def encode(fa: FieldArrays, x: np.ndarray, frames, feat_gpu: Optional[np.ndarray] = None,
           mutant: Optional[str] = None) -> Encoding:
    """x: fp32 [N, 3] normalised positions (load_query / load_rays), frames [N].  feat_gpu: u16 [N, 32] composed
    features a kernel wrote; with it the result's `check` reports, over rows with a segment, the outputs no contraction
    variant explains (`mismatch`, and their rows), the ambiguous ones, and how many outputs each variant reproduces.
    mutant: one of MUTANTS, a deliberately wrong reference."""
    assert mutant is None or mutant in MUTANTS, mutant
    x = f32(x)
    n = x.shape[0]
    seg, t = segment_and_time(fa, frames, t_half_offset=mutant == "t_half_offset")
    coords = np.concatenate((x, t[:, None]), axis=1)     # [N, 4]: x, y, z, t
    vr = fa.vec_res
    taps = [row_tap(coords[:, a], vr) for a in range(4)]
    egrid = np.zeros((4 * N_LEVELS, n), np.uint32)
    feat = np.zeros((n, 32), np.uint16)
    amb = np.zeros((n, 32), bool)
    nv = len(VARIANTS)
    chk = None
    if feat_gpu is not None:
        feat_gpu = np.asarray(feat_gpu).view(np.uint16).reshape(n, 32)
        chk = dict(outputs=0, mismatch=0, ambiguous=0, mismatch_rows=set(), matched=np.zeros(nv, np.int64))
    truncate = mutant == "bf16_truncate"
    lerp_how = ("two_products",) if mutant == "lerp_two_products" else ("fused", "unfused")
    for s in range(len(fa.tables)):
        rows = np.nonzero(seg == s)[0]
        if rows.size == 0:
            continue
        lt = fa.levels[s]
        c = coords[rows]
        vec = fa.vectors[s]
        # vector taps of every axis for both lerp forms: [form][axis] -> [n_s, 32]
        vl = {}
        for how in lerp_how:
            vl[how] = []
            for a in range(4):
                i0, i1, fr = (q[rows] for q in taps[a])
                vl[how].append(lerp(vec[a][i0], vec[a][i1], fr[:, None], how))
        for l in range(N_LEVELS):
            scale = lt.scale[l]
            if mutant == "scale_ulp_up" and l == MUTANT_SCALE_LEVEL:
                scale = np.nextafter(scale, F32(np.inf))
            cells = [to_cell(scale, c[:, a], fused=mutant != "to_cell_unfused") for a in range(4)]
            tab = [t_[int(lt.offset[l]):int(lt.offset[l]) + int(lt.size[l])] for t_ in fa.tables[s]]
            e = []
            for k in range(4):
                ax = GRID_AXES[k]
                ek = gather_level(tab[k], bool(lt.hashed[l]), int(lt.res[l]), int(lt.size[l]), cells[ax[0]], cells[ax[1]],
                                  cells[ax[2]], reverse=mutant == "corners_reversed")
                e.append(ek)
                egrid[4 * l + k, rows] = pack_bf16x2(bf16_bits(ek[:, 0], truncate), bf16_bits(ek[:, 1], truncate))
            # every contraction variant of the composition: [V, n_s, 2] bf16 bits
            bits = np.empty((nv, rows.size, 2), np.uint16)
            for vi, var in enumerate(VARIANTS):
                how = lerp_how[0] if len(lerp_how) == 1 else var[0]
                v = [vl[how][VECTOR_OF_TERM[k]][:, 2 * l:2 * l + 2] for k in range(4)]
                bits[vi] = bf16_bits(compose(e, v, var), truncate)
            feat[rows, 2 * l:2 * l + 2] = bits[0]
            amb_l = (bits != bits[0]).any(axis=0)
            amb[rows, 2 * l:2 * l + 2] = amb_l
            if chk is not None:
                got = feat_gpu[rows, 2 * l:2 * l + 2]
                hit = bits == got[None]
                chk["matched"] += hit.reshape(nv, -1).sum(axis=1)
                bad = ~hit.any(axis=0)
                chk["outputs"] += got.size
                chk["mismatch"] += int(bad.sum())
                chk["ambiguous"] += int(amb_l.sum())
                chk["mismatch_rows"].update(rows[bad.any(axis=1)].tolist())
    if chk is not None:
        chk["matched"] = {variant_name(v): int(m) for v, m in zip(VARIANTS, chk["matched"])}
    return Encoding(seg, egrid, feat, amb, chk)


def _step_ulps(x: np.ndarray, k: int) -> np.ndarray:
    """x moved by k fp32 ulps (x > 0)."""
    return (x.view(np.int32) + np.int32(k)).view(F32)


def level_edges(lt: LevelTable, rng: np.random.Generator, per_level: int = 8) -> np.ndarray:
    """Normalised coordinates in [0.25, 1] (so that x - 0.5 is exact and a position p = x - 0.5 loads back as x) whose
    fused scale_l * x + 0.5 is an integer for some level l -- exactly, or rounded onto it from either side -- together
    with their fp32 neighbours on both sides."""
    out = []
    for l in range(N_LEVELS):
        s = lt.scale[l]
        lo, hi = int(np.ceil(0.25 * float(s) + 0.5)) + 1, int(np.floor(float(s) + 0.5)) - 1
        ns = rng.integers(lo, hi + 1, per_level) if hi >= lo else np.zeros(0, np.int64)
        for n in ns:
            x0 = np.array([(n - 0.5) / float(s)], F32)
            cand = np.concatenate([_step_ulps(x0, k) for k in range(-3, 4)])
            hit = cand[fma32(s, cand, F32(0.5)) == F32(n)]
            for x in hit:
                out += [_step_ulps(np.array([x], F32), k)[0] for k in (-1, 0, 1)]
    e = np.unique(np.array(out, F32))
    return e[(e >= 0.25) & (e <= 1.0)]


def special_coordinates() -> np.ndarray:
    """x = 0, the smallest positive x a position can load as (x = p + 0.5 is a multiple of 2^-25 below 0.5, so the
    smallest fp32 subnormal itself cannot be reached as a coordinate), nextafter(1, 0) and 1 (every dense level at its
    largest cell, the single-subtraction wrap), the row-tap clamps at both ends, and the tap rows' own boundaries."""
    vals = [0.0, 2.0 ** -25, float(np.nextafter(F32(1), F32(0))), 1.0, 0.5, 1.0 / 4096, 0.5 / 2048, 1.0 - 1.0 / 4096,
            (2047 + 0.5) / 2048, 3.5 / 2048]
    return np.array(vals, F32)


def edge_positions(lts: Sequence[LevelTable], n: int, rng: np.random.Generator, outside: float = 0.15) -> np.ndarray:
    """n positions (fp32 [n, 3], world units: x - 0.5) whose coordinates are drawn from every level's integer-landing
    set, the special coordinates and (share `outside`) uniform values in [-4, 4] beyond the unit cube on both sides
    (the cold modulo and negative cells through (uint32)(int)).  Positions that reach p = +-(smallest subnormal) are
    included as well."""
    pool = np.concatenate([level_edges(lt, rng) for lt in lts] + [special_coordinates()])
    x = pool[rng.integers(0, pool.size, (n, 3))]
    far = rng.random((n, 3)) < outside
    out = rng.uniform(-4.0, 4.0, (n, 3)).astype(F32)
    out = np.where(np.abs(out) < 1.5, np.sign(out) * (1.5 + np.abs(out)), out).astype(F32)   # clearly outside [0, 1]
    x = np.where(far, out, x).astype(F32)
    p = fsub(x, F32(0.5))
    tiny = np.float32(np.finfo(F32).smallest_subnormal)
    p[: min(n, 2)] = np.array([[tiny, -tiny, 0.0], [-tiny, tiny, -0.5]], F32)[: min(n, 2)]
    return p


def egrid_mismatch(enc: Encoding, egrid_gpu: np.ndarray) -> Dict[str, int]:
    """Per-grid features of every row with a segment, bit for bit: count of differing u32 words and of rows."""
    rows = enc.seg >= 0
    g = np.asarray(egrid_gpu).view(np.uint32).reshape(4 * N_LEVELS, -1)[:, rows]
    bad = g != enc.egrid[:, rows]
    return dict(words=int(bad.sum()), rows=int(bad.any(axis=0).sum()), checked=int(bad.size))
