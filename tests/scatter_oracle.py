"""The table / vector gradient scatter of the field backward (hrf_field_backward_tables: csrc/scatter_pairs.cuh walked by
scatter_v6.cu and scatter_v5.cu) restated in numpy as a float64 sum, with an error bound per gradient entry derived
from the kernels' operation order.

TEST INFRASTRUCTURE ONLY.  The scatter is the adjoint of the encode, so every index and fp32 weight comes from the
encode reference (tests/encode_oracle.py: to_cell, corner_index, the weight product order (w_a * w_b) * w_c of
gather_level, row_tap), which is checked bit for bit against the kernels.  The inputs are the scatter's own: the
workspace's normalised (x, y, z, t), segment byte and d(features), plus the saved per-grid features (egrid) or the bf16
shadow tables for the re-gather.  A sample contributes iff it is below the live count and its segment byte is not 255.

Exact value of one entry (float64, `Reference`):
  table entry j of (segment, grid k, level l), feature f:   S = sum over samples and corners c with index j of
      w_c * v * dO,  v = v0 + frac * (v1 - v0)  (the fp32 vector rows of the grid's vector axis and row_tap's fp32 frac);
  vector row r of (segment, axis a, feature 2l + f):        S = sum over samples and both taps of  e * dO * tw,
      tw = 1 - frac for row i0 and frac for row i1 (both taps land on the same row at the clamps); e is the saved bf16
      value with egrid, and the exact blend sum_c w_c * b_c of the bf16 table values when the scatter re-gathers.

Bound.  u = 2^-24, gamma_k = k u / (1 - k u).  Each term is one LEAF of the fp32 sum the kernel forms; with |leaf error|
<= err_i and |computed leaf| <= mag_i, and m the number of leaves that can be nonzero,
      |kernel - S| <= sum_i err_i + gamma_{m-1} * sum_i mag_i + m * 2^-148,
because the kernel adds the leaves (and exact zeros, which are exact) in some binary tree: the per-slot run
`accx = __fmaf_rn(w, g, accx)` (scatter_pairs.cuh:223, the product inside the fma is exact), the REDs of flushed runs in
any order (:145, :205, :249, and the cold path's :86), the vector runs `va = __fmaf_rn(x, tw, va)` (:244) and the
butterfly of warp_combine_red2 (field_common.cuh:481-485, which adds zeros for the lanes of other rows).  Any tree over
m nonzero leaves rounds at most m - 1 times on any path.  The last term covers underflow (a subnormal result is off by at
most 2^-150 per rounding).  A buffer that holds B != 0 before the launch is one more leaf of magnitude |B|.

Table leaf  w * g,  g = fl(v^ * dO):
  * v^: the lerp `tv0.x + tp.frac * (tv1.x - tv0.x)` (:219) is left to nvcc's contraction: unfused it rounds three
    times, fused twice, so |v^ - v| <= Ev = u |v| + gamma_2 (1 + u) |frac (v1 - v0)| either way;
  * g = fl(v^ dO) (:220): |g - v dO| <= Eg = |dO| Ev + u |dO| (|v| + Ev);
  * the hot path's leaf is the exact product w * g inside the fma (:223); the cold path rounds fl(w * g) first (:86):
    err = |w| Eg + u |w| (|v dO| + Eg),  mag = (1 + u) |w| (|v dO| + Eg).
Vector leaf  x * tw,  x = fl(e^ * dO):
  * e^: egrid: the saved bf16 value, exact.  Re-gather: two 4-fma chains (:232-233) and the pair's shuffle add (:238),
    or the cold path's 8-fma chain (:81-84): |e^ - e| <= Ee = gamma_8 sum_c |w_c b_c|;
  * x = fl(e^ dO) (:244 / :87), tw = fl(1 - frac) (:243 / :88; frac itself is exact), and the cold path's product
    fl(x * tw) (:88-89): three roundings, so err = |dO tw| (Ee + gamma_3 (|e| + Ee)),  mag = (1 + gamma_3) |dO tw| (|e| + Ee).
Where m is 1 this is a few ulps of the one term.

MUTANTS are deliberately wrong references, each a plausible kernel bug; the tests show that each exceeds twice the
faithful bound on some entry of the GPU test's inputs.  The walk-structure mutants need the kernel's chunking, which
`walk` restates: samples [8c, 8c + 8) walked by one lane pair (lane p owns the corners whose first-axis vertex has
parity p, and row i_p), a slot flushed when either lane's entry changes, a new segment flushing everything, and
128-sample warps.  The plain reference does not use it; `walk_sum` adds the terms run by run and must agree with it.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

import encode_oracle as E
from encode_oracle import F32, F64, GRID_AXES, N_LEVELS, VECTOR_OF_TERM

U = 2.0 ** -24
TINY = 2.0 ** -148
CHUNK, WARP_SAMPLES = 8, 128
MUTANTS = ("to_cell_unfused", "scale_ulp_up", "parity_weight_swap", "chunk_tail_unflushed", "segment_change_misrouted",
           "cold_as_hot", "vector_taps_swapped", "time_rows_keyed_by_row", "regather_one_lane", "past_live_scattered")
WALK_MUTANTS = ("chunk_tail_unflushed", "segment_change_misrouted", "time_rows_keyed_by_row")


def gamma(k):
    k = np.maximum(np.asarray(k, F64), 0.0)
    return k * U / (1.0 - k * U)


@dataclass
class ScatterInputs:
    """What the scatter reads: pos4 f32 [n, 4] (x, y, z, t normalised), seg8 u8 [n] (255: no segment), dfeat f32
    [16, n, 2] (level-major d(features)), the live count, and egrid u32 [64, n] (bf16x2 of e_k of sample i at row
    4 l + k) or None for the re-gather of the bf16 tables."""
    pos4: np.ndarray
    seg8: np.ndarray
    dfeat: np.ndarray
    live: int
    egrid: Optional[np.ndarray] = None

    @property
    def n(self) -> int:
        return int(self.pos4.shape[0])


# ---------------------------------------------------------------------------------------------------- per-level terms
@dataclass
class LevelTerms:
    """The terms of one (grid k, level l) over the counted samples `rows`: table entry (level-local; for "cold_as_hot"
    a grid-global index in `gidx`) [T, 8 corners], and the leaves' value / err / mag / nonzero [T, 8, 2]; vector rows
    [T, 2 taps] and their leaves [T, 2, 2]."""
    rows: np.ndarray
    seg: np.ndarray
    cold: np.ndarray
    cells: tuple
    idx: np.ndarray
    t_val: np.ndarray
    t_err: np.ndarray
    t_mag: np.ndarray
    t_nz: np.ndarray
    vrow: np.ndarray
    v_val: np.ndarray
    v_err: np.ndarray
    v_mag: np.ndarray
    v_nz: np.ndarray
    gidx: Optional[np.ndarray] = None
    t_leaf: Optional[np.ndarray] = None      # one legal fp32 evaluation of each leaf (the kernel's roundings)
    v_leaf: Optional[np.ndarray] = None


def counted(inp: ScatterInputs, n_segments: int, mutant: Optional[str] = None) -> np.ndarray:
    seg = inp.seg8.astype(np.int64)
    ok = (seg != 255) & (seg < n_segments)
    if mutant != "past_live_scattered":
        ok &= np.arange(inp.n) < inp.live
    return ok


def corner_of_slot(p, q, ga, gb, gc):
    """The corner (bit d: +1 along dimension d) that lane p's parity slot q holds in the cell (ga, gb, gc)."""
    dx = (np.uint32(p) ^ (ga & np.uint32(1))).astype(np.int64)
    dy = (np.uint32(q & 1) ^ (gb & np.uint32(1))).astype(np.int64)
    dz = (np.uint32(q >> 1) ^ (gc & np.uint32(1))).astype(np.int64)
    return dx | (dy << 1) | (dz << 2)


def level_terms(fa: E.FieldArrays, inp: ScatterInputs, k: int, l: int, mutant: Optional[str] = None,
                lerp: Optional[str] = None) -> LevelTerms:
    """`lerp` ("fused" | "unfused"): also evaluate every leaf in fp32 (t_leaf / v_leaf) with that contraction of the
    vector lerp."""
    assert mutant is None or mutant in MUTANTS, mutant
    ok = counted(inp, len(fa.tables), mutant)
    rows = np.nonzero(ok)[0]
    seg = inp.seg8[rows].astype(np.int64)
    c = inp.pos4[rows]
    lt0 = fa.levels[0]
    scale = lt0.scale[l]
    if mutant == "scale_ulp_up" and l == E.MUTANT_SCALE_LEVEL:
        scale = np.nextafter(scale, F32(np.inf))
    res = int(lt0.res[l])
    ax = GRID_AXES[k]
    cells = [E.to_cell(scale, c[:, a], fused=mutant != "to_cell_unfused") for a in ax]
    (ga, fa_), (gb, fb), (gc, fc) = cells
    T = rows.size
    one = F32(1)
    wd = ((E.fsub(one, fa_), fa_), (E.fsub(one, fb), fb), (E.fsub(one, fc), fc))
    swap = (ga & np.uint32(1)) == 1 if mutant == "parity_weight_swap" else np.zeros(T, bool)
    idx = np.zeros((T, 8), np.int64)
    gidx = np.zeros((T, 8), np.int64) if mutant == "cold_as_hot" else None
    w = np.zeros((T, 8), F32)
    bvals = np.zeros((T, 8, 2), F64)
    cold = np.zeros(T, bool)
    for s in range(len(fa.tables)):
        sel = np.nonzero(seg == s)[0]
        if sel.size == 0:
            continue
        lt = fa.levels[s]
        hashed, size, off = bool(lt.hashed[l]), int(lt.size[l]), int(lt.offset[l])
        a_, b_, c_ = ga[sel], gb[sel], gc[sel]
        cold_s = np.zeros(sel.size, bool) if hashed else ((a_ >= res) | (b_ >= res) | (c_ >= res))
        cold[sel] = cold_s
        sw = swap[sel] & ~cold_s
        for q in range(8):
            ix = E.corner_index(q, hashed, res, size, a_, b_, c_).astype(np.int64)
            idx[sel, q] = ix
            if gidx is not None:
                gidx[sel, q] = off + ix
                if not hashed:    # the hot path's single subtraction on a cold sample: lands outside the level
                    one_u = np.uint32(1)
                    t = ((a_ + one_u if q & 1 else a_) + (b_ + one_u if q & 2 else b_) * np.uint32(res)
                         + (c_ + one_u if q & 4 else c_) * np.uint32(res * res)).astype(np.int64)
                    t = np.where(t >= size, t - size, t)
                    gidx[sel[cold_s], q] = ((off + t) % lt.n_entries)[cold_s]
            wx = np.where(sw, wd[0][1 - (q & 1)][sel], wd[0][q & 1][sel])
            w[sel, q] = E.fmul(E.fmul(wx, wd[1][(q >> 1) & 1][sel]), wd[2][(q >> 2) & 1][sel])
            tab = fa.tables[s][k]
            bvals[sel, q] = E.bf16_to_f32(tab[off + ix]).astype(F64)
    # the vector axis of grid k and its lerp
    va = VECTOR_OF_TERM[k]
    i0, i1, frac = E.row_tap(c[:, va], fa.vec_res)
    v0 = np.zeros((T, 2), F64)
    v1 = np.zeros((T, 2), F64)
    for s in range(len(fa.tables)):
        sel = seg == s
        v0[sel] = fa.vectors[s][va][i0[sel], 2 * l:2 * l + 2]
        v1[sel] = fa.vectors[s][va][i1[sel], 2 * l:2 * l + 2]
    fr = frac.astype(F64)[:, None]
    dv = np.abs(fr * (v1 - v0))
    v = v0 + fr * (v1 - v0)
    dO = inp.dfeat[l, rows].astype(F64)
    Ev = U * np.abs(v) + gamma(2) * (1 + U) * dv
    Eg = np.abs(dO) * Ev + U * np.abs(dO) * (np.abs(v) + Ev)
    wf = w.astype(F64)[:, :, None]
    vd = np.abs(v * dO)[:, None, :]
    t_val = wf * (v * dO)[:, None, :]
    t_err = np.abs(wf) * Eg[:, None, :] + U * np.abs(wf) * (vd + Eg[:, None, :])
    t_mag = (1 + U) * np.abs(wf) * (vd + Eg[:, None, :])
    t_nz = (wf != 0) & (dO != 0)[:, None, :] & ((v0 != 0) | (v1 != 0))[:, None, :]
    # the feature e each tap multiplies
    wb = wf * bvals
    if inp.egrid is None:
        if mutant == "regather_one_lane":   # lane p blends only the corners whose first-axis vertex has parity p
            e = np.zeros((T, 2, 2), F64)
            for p in range(2):
                for q in range(8):
                    mine = ((ga.astype(np.int64) + (q & 1)) & 1) == p
                    e[:, p] += np.where((mine | cold)[:, None], wb[:, q], 0.0)
        else:
            e = np.repeat(wb.sum(axis=1)[:, None, :], 2, axis=1)
        Ee = np.repeat((gamma(8) * np.abs(wb).sum(axis=1))[:, None, :], 2, axis=1)
        e_nz = np.repeat((wb != 0).any(axis=1)[:, None, :], 2, axis=1)
    else:
        word = inp.egrid[4 * l + k, rows]
        ef = np.stack((E.bf16_to_f32((word & 0xFFFF).astype(np.uint16)), E.bf16_to_f32((word >> 16).astype(np.uint16))),
                      axis=1).astype(F64)
        e = np.repeat(ef[:, None, :], 2, axis=1)
        Ee = np.zeros_like(e)
        e_nz = e != 0
    tw = np.stack((1.0 - frac.astype(F64), frac.astype(F64)), axis=1)      # [T, 2 taps]
    if mutant == "vector_taps_swapped":
        tw = tw[:, ::-1]
    dt = np.abs(dO[:, None, :] * tw[:, :, None])
    v_val = e * dO[:, None, :] * tw[:, :, None]
    v_err = dt * (Ee + gamma(3) * (np.abs(e) + Ee))
    v_mag = (1 + gamma(3)) * dt * (np.abs(e) + Ee)
    v_nz = e_nz & (dO != 0)[:, None, :] & (tw != 0)[:, :, None]
    vrow = np.stack((i0, i1), axis=1).astype(np.int64)
    if lerp is None:
        return LevelTerms(rows, seg, cold, (ga, gb, gc), idx, t_val, t_err, t_mag, t_nz, vrow, v_val, v_err, v_mag, v_nz,
                          gidx)
    # fp32 leaves: g = fl(lerp * dO), leaf w * g; x = fl(e^ dO), leaf x * fl(1 - frac) (e^ of the 8-fma chain)
    dO32 = inp.dfeat[l, rows]
    g32 = E.fmul(E.lerp(v0.astype(F32), v1.astype(F32), frac[:, None], lerp), dO32)
    t_leaf = wf * g32.astype(F64)[:, None, :]
    if inp.egrid is None:
        e32 = np.zeros((T, 2), F32)
        for q in range(8):
            e32 = E.fma32(w[:, q][:, None], bvals[:, q].astype(F32), e32)
    else:
        e32 = ef.astype(F32)
    x32 = E.fmul(e32, dO32).astype(F64)
    tw32 = np.stack((E.fsub(F32(1), frac), frac), axis=1).astype(F64)
    if mutant == "vector_taps_swapped":
        tw32 = tw32[:, ::-1]
    v_leaf = x32[:, None, :] * tw32[:, :, None]
    return LevelTerms(rows, seg, cold, (ga, gb, gc), idx, t_val, t_err, t_mag, t_nz, vrow, v_val, v_err, v_mag, v_nz,
                      gidx, t_leaf, v_leaf)


# ---------------------------------------------------------------------------------------------------- accumulation
@dataclass
class Sums:
    """Per entry: S (float64), sum of leaf errors, sum of leaf magnitudes, m -- arrays of one shape [..., 2]."""
    val: np.ndarray
    err: np.ndarray
    mag: np.ndarray
    m: np.ndarray

    @staticmethod
    def zeros(shape):
        return Sums(np.zeros(shape, F64), np.zeros(shape, F64), np.zeros(shape, F64), np.zeros(shape, np.int64))

    def add(self, flat_index, val, err, mag, nz):
        """Scatter-add leaves (arrays [L, 2]) at rows `flat_index` [L] of the [entries, 2] view."""
        n = self.val.reshape(-1, 2).shape[0]
        for f in range(2):
            for arr, src in ((self.val, val), (self.err, err), (self.mag, mag), (self.m, nz)):
                a = arr.reshape(-1, 2)
                a[:, f] += np.bincount(flat_index, weights=src[:, f].astype(F64), minlength=n)[:n].astype(a.dtype)

    def bound(self, base=None) -> np.ndarray:
        m = self.m.astype(F64)
        mag = self.mag
        if base is not None:
            b = np.abs(np.asarray(base, F64).reshape(self.val.shape))
            m = m + (b != 0)
            mag = mag + b
        return self.err + gamma(m - 1) * mag + m * TINY


@dataclass
class Reference:
    """tables[s][k]: Sums [n_entries, 2] of grid k of segment s; vectors[s]: Sums [4, VR, 32]."""
    tables: List[List[Sums]]
    vectors: List[Sums]


def _vec_flat(vr: int, axis: int, rows, l: int):
    return (axis * vr + rows) * (N_LEVELS) + l          # row of the [4 * VR * 16, 2] view of [4, VR, 32]


def reference(fa: E.FieldArrays, inp: ScatterInputs, mutant: Optional[str] = None, grids=range(4),
              levels=range(N_LEVELS)) -> Reference:
    """The float64 gradients of every table and vector entry (the plain sum; the walk-structure mutants go through
    `walk`)."""
    ns, vr = len(fa.tables), fa.vec_res
    ref = Reference([[Sums.zeros((fa.levels[s].n_entries, 2)) for _ in range(4)] for s in range(ns)],
                    [Sums.zeros((4, vr, 32)) for _ in range(ns)])
    for k in grids:
        for l in levels:
            lt = level_terms(fa, inp, k, l, None if mutant in WALK_MUTANTS else mutant)
            if mutant in WALK_MUTANTS:
                _walk_route(fa, inp, lt, k, l, mutant, ref)
                continue
            for s in range(ns):
                sel = lt.seg == s
                if not sel.any():
                    continue
                gi = (lt.gidx[sel] if lt.gidx is not None else lt.idx[sel] + int(fa.levels[s].offset[l])).reshape(-1)
                ref.tables[s][k].add(gi, *(a[sel].reshape(-1, 2) for a in (lt.t_val, lt.t_err, lt.t_mag, lt.t_nz)))
                vi = _vec_flat(vr, VECTOR_OF_TERM[k], lt.vrow[sel], l).reshape(-1)
                ref.vectors[s].add(vi, *(a[sel].reshape(-1, 2) for a in (lt.v_val, lt.v_err, lt.v_mag, lt.v_nz)))
    return ref


def reference_level(fa: E.FieldArrays, inp: ScatterInputs, k: int, l: int, vectors: List[Sums]) -> List[Sums]:
    """The table gradients of one (grid, level) per segment, level-local [size, 2] (large models); the level's vector
    leaves are added into `vectors`."""
    lt = level_terms(fa, inp, k, l)
    out = []
    for s in range(len(fa.tables)):
        sums = Sums.zeros((int(fa.levels[s].size[l]), 2))
        sel = lt.seg == s
        if sel.any():
            sums.add(lt.idx[sel].reshape(-1), *(a[sel].reshape(-1, 2) for a in (lt.t_val, lt.t_err, lt.t_mag, lt.t_nz)))
            vi = _vec_flat(fa.vec_res, VECTOR_OF_TERM[k], lt.vrow[sel], l).reshape(-1)
            vectors[s].add(vi, *(a[sel].reshape(-1, 2) for a in (lt.v_val, lt.v_err, lt.v_mag, lt.v_nz)))
        out.append(sums)
    return out


# ---------------------------------------------------------------------------------------------------- the walk
@dataclass
class Walk:
    """The runs of one (grid, level).  Table: run of lane p's slot q holding term (sample j, corner c) in `t_run`
    [T, 8] (-1: a cold term, RED on its own); per run its segment, entry, how it ended (0 flush, 1 new segment, 2 end
    of the chunk) and the segment that ended it.  Vector: `v_run` [T, 2 taps] likewise, with the row and, for runs that
    end with the chunk, the lane (0..31) and warp that hold them."""
    t_run: np.ndarray
    r_seg: np.ndarray
    r_entry: np.ndarray
    r_end: np.ndarray
    r_next: np.ndarray
    v_run: np.ndarray
    q_seg: np.ndarray
    q_row: np.ndarray
    q_end: np.ndarray
    q_next: np.ndarray
    q_lane: np.ndarray
    q_warp: np.ndarray


def walk(inp: ScatterInputs, lt: LevelTerms) -> Walk:
    """scatter_level_pairs' run structure over every 8-sample chunk (vectorised over chunks, one step per position)."""
    n = inp.n
    nch = -(-n // CHUNK)
    T = lt.rows.size
    pos_of = np.full(nch * CHUNK, -1, np.int64)          # sample -> term row (-1: not counted)
    pos_of[lt.rows] = np.arange(T)
    ga, gb, gc = lt.cells
    t_run = np.full((T, 8), -1, np.int64)
    v_run = np.full((T, 2), -1, np.int64)
    runs = dict(seg=[], entry=[], end=[], nxt=[])
    vruns = dict(seg=[], row=[], end=[], nxt=[], lane=[], warp=[])
    cur = np.full(nch, -1, np.int64)
    rid = np.full((nch, 2, 4), -1, np.int64)
    ridx = np.zeros((nch, 2, 4), np.int64)
    vid = np.full((nch, 2), -1, np.int64)
    vto = np.zeros((nch, 2), np.int64)
    nrun = [0, 0]
    ch_all = np.arange(nch)

    def new_runs(mask3, segs, entries):      # mask [nch, 2, 4]
        cnt = int(mask3.sum())
        ids = nrun[0] + np.arange(cnt)
        nrun[0] += cnt
        rid[mask3] = ids
        runs["seg"].append(np.broadcast_to(segs[:, None, None], mask3.shape)[mask3])
        runs["entry"].append(entries[mask3])
        runs["end"].append(np.full(cnt, -1))
        runs["nxt"].append(np.full(cnt, -1))

    def new_vruns(mask2, segs, rows_):
        cnt = int(mask2.sum())
        ids = nrun[1] + np.arange(cnt)
        nrun[1] += cnt
        vid[mask2] = ids
        ch, p = np.nonzero(mask2)
        vruns["seg"].append(segs[ch])
        vruns["row"].append(rows_[mask2])
        vruns["end"].append(np.full(cnt, -1))
        vruns["nxt"].append(np.full(cnt, -1))
        vruns["lane"].append((ch % 16) * 2 + p)
        vruns["warp"].append(ch // 16)

    ends, vends = [], []        # (ids, reason, next segment)

    # slot entries of every term row: [T, 2 lanes, 4 slots]
    slot_c = np.stack([np.stack([corner_of_slot(p, q, ga, gb, gc) for q in range(4)], axis=1) for p in range(2)], axis=1)
    slot_e = np.take_along_axis(lt.idx[:, None, :].repeat(2, 1), slot_c, axis=2)
    for j in range(CHUNK):
        tr = pos_of[ch_all * CHUNK + j]
        ok = tr >= 0
        trs = np.where(ok, tr, 0)
        sg = np.where(ok, lt.seg[trs], -1)
        cold = ok & lt.cold[trs]
        hot = ok & ~cold
        nidx = np.where(hot[:, None, None], slot_e[trs], 0)
        trow = lt.vrow[trs]                                              # [nch, 2]
        segch = ok & (sg != cur)
        had = segch & (cur >= 0)
        m3 = np.broadcast_to(had[:, None, None], rid.shape)
        ends.append((rid[m3], 1, np.broadcast_to(sg[:, None, None], rid.shape)[m3]))
        m2 = np.broadcast_to(had[:, None], vid.shape)
        vends.append((vid[m2], 1, np.broadcast_to(sg[:, None], vid.shape)[m2]))
        ridx[segch] = nidx[segch]
        new_runs(np.broadcast_to(segch[:, None, None], rid.shape), sg, ridx)
        vto[segch] = trow[segch]
        new_vruns(np.broadcast_to(segch[:, None], vid.shape), sg, vto)
        cur = np.where(segch, sg, cur)
        changed = hot[:, None, None] & (nidx != ridx)
        flush = np.broadcast_to((changed[:, 0] | changed[:, 1])[:, None, :], rid.shape) & hot[:, None, None]
        ends.append((rid[flush], 0, np.full(int(flush.sum()), -1)))
        ridx[flush] = nidx[flush]
        new_runs(flush, cur, ridx)
        vch = hot[:, None] & (trow != vto)
        vends.append((vid[vch], 0, np.full(int(vch.sum()), -1)))
        vto[vch] = trow[vch]
        new_vruns(vch, cur, vto)
        h = np.nonzero(hot)[0]
        for p in range(2):
            for q in range(4):
                t_run[tr[h], slot_c[tr[h], p, q]] = rid[h, p, q]
            v_run[tr[h], p] = vid[h, p]
    live_ch = cur >= 0
    m3 = np.broadcast_to(live_ch[:, None, None], rid.shape)
    ends.append((rid[m3], 2, np.full(int(m3.sum()), -1)))
    m2 = np.broadcast_to(live_ch[:, None], vid.shape)
    vends.append((vid[m2], 2, np.full(int(m2.sum()), -1)))
    cat = lambda d, key: np.concatenate(d[key]) if d[key] else np.zeros(0, np.int64)
    r_end, r_next = cat(runs, "end"), cat(runs, "nxt")
    for ids, why, nx in ends:
        r_end[ids], r_next[ids] = why, nx
    q_end, q_next = cat(vruns, "end"), cat(vruns, "nxt")
    for ids, why, nx in vends:
        q_end[ids], q_next[ids] = why, nx
    # a cold term is its own RED; its entry checks the table-run bookkeeping too
    return Walk(t_run, cat(runs, "seg"), cat(runs, "entry"), r_end, r_next, v_run, cat(vruns, "seg"), cat(vruns, "row"),
                q_end, q_next, cat(vruns, "lane"), cat(vruns, "warp"))


def _walk_route(fa, inp, lt: LevelTerms, k: int, l: int, mutant: Optional[str], ref: Reference) -> None:
    """Add the (grid, level)'s leaves to `ref` the way the walk routes them: each hot table leaf to its run's segment and
    entry (not the leaf's own index), each vector leaf to its run's row; `mutant` re-routes or drops runs."""
    wk = walk(inp, lt)
    vr, axis = fa.vec_res, VECTOR_OF_TERM[k]
    # table leaves
    hot = wk.t_run >= 0
    r = np.where(hot, wk.t_run, 0)
    seg = np.where(hot, wk.r_seg[r], lt.seg[:, None])
    entry = np.where(hot, wk.r_entry[r], lt.idx)
    keep = np.ones_like(hot)
    if mutant == "chunk_tail_unflushed":
        keep = ~(hot & (wk.r_end[r] == 2))
    if mutant == "segment_change_misrouted":
        seg = np.where(hot & (wk.r_end[r] == 1), wk.r_next[r], seg)
    for s in range(len(fa.tables)):
        sel = keep & (seg == s)
        gi = (entry[sel] + int(fa.levels[s].offset[l])) % fa.levels[s].n_entries
        ref.tables[s][k].add(gi, *(a[sel] for a in (lt.t_val, lt.t_err, lt.t_mag, lt.t_nz)))
    # vector leaves: hot ones through their runs, cold ones on their own
    hv = wk.v_run >= 0
    q = np.where(hv, wk.v_run, 0)
    vseg = np.where(hv, wk.q_seg[q], lt.seg[:, None])
    vrow = np.where(hv, wk.q_row[q], lt.vrow)
    vkeep = np.ones_like(hv)
    if mutant == "chunk_tail_unflushed" and axis != 3:
        vkeep = ~(hv & (wk.q_end[q] == 2))
    if mutant == "segment_change_misrouted":
        vseg = np.where(hv & (wk.q_end[q] == 1), wk.q_next[q], vseg)
    if mutant == "time_rows_keyed_by_row" and axis == 3:
        # warp_combine_red2 keyed by the row alone: every end-of-chunk run of a warp with that row goes to the segment
        # of the lowest lane holding the row
        e = np.nonzero(wk.q_end == 2)[0]
        order = np.lexsort((wk.q_lane[e], wk.q_row[e], wk.q_warp[e]))
        e = e[order]
        key = wk.q_warp[e] * (1 << 40) + wk.q_row[e]
        first = np.r_[True, key[1:] != key[:-1]]
        leader_seg = wk.q_seg[e][np.maximum.accumulate(np.where(first, np.arange(e.size), 0))]
        new_seg = wk.q_seg.copy()
        new_seg[e] = leader_seg
        vseg = np.where(hv & (wk.q_end[q] == 2), new_seg[q], vseg)
    for s in range(len(fa.tables)):
        sel = vkeep & (vseg == s)
        vi = _vec_flat(vr, axis, vrow[sel], l)
        ref.vectors[s].add(vi, *(a[sel] for a in (lt.v_val, lt.v_err, lt.v_mag, lt.v_nz)))


def walk_sum(fa: E.FieldArrays, inp: ScatterInputs, grids=range(4), levels=range(N_LEVELS)) -> Reference:
    """The unmutated gradients routed through `walk`: every hot leaf lands where its run's slot points."""
    ns, vr = len(fa.tables), fa.vec_res
    ref = Reference([[Sums.zeros((fa.levels[s].n_entries, 2)) for _ in range(4)] for s in range(ns)],
                    [Sums.zeros((4, vr, 32)) for _ in range(ns)])
    for k in grids:
        for l in levels:
            _walk_route(fa, inp, level_terms(fa, inp, k, l), k, l, None, ref)
    return ref


# ---------------------------------------------------------------------------------------------------- comparison
def ratio(got, ref_val, bound) -> np.ndarray:
    """|got - ref| / bound per entry; an error where the bound is 0 is infinite, a NaN anywhere is infinite."""
    got = np.asarray(got, F64)
    err = np.abs(got - ref_val)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return np.where(np.isnan(r) | np.isnan(got), np.inf, r)
