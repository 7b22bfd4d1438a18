"""Seeded inputs of the gradient-scatter tests (tests/test_scatter_oracle_gpu.py), built in numpy so that the CPU tests
can rebuild exactly what the GPU test feeds the kernels (tests/test_scatter_oracle_cpu.py runs the mutants on them).

A model is a FieldArrays of bf16-representable tables and fp32 vectors drawn from a seed (`model`); an input set is a
ScatterInputs: the workspace's (x, y, z, t), segment byte and d(features), and the live count.
  B "edges":      runs in one cell of 1-20 samples across the 8 / 128 / 1024 borders, single-cell steps along the axes
                  and the face and body diagonals, A,B,A,B alternation, frac exactly 0, far-outside samples inside hot
                  runs, t at 0, 1 and the row-tap clamps;
  C "collisions": cells where two corners share a table entry at a hashed level, in one lane and across the pair;
  D "segments":   three segments changing at every chunk position, on chunk / warp / CTA borders, warps spanning two
                  and three segments, samples without a segment (255) inside runs;
  E "live":       one set cut at live counts 0, 1, 1023, 1025 and the capacity, with poisoned rows past the count.
The small model has segments of 6 frames (log2T 15, the smallest tables).
"""
from __future__ import annotations

import numpy as np

import encode_oracle as E
from encode_oracle import F32, N_LEVELS
from scatter_oracle import ScatterInputs

SMALL = (6, 6, 6)
FIRST_FRAME = 15
VEC_RES = 2048          # Decomposition4D's vectors_finest_resolution
LIVE_COUNTS = (0, 1, 1023, 1025, None)     # None: the capacity


def frames_of(segs):
    return tuple(range(FIRST_FRAME, FIRST_FRAME + sum(segs)))


def model(segs=SMALL, seed=7) -> E.FieldArrays:
    """bf16-representable fp32 tables N(0, 0.5) (so the fp32 masters and the bf16 shadows hold the same values) and
    fp32 vectors N(0, 1), 5 % of each exactly zero."""
    rng = np.random.default_rng(seed)
    tabs, vecs = [], []
    for s in segs:
        n = E.level_table(E.segment_log2_hashmap_size(s)).n_entries
        gs = []
        for _ in range(4):
            x = (rng.standard_normal(2 * n, dtype=F32) * F32(0.5))
            x[rng.random(2 * n) < 0.05] = 0
            gs.append(E.bf16_bits(x).reshape(-1, 2))
        tabs.append(gs)
        v = rng.standard_normal((4, VEC_RES, 32), dtype=F32)
        v[rng.random(v.shape) < 0.05] = 0
        vecs.append(v)
    return E.FieldArrays(tabs, vecs, [E.segment_log2_hashmap_size(s) for s in segs], frames_of(segs), segs)


def fp32_tables(fa: E.FieldArrays):
    """The fp32 masters of the bf16 tables (flat, tcnn order), what the module holds."""
    return [[E.bf16_to_f32(t).reshape(-1) for t in ts] for ts in fa.tables]


def d_features(rng, n) -> np.ndarray:
    """[16, n, 2] d(features): mixed signs, per-sample scales 2^U(-20, 20), every 7th row zero, 3 % exact zeros."""
    d = rng.standard_normal((N_LEVELS, n, 2)) * 2.0 ** rng.uniform(-20, 20, (1, n, 1))
    d[:, ::7] = 0
    d[rng.random(d.shape) < 0.03] = 0
    return d.astype(F32)


def egrid_of(fa: E.FieldArrays, pos4, seg8) -> np.ndarray:
    """The saved per-grid features the training forward writes (bf16x2 of gather_level), for any (x, y, z, t)."""
    n = pos4.shape[0]
    eg = np.zeros((4 * N_LEVELS, n), np.uint32)
    for s in range(len(fa.tables)):
        rows = np.nonzero(seg8 == s)[0]
        if rows.size == 0:
            continue
        lt = fa.levels[s]
        c = pos4[rows]
        for l in range(N_LEVELS):
            cells = [E.to_cell(lt.scale[l], c[:, a]) for a in range(4)]
            for k in range(4):
                ax = E.GRID_AXES[k]
                tab = fa.tables[s][k][int(lt.offset[l]):int(lt.offset[l]) + int(lt.size[l])]
                e = E.gather_level(tab, bool(lt.hashed[l]), int(lt.res[l]), int(lt.size[l]), *(cells[a] for a in ax))
                eg[4 * l + k, rows] = E.pack_bf16x2(E.bf16_bits(e[:, 0]), E.bf16_bits(e[:, 1]))
    return eg


# ---------------------------------------------------------------------------------------------------- sequences
class _Seq:
    """Samples appended in order: rows (x, y, z, t) and segment bytes; `pad_to` fills with ray-like walks."""

    def __init__(self, rng, n_segments, t_pool):
        self.rng, self.ns, self.t_pool = rng, n_segments, t_pool
        self.pos, self.seg = [], []

    def __len__(self):
        return sum(p.shape[0] for p in self.pos)

    def add(self, xyz, t=None, seg=None):
        xyz = np.atleast_2d(np.asarray(xyz, F32))
        n = xyz.shape[0]
        t = np.full(n, self.rng.choice(self.t_pool) if t is None else t, F32) if np.ndim(t) == 0 else np.asarray(t, F32)
        s = np.full(n, self.rng.integers(0, self.ns) if seg is None else seg, np.uint8) if np.ndim(seg) == 0 else np.asarray(seg, np.uint8)
        self.pos.append(np.concatenate((xyz, t[:, None]), axis=1).astype(F32))
        self.seg.append(s)

    def ray(self, n, step=4e-4):
        o = self.rng.uniform(0.2, 0.8, 3)
        d = self.rng.standard_normal(3)
        d /= np.linalg.norm(d)
        self.add(o + np.arange(n)[:, None] * step * d)

    def pad_to(self, pos):
        while len(self) < pos:
            self.ray(min(int(self.rng.integers(5, 40)), pos - len(self)))

    def build(self, rng) -> ScatterInputs:
        pos4 = np.concatenate(self.pos)
        seg8 = np.concatenate(self.seg)
        return ScatterInputs(pos4, seg8, d_features(rng, pos4.shape[0]), pos4.shape[0])


def _t_pool(vr=VEC_RES):
    local = [k / 6 for k in range(6)]
    return np.array(local + [0.0, 1.0, 0.5 / vr, 1 - 0.5 / vr, 0.25 / vr, 1 - 0.25 / vr, 1.5 / vr], F32)


def _far(rng, n):
    out = rng.uniform(1.5, 4.0, (n, 3)) * np.where(rng.random((n, 3)) < 0.5, -1, 1)
    return (out + 0.5).astype(F32)


def set_edges(fa: E.FieldArrays, seed=101) -> ScatterInputs:
    rng = np.random.default_rng(seed)
    q = _Seq(rng, len(fa.tables), _t_pool(fa.vec_res))
    lt = fa.levels[0]
    pool = np.concatenate([E.level_edges(lt, rng)] + [E.special_coordinates()])
    pool = pool[(pool >= 0) & (pool <= 1)]

    def point():
        return pool[rng.integers(0, pool.size, 3)]

    # runs in one cell across the chunk, warp and CTA borders
    for border, runs in ((8, ((1, 0), (2, 1), (7, 3), (9, 8), (16, 8), (20, 13), (20, 1))),
                         (128, ((1, 0), (7, 3), (9, 8), (20, 13))), (1024, ((9, 8), (20, 13), (2, 1)))):
        for L_, off in runs:
            q.pad_to(border * ((len(q) + L_) // border + 1) - off)
            q.add(np.repeat(point()[None], L_, axis=0))
    # single-cell steps along the axes, face diagonals and body diagonals at a hashed and a dense level
    dirs = [d for d in np.ndindex(2, 2, 2) if any(d)]
    for lvl in (0, 3, 9, 15):
        w = 1.0 / float(lt.scale[lvl])
        for d in dirs:
            for sgn in (1, -1):
                x0 = rng.uniform(0.3, 0.7, 3)
                steps = np.arange(6)[:, None] * sgn * w * np.array(d)
                reps = rng.integers(1, 4, 6)
                q.add(np.repeat(x0 + steps, reps, axis=0))
    # A,B,A,B alternation
    for _ in range(6):
        a, b = point(), point()
        q.add(np.stack([a, b] * 6))
    # frac exactly 0 (level_edges land on integers) in runs; far-outside samples inside hot runs at every position
    for _ in range(10):
        q.add(np.repeat(point()[None], int(rng.integers(2, 10)), axis=0))
    for j in range(8):
        q.pad_to(8 * (len(q) // 8 + 1))
        x0 = rng.uniform(0.3, 0.7, 3)
        run = np.repeat(x0[None], 12, axis=0)
        run[j] = _far(rng, 1)[0]
        run[(j + 5) % 12] = _far(rng, 1)[0]
        q.add(run)
    # t at 0, 1 and the row-tap clamps, dense samples outside the grid on both sides
    for t in (0.0, 1.0, 0.25 / fa.vec_res, 1 - 0.25 / fa.vec_res, 1 - 0.5 / fa.vec_res):
        q.add(np.repeat(rng.uniform(0.2, 0.8, 3)[None], 3, axis=0), t=t)
    q.add(_far(rng, 60))
    q.pad_to(3 * 1024 + 77)
    return q.build(rng)


def _collision_cells(lt, l, same_lane, rng, want):
    """Up to `want` cells (g0, g1, g2) inside [0, res) whose corners c != c' share a hashed entry of level l (same_lane:
    corners with the same first-axis offset; otherwise corners of the two lanes of a pair)."""
    res = int(lt.res[l])
    out = []
    for _ in range(12):
        g = rng.integers(0, res - 1, (1 << 18, 3)).astype(np.uint32)
        idx = np.stack([E.corner_index(c, True, res, int(lt.size[l]), g[:, 0], g[:, 1], g[:, 2]) for c in range(8)], axis=1)
        hit = np.zeros(g.shape[0], bool)
        for a in range(8):
            for b in range(a + 1, 8):
                if ((a & 1) == (b & 1)) == same_lane:
                    hit |= idx[:, a] == idx[:, b]
        out += list(g[hit])
        if len(out) >= want:
            break
    return np.array(out[:want], np.uint32)


def set_collisions(fa: E.FieldArrays, seed=202) -> ScatterInputs:
    rng = np.random.default_rng(seed)
    q = _Seq(rng, len(fa.tables), _t_pool(fa.vec_res))
    lt = fa.levels[0]
    assert all(E.segment_log2_hashmap_size(s) == fa.log2T[0] for s in fa.segment_sizes)
    found = 0
    for l in (11, 12, 13, 14, 15):     # (coarser levels have too few cells for the hash to collide inside one)
        s = float(lt.scale[l])
        for same_lane in (True, False):
            cells = _collision_cells(lt, l, same_lane, rng, 12)
            for i, g in enumerate(cells):
                k = i % 4
                ax = E.GRID_AXES[k]
                f = rng.uniform(0.05, 0.95, 3)
                xyzt = rng.uniform(0.2, 0.8, 4)
                xyzt[list(ax)] = (g.astype(np.float64) + f - 0.5) / s
                xyzt = xyzt.astype(F32)
                got = [E.to_cell(lt.scale[l], xyzt[a:a + 1])[0][0] for a in ax]
                if list(got) != list(g):
                    continue
                found += 1
                reps = int(rng.integers(1, 6))
                q.add(np.repeat(xyzt[None, :3], reps, axis=0), t=np.full(reps, xyzt[3]))
                if i % 3 == 0:
                    q.ray(int(rng.integers(3, 12)))
    assert found >= 40, found
    q.pad_to(2 * 1024 + 333)
    return q.build(rng)


def set_segments(fa: E.FieldArrays, seed=303) -> ScatterInputs:
    rng = np.random.default_rng(seed)
    ns = len(fa.tables)
    assert ns >= 3
    pos, seg = [], []
    n = 5 * 1024 + 200
    # one slow walk: neighbouring samples share cells and time rows; t shared across segments (the same time rows)
    o = rng.uniform(0.25, 0.75, 3)
    d = rng.standard_normal(3)
    d /= np.linalg.norm(d)
    xyz = (o + np.arange(n)[:, None] * 1e-4 * d)
    xyz = np.where((xyz < 0.05) | (xyz > 0.95), 0.5, xyz)
    t = np.repeat(np.array([0.0, 1 / 6, 0.5, 0.5], F32), -(-n // 4))[:n]
    seg8 = np.zeros(n, np.uint8)
    cur = 0
    events = []
    for c in range(60):                          # changes at every position inside a chunk
        events.append(8 * (2 + 3 * c) + (c % 7) + 1)
    events += [8 * 200, 8 * 201, 128 * 3, 128 * 4, 1024, 2048, 3072]      # on chunk / warp / CTA borders
    events += [128 * 6 + 40, 128 * 6 + 90, 128 * 7 + 30, 128 * 7 + 50, 128 * 7 + 100]   # warps with 2 and 3 segments
    for e in sorted(set(events)):
        cur = (cur + 1 + int(rng.integers(0, ns - 1))) % ns
        seg8[e:] = cur
    holes = rng.choice(n, 200, replace=False)
    seg8[holes] = 255                            # no segment, inside runs
    seg8[4000:4012] = 255
    return ScatterInputs(np.concatenate((xyz, t[:, None]), axis=1).astype(F32), seg8, d_features(rng, n), n)


def set_live(fa: E.FieldArrays, live, seed=404) -> ScatterInputs:
    """A capacity of 2 CTAs + 309 samples (edges and rays), cut at `live` (None: the capacity); rows past it hold NaN
    d(features), in-cube positions and valid segment bytes."""
    base = set_edges(fa, seed)
    rng = np.random.default_rng(seed + 1)
    n = 2 * 1024 + 309
    pos4, seg8, df = base.pos4[:n].copy(), base.seg8[:n].copy(), base.dfeat[:, :n].copy()
    live = n if live is None else live
    df[:, live:] = np.nan
    pos4[live:, :3] = rng.uniform(0.3, 0.7, (n - live, 3)).astype(F32)
    seg8[live:] = rng.integers(0, len(fa.tables), n - live).astype(np.uint8)
    return ScatterInputs(pos4, seg8, df, live)


SMALL_SETS = ("edges", "collisions", "segments") + tuple(f"live{'cap' if lc is None else lc}" for lc in LIVE_COUNTS)


def small_set(fa: E.FieldArrays, name: str) -> ScatterInputs:
    """Set B, C, D or one cut of E by name (SMALL_SETS)."""
    if name.startswith("live"):
        return set_live(fa, LIVE_COUNTS[SMALL_SETS.index(name) - 3])
    return {"edges": set_edges, "collisions": set_collisions, "segments": set_segments}[name](fa)


def base_values(shape, seed) -> np.ndarray:
    """What a gradient buffer holds before the launch: random fp32 in a third of the entries, +0 elsewhere."""
    rng = np.random.default_rng(seed)
    b = (rng.standard_normal(shape) * 2.0 ** rng.uniform(-12, 2, shape)).astype(F32)
    b[rng.random(shape) < 2 / 3] = 0
    return b
