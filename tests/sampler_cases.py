"""Seeded edge cases for the ray sampler (csrc/sampler.cu, oracle/sampler.py).

Every scene is a dict in the shape `humanrf_b200.synthetic_scene.make_scene` returns, so `oracle.sampler.get_data` and
the `ray_sampler_native` entry points take it unchanged, plus `world2pixel` [B,4,4] float64: each image's
`projection_matrix_world2pixel` (ActorsHQ camera model), NaN for the degenerate cameras that have none.

Most cameras are built from their sampler table directly.  Columns R·(1,0,0), R·(0,1,0), R·(-cx,-cy,f) with R a signed
permutation give v = R·(px+1/2-cx, py+1/2-cy, f) exactly, so the pixel (cx-1/2, cy-1/2) looks along ±x, ±y or ±z with
direction components that are exactly +0 (f is a power of two, so the direction is exactly ±1 on its axis).  A table
whose row k is -0 gives every ray of the camera a direction component of exactly -0.

Families (`family(name)`), each in landscape and portrait images:
  axis    axis-aligned rays inside the slabs, on face planes, on edge lines, outside; -0 components
  origin  camera origins inside the box, on a face, at a corner
  graze   rays that touch the box only at an edge or a corner (tmin == tmax up to rounding)
  miss    cameras looking away from the box
  ring    cameras on a ring at distance 2 looking at the origin (as the synthetic scene), box wider than the grid
  placed  rays whose first occupied march step is lane 0 of round 0, lane 31, or lane 0 of a later round (forward and
          backward march)
  counts  candidate counts 0, 1, 31, 32, 33, 1023, 1025 on chosen rays
Grids: `pattern(name, G)` for G in GRID_SIZES; batches: `batches()`.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
from scipy.spatial.transform import Rotation

from humanrf_b200.dataset.cameras import inverse_kr, projection_matrix_world2pixel
from humanrf_b200.synthetic_scene import look_at_camera
from oracle import sampler as S

f32 = np.float32
W, H = 40, 24                     # landscape image; portrait images are H x W
F_WIDE, F_NARROW = 32.0, 128.0    # focal lengths in pixels (powers of two)
AABB = np.array([[-0.45, -0.5, -0.4], [0.5, 0.45, 0.5]], f32)
AABB_WIDE = np.array([[-0.55, -0.6, -0.52], [0.6, 0.55, 0.58]], f32)  # reaches past the grid's [-0.5, 0.5]^3
GRID_SIZES = (1, 2, 3, 31, 33, 100, 128, 257, 512)
PATTERNS = ("empty", "full", "corners", "checker", "shell", "ellipsoid")
COUNT_TARGETS = (0, 1, 31, 32, 33, 1023, 1025)
LANE_TARGETS = (0, 31, 32, 33, 63, 64)
STEP = 2e-3


# ---------------------------------------------------------------------------------------------------------------- grids
def pattern(name: str, G: int, seed: int = 0) -> np.ndarray:
    """uint8 [G,G,G] indexed [z][y][x], occupied = 255."""
    if name == "empty":
        return np.zeros((G, G, G), np.uint8)
    if name == "full":
        return np.full((G, G, G), 255, np.uint8)
    if name == "corners":  # one voxel at each corner and at the centre of each face: the filter's clamp at G - 1
        g = np.zeros((G, G, G), np.uint8)
        e, m = G - 1, G // 2
        for z in (0, e):
            for y in (0, e):
                for x in (0, e):
                    g[z, y, x] = 255
        for k in range(3):
            for v in (0, e):
                c = [m, m, m]
                c[k] = v
                g[tuple(c)] = 255
        return g
    i = np.arange(G)
    if name == "checker":  # the march's bisection flips at every step, counts with holes
        par = (i % 2).astype(np.uint8)
        return ((1 - (par[:, None, None] ^ par[None, :, None] ^ par[None, None, :])) * 255).astype(np.uint8)
    c = ((i + 0.5) / G - 0.5).astype(np.float32)
    out = np.zeros((G, G, G), np.uint8)
    if name == "shell":  # two thin spherical shells
        t = max(1.0 / G, 0.01)
        for z in range(G):  # one z layer at a time keeps G = 512 within a few MB
            r = np.sqrt(c[None, :] ** 2 + c[:, None] ** 2 + c[z] ** 2)
            out[z] = ((np.abs(r - 0.4) < t) | (np.abs(r - 0.2) < t)) * 255
        return out
    if name == "ellipsoid":
        rng = np.random.default_rng(seed)
        ctr, rad = rng.uniform(-0.15, 0.15, 3), rng.uniform(0.15, 0.4, 3)
        for z in range(G):
            q = ((c[None, :] - ctr[0]) / rad[0]) ** 2 + ((c[:, None] - ctr[1]) / rad[1]) ** 2 + ((c[z] - ctr[2]) / rad[2]) ** 2
            out[z] = (q <= 1.0) * 255
        return out
    raise ValueError(name)


def slab_grid(G: int, z0: int, z1: int) -> np.ndarray:
    g = np.zeros((G, G, G), np.uint8)
    g[z0:z1 + 1] = 255
    return g


# -------------------------------------------------------------------------------------------------------------- cameras
@dataclass
class Cam:
    table: np.ndarray             # [3,3] float32, row i = GLM column i
    origin: np.ndarray            # [3] float32
    landscape: bool
    w2p: np.ndarray | None        # [4,4] float64 projection_matrix_world2pixel, None for degenerate tables
    pixels: list = field(default_factory=list)   # (x, y) pixels to sample

    @property
    def wh(self):
        return (W, H) if self.landscape else (H, W)


def axis_rotation(axis: int, sign: int) -> np.ndarray:
    """Camera-to-world signed permutation (columns right, down, forward) looking along sign·e_axis, det +1."""
    fwd = np.zeros(3)
    fwd[axis] = sign
    right = np.zeros(3)
    right[(axis + 1) % 3] = 1.0
    return np.stack([right, np.cross(fwd, right), fwd], 1)


def axis_cam(R, origin, cx, cy, landscape, f=F_WIDE) -> Cam:
    """Pinhole with focal length f and principal point (cx, cy) in pixels; exact table entries for half-integer c."""
    T = np.stack([R[:, 0], R[:, 1], R @ np.array([-cx, -cy, f])]).astype(f32)
    w, h = (W, H) if landscape else (H, W)
    w2p = projection_matrix_world2pixel(w, h, Rotation.from_matrix(R).as_rotvec(), np.asarray(origin, np.float64),
                                        np.array([f / w, f / h]), np.array([cx / w, cy / h]))
    return Cam(T, np.asarray(origin, f32), landscape, w2p)


def plane_cam(k: int, origin, cx, cy, landscape, f=F_WIDE) -> Cam:
    """Row k of the table is -0: v_k = fma(-0, 1, fma(-0, py, -0·px)) = -0 for every pixel, so every ray has d_k = -0.
    The other two components are (px + 1/2 - cx, py + 1/2 - cy + f) on axes k+1, k+2."""
    a, b = (k + 1) % 3, (k + 2) % 3
    T = np.zeros((3, 3), f32)
    T[:, k] = -0.0
    T[0, a], T[2, a] = 1.0, -cx
    T[1, b], T[2, b] = 1.0, f - cy
    return Cam(T, np.asarray(origin, f32), landscape, None)


def ring_cam(i, n, rng, landscape, dist=2.0) -> Cam:
    a = 2 * np.pi * i / n + 0.3
    pos = np.array([dist * np.cos(a), rng.uniform(-0.4, 0.4), dist * np.sin(a)])
    w, h = (W, H) if landscape else (H, W)
    M = look_at_camera(pos, w, h)
    return Cam(inverse_kr(M), pos.astype(f32), landscape, M)


def pixel_index(cams, b, x, y) -> int:
    w, _ = cams[b].wh
    return b * W * H + y * w + x


def directions(cam: Cam, pixels):
    """The oracle's (origin, direction) of `pixels` of one camera."""
    idx = np.array([y * cam.wh[0] + x for x, y in pixels], np.int64)
    return S.ray_directions(cam.table[None], cam.origin[None], np.array([cam.landscape]), idx, W, H)[:2]


# --------------------------------------------------------------------------------------------------------------- scenes
@dataclass
class Case:
    family: str
    scene: dict
    idx: np.ndarray
    steps: tuple = (STEP,)


def make(cams, grids, G, aabb=AABB, seed=0, light_all=False) -> dict:
    rng = np.random.default_rng(seed + 1000)
    B = len(cams)
    P = B * W * H
    return dict(
        inverse_krs=np.stack([c.table for c in cams]).astype(f32), camera_origins=np.stack([c.origin for c in cams]),
        landscape=np.array([c.landscape for c in cams]), grids=list(grids), G=G, width=W, height=H,
        frame_numbers=(15 + np.arange(B) % 6).astype(np.int32), camera_numbers=rng.integers(0, 160, B).astype(np.int32),
        rgba=rng.integers(0, 256, (P, 4)).astype(np.uint8),
        light_mask=np.ones(P, bool) if light_all else rng.random(P) < 0.1,
        aabb=np.array(aabb, f32),
        world2pixel=np.stack([c.w2p if c.w2p is not None else np.full((4, 4), np.nan) for c in cams]))


def grids_for(n_images, G, patterns=PATTERNS, seed=0):
    """One grid per image, the patterns dealt round-robin (shared arrays, so large G stays cheap)."""
    made = {p: pattern(p, G, seed) for p in patterns[:n_images]}
    return [made[patterns[i % len(patterns)]] for i in range(n_images)]


def indices(cams) -> np.ndarray:
    return np.array([pixel_index(cams, b, x, y) for b, c in enumerate(cams) for x, y in c.pixels], np.int64)


def unbounded(o, d, aabb):
    """Rays the glm slab test keeps with tmin = -inf or tmax = +inf.  Only one configuration does it: d_x = d_y = 0,
    the origin strictly inside the x slab and exactly on the lower y face (the y face's NaN hides the y and z slabs,
    see test_sampler_oracle_cpu.expected_slab).  Its march would never end, so no case contains it."""
    tmin, tmax = S.aabb_minmax(o, d, aabb)
    return (tmin < tmax) & ~(np.isfinite(tmin) & np.isfinite(tmax))


def _drop_unbounded(cams, aabb):
    for c in cams:
        if not c.pixels:
            continue
        o, d = directions(c, c.pixels)
        bad = unbounded(o, d, aabb)
        for j in np.nonzero(bad)[0]:
            assert d[j, 0] == 0 and d[j, 1] == 0 and o[j, 1] == aabb[0, 1] and aabb[0, 0] < o[j, 0] < aabb[1, 0]
        c.pixels = [p for p, b in zip(c.pixels, bad) if not b]


def _around(cam: Cam, x0, y0, rng, n_random=4):
    w, h = cam.wh
    px = [(x0 + dx, y0 + dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if 0 <= x0 + dx < w and 0 <= y0 + dy < h]
    px += [(int(rng.integers(0, w)), int(rng.integers(0, h))) for _ in range(n_random)]
    return px


# ------------------------------------------------------------------------------------------------------------- families
def _pos(where, k, rng, aabb):
    lo, hi = float(aabb[0, k]), float(aabb[1, k])
    return {"in": rng.uniform(lo + 0.05, hi - 0.05), "lo": lo, "hi": hi, "out_lo": lo - 0.2, "out_hi": hi + 0.2}[where]


def axis_cams(rng, aabb=AABB):
    cams = []
    places = ("in", "lo", "hi", "out_lo", "out_hi")
    n = 0
    for axis in range(3):
        for sign in (1, -1):
            R = axis_rotation(axis, sign)
            a, b = (axis + 1) % 3, (axis + 2) % 3
            for pa in places:
                for pb in places:
                    o = np.zeros(3)
                    o[axis] = 0.5 * (aabb[0, axis] + aabb[1, axis]) - sign * 2.0
                    o[a], o[b] = _pos(pa, a, rng, aabb), _pos(pb, b, rng, aabb)
                    ls = n % 2 == 0
                    w, h = (W, H) if ls else (H, W)
                    x0, y0 = int(rng.integers(1, w - 1)), int(rng.integers(1, h - 1))
                    c = axis_cam(R, o, x0 + 0.5, y0 + 0.5, ls)
                    c.pixels = _around(c, x0, y0, rng)
                    cams.append(c)
                    n += 1
    for k in range(3):  # -0 direction components
        a, b = (k + 1) % 3, (k + 2) % 3
        for where in ("in", "lo", "hi", "out_lo"):
            o = np.zeros(3)
            o[k] = _pos(where, k, rng, aabb)
            o[b] = aabb[0, b] - 1.5
            ls = n % 2 == 0
            w, h = (W, H) if ls else (H, W)
            c = plane_cam(k, o, w / 2 + 0.25, h / 2 + 0.25, ls)
            c.pixels = [(int(rng.integers(0, w)), int(rng.integers(0, h))) for _ in range(12)]
            cams.append(c)
            n += 1
    return cams


def origin_cams(rng, aabb=AABB):
    lo, hi = aabb[0].astype(np.float64), aabb[1].astype(np.float64)
    origins = [lo + rng.uniform(0.1, 0.9, 3) * (hi - lo) for _ in range(4)]
    for k in range(3):
        for v in (lo[k], hi[k]):
            p = lo + rng.uniform(0.2, 0.8, 3) * (hi - lo)
            p[k] = v
            origins.append(p)
    origins += [np.array([(lo, hi)[(c >> k) & 1][k] for k in range(3)]) for c in range(8)]
    cams = []
    for n, o in enumerate(origins):
        R = axis_rotation(int(rng.integers(0, 3)), int(rng.choice([-1, 1])))
        ls = n % 2 == 0
        w, h = (W, H) if ls else (H, W)
        x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
        c = axis_cam(R, o, x0 + 0.5, y0 + 0.5, ls)
        sel = rng.choice(w * h, 90, replace=False)
        c.pixels = [(x0, y) for y in range(h)] + [(x, y0) for x in range(w)] + [(int(i % w), int(i // w)) for i in sel]
        cams.append(c)
    return cams


def graze_cams(rng, aabb=AABB):
    """Each camera's first pixel touches the box only at one edge or corner point: the line passes through the point,
    and the direction leaves through one of the point's faces on either side (outward components of both signs)."""
    lo, hi = aabb[0].astype(np.float64), aabb[1].astype(np.float64)
    targets = []
    for k in range(3):  # 12 edges: axis k free
        a, b = (k + 1) % 3, (k + 2) % 3
        for sa in (-1, 1):
            for sb in (-1, 1):
                targets.append({a: sa, b: sb})
    targets += [{0: sx, 1: sy, 2: sz} for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
    cams = []
    for t_i, normals in enumerate(targets):
        for rep in range(3):
            e = lo + rng.uniform(0.2, 0.8, 3) * (hi - lo)
            for k, s in normals.items():
                e[k] = hi[k] if s > 0 else lo[k]
            ls = (t_i + rep) % 2 == 0
            w, h = (W, H) if ls else (H, W)
            for _ in range(1000):
                R = axis_rotation(int(rng.integers(0, 3)), int(rng.choice([-1, 1])))
                c = axis_cam(R, np.zeros(3), w / 2, h / 2, ls)
                px = (int(rng.integers(0, w)), int(rng.integers(0, h)))
                d = directions(c, [px])[1][0].astype(np.float64)
                out = [s * d[k] for k, s in normals.items()]
                if max(out) > 0.05 and min(out) < -0.05:
                    break
            else:
                raise AssertionError("no grazing direction found")
            c = axis_cam(R, e - 1.5 * d, w / 2, h / 2, ls)
            c.pixels = [px] + [(px[0] + dx, px[1] + dy) for dx, dy in ((-1, 0), (1, 0), (0, -1), (0, 1))
                               if 0 <= px[0] + dx < w and 0 <= px[1] + dy < h]
            cams.append(c)
    return cams


def miss_cams(rng, aabb=AABB):
    """Narrow cameras beside the box looking parallel to one of its axes: every line misses it.  (A camera behind the
    box looking away from it still intersects the line at negative t; the slab test does not clip t >= 0.)"""
    cams = []
    n = 0
    for axis in range(3):
        for side in (-1, 1):
            o = np.zeros(3)
            o[axis] = -2.0
            o[(axis + 1) % 3] = side * 1.5
            ls = n % 2 == 0
            w, h = (W, H) if ls else (H, W)
            c = axis_cam(axis_rotation(axis, 1), o, w / 2, h / 2, ls, f=F_NARROW)
            sel = rng.choice(w * h, 40, replace=False)
            c.pixels = [(int(i % w), int(i // w)) for i in sel]
            cams.append(c)
            n += 1
    return cams


def ring_cams(rng, n=6, per_image=150):
    cams = []
    for i in range(n):
        c = ring_cam(i, n, rng, landscape=i % 3 != 2)
        w, h = c.wh
        sel = rng.choice(w * h, per_image, replace=False)
        c.pixels = [(int(i % w), int(i // w)) for i in sel]
        cams.append(c)
    return cams


def march_indices(o, d, aabb, grids, img, G):
    """Per ray, the number of `t += step` (forward) and `t -= step` (backward) moves the oracle's march makes before it
    stops (the oracle's own fp32 sequence, vectorised over rays); -1 when that march does not start."""
    tmin0, tend = S.aabb_minmax(o, d, aabb)
    tmin_ref, _ = S.occupancy_minmax(o, d, aabb, grids, img, G)
    step = f32(0.5) / f32(G)

    def occ(ids, t):
        p = (S.fma32(d[ids], t[:, None], o[ids]) + f32(0.5)).astype(f32)
        out = np.zeros(ids.size, bool)
        for g in np.unique(img[ids]):
            s = img[ids] == g
            out[s] = S.tex_occupied(grids[g], p[s])
        return out

    res = []
    for fwd in (True, False):
        t = (tmin0 if fwd else tend).copy()
        n = np.where(tmin0 < tend, 0, -1)
        active = tmin0 < tend
        while active.any():
            ids = np.nonzero(active)[0]
            stop = ~(t[ids] < tend[ids]) | occ(ids, t[ids]) if fwd else ~(t[ids] > tmin_ref[ids]) | occ(ids, t[ids])
            active[ids[stop]] = False
            go = ids[~stop]
            t[go] = (t[go] + step if fwd else t[go] - step).astype(f32)
            n[go] += 1
        res.append(n)
    return res[0], res[1]


def placed_case(rng, G=128):
    """Half a dozen cameras just in front of the box's z entry face (f = 32, so the path to a z slab of occupied voxels
    grows by up to 25 % across the image) and slabs that start and end at chosen voxel layers; pixels are picked whose
    forward / backward march stops after exactly 0, 31, 32, 33, 63 or 64 moves (lane 0 / 31 / 0 / 1 / 31 / 0 of
    rounds 0, 0, 1, 1, 1, 2)."""
    slabs = [(12, 127), (27, 111), (43, 95)]
    cams, grids = [], []
    for n in range(6):
        ls = n % 2 == 0
        w, h = (W, H) if ls else (H, W)
        c = axis_cam(axis_rotation(2, 1), [0.01, -0.02, -0.45], w / 2, h / 2, ls)
        c.pixels = [(x, y) for y in range(h) for x in range(w)]
        cams.append(c)
        grids.append(slab_grid(G, *slabs[n // 2]))
    sc = make(cams, grids, G, seed=7)
    idx = indices(cams)
    o, d, img = S.ray_directions(sc["inverse_krs"], sc["camera_origins"], sc["landscape"], idx, W, H)
    nf, nb = march_indices(o, d, AABB, grids, img, G)
    pick = []
    for t in LANE_TARGETS:
        for n in (nf, nb):
            hits = np.nonzero(n == t)[0]
            assert hits.size, f"no ray stops after {t} march moves"
            pick += list(rng.choice(hits, min(4, hits.size), replace=False))
    pick += list(rng.choice(idx.size, 60, replace=False))
    return Case("placed", sc, idx[np.sort(np.unique(pick))])


def counts_cases(rng, G=33):
    """A narrow camera looking along +z through the box; for each target c one step = L / (c + 1/2), L the axis ray's
    fp32 box length, so that ray has exactly c candidates (its neighbours one or two more)."""
    cams = []
    for ls in (True, False):
        w, h = (W, H) if ls else (H, W)
        x0, y0 = w // 2, h // 2
        c = axis_cam(axis_rotation(2, 1), [0.02, -0.03, -2.0], x0 + 0.5, y0 + 0.5, ls, f=F_NARROW)
        c.pixels = _around(c, x0, y0, rng, n_random=20)
        cams.append(c)
    o, d = directions(cams[0], cams[0].pixels[4:5])
    tmin, tmax = S.aabb_minmax(o, d, AABB)
    L = float(f32(tmax[0] - tmin[0]))
    steps = tuple(float(f32(L / (c + 0.5))) for c in COUNT_TARGETS)
    sc = make(cams, [pattern("full", G), pattern("checker", G)], G, seed=11)
    return Case("counts", sc, indices(cams), steps=steps)


def family(name: str, G: int = 128, patterns=PATTERNS, seed: int = 0) -> Case:
    rng = np.random.default_rng([seed, FAMILIES.index(name)])
    if name == "placed":
        return placed_case(rng)
    if name == "counts":
        return counts_cases(rng)
    if name == "ring":
        aabb, cams = AABB_WIDE, ring_cams(rng)
    else:
        aabb, cams = AABB, {"axis": axis_cams, "origin": origin_cams, "graze": graze_cams, "miss": miss_cams}[name](rng)
    _drop_unbounded(cams, aabb)
    return Case(name, make(cams, grids_for(len(cams), G, patterns, seed), G, aabb, seed), indices(cams))


FAMILIES = ("axis", "origin", "graze", "miss", "ring", "placed", "counts")


def count_check(case: Case):
    """The axis ray of the counts family has exactly COUNT_TARGETS[i] candidates at steps[i] (aabb mode)."""
    sc = case.scene
    got = []
    for s in case.steps:
        o, d, _ = S.ray_directions(sc["inverse_krs"], sc["camera_origins"], sc["landscape"], case.idx[4:5], W, H)
        tmin, tmax = S.aabb_minmax(o, d, sc["aabb"])
        got.append(int((f32(tmax[0] - tmin[0]) * (f32(1.0) / f32(s))).astype(f32)))
    return got


# -------------------------------------------------------------------------------------------------------------- batches
def batches(seed=0, G=31):
    """Batches at the scan's 1024-ray chunk seams on a ring scene whose image 2 looks away from the box (all its rays
    miss).  Returns (name, scene, idx, samples_ok) with samples_ok False for the 2^20-ray batch (rays entry points, or
    a coarse step, only)."""
    rng = np.random.default_rng(seed + 77)
    cams = ring_cams(rng, n=4)
    miss = miss_cams(rng)[0]
    cams.insert(2, miss)
    n_img = len(cams)
    sc = make(cams, grids_for(n_img, G, ("ellipsoid", "checker", "empty", "shell", "full")), G, AABB_WIDE, seed)
    P = n_img * W * H
    o, d, _ = S.ray_directions(sc["inverse_krs"], sc["camera_origins"], sc["landscape"], np.arange(P), W, H)
    tmin, tmax = S.aabb_minmax(o, d, sc["aabb"])
    hit = np.nonzero(tmin < tmax)[0]
    missed = np.arange(2 * W * H, 3 * W * H)
    assert not (tmin[missed] < tmax[missed]).any()
    out = []
    for R in (1, 31, 32, 33, 1023, 1024, 1025, 3 * 1024 + 7):
        out.append((f"R={R}", sc, rng.integers(0, P, R).astype(np.int64), True))
    idx = rng.integers(0, P, 3 * 1024 + 7)
    idx[1024:2048] = rng.choice(missed, 1024)              # a whole masked chunk
    out.append(("masked chunk 1", sc, idx, True))
    idx = rng.choice(missed, 3 * 1024 + 7)
    idx[-1] = hit[hit >= (n_img - 1) * W * H][-1]           # only the last ray kept, a pixel of the last image
    out.append(("last ray only", sc, idx, True))
    out.append(("duplicates", sc, rng.choice(rng.integers(0, P, 40), 1025), True))
    idx = rng.integers((n_img - 1) * W * H, P, 1023)
    idx[-1] = P - 1
    out.append(("last image", sc, idx, True))
    out.append(("R=2^20+3", sc, rng.integers(0, P, 2 ** 20 + 3).astype(np.int64), False))
    return out
