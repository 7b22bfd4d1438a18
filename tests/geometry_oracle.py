"""numpy restatement of hrf_mesh_distance (include/humanrf_b200.h, DESIGN.md §3.11): face eligibility, the integer-driven
area sampling (splitmix64, the uint64 CDF, the fp32 barycentric point) bit for bit, the fp32 closest-point routine
operation for operation, a brute-force scan with the kernel's tie rule, an fp64 reference distance, and the score
definitions.  Every fp32 value is a numpy float32 array, so each operation rounds on its own, as the kernel's __f*_rn.

The three ``wrong=`` switches are deliberately broken variants the tests use to show that the comparators catch them:
"plane" (distance to the triangle's plane), "nosqrt" (barycentrics without the square root) and "highest" (ties to the
highest face id)."""
from __future__ import annotations

import numpy as np

F32 = np.float32
M64 = np.uint64((1 << 64) - 1)


def _f(x):
    return np.asarray(x, np.float32)


# ---------------------------------------------------------------- faces
def face_info(V, F):
    """(eligible bool [F], unit normal f32 [F,3], area f32 [F]) as prep_kernel computes them."""
    V, F = _f(V).reshape(-1, 3), np.asarray(F, np.int64).reshape(-1, 3)
    ok = ((F >= 0) & (F < len(V))).all(1)
    Fs = np.where(ok[:, None], F, 0)
    if len(V) == 0:
        return ok & False, np.zeros((len(F), 3), F32), np.zeros(len(F), F32)
    a, b, c = V[Fs[:, 0]], V[Fs[:, 1]], V[Fs[:, 2]]
    e1, e2 = b - a, c - a
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    with np.errstate(all="ignore"):
        nn = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
        elig = ok & (nn > 0) & (nn < np.inf)
        ln = np.sqrt(nn)
        unit = np.where(elig[:, None], n / ln[:, None], F32(0))
        area = np.where(elig, F32(0.5) * ln, F32(0))
    return elig, unit.astype(F32), area.astype(F32)


def weights(area, elig):
    """q_f = floor(area_f / area_max * 2^32) (uint64), 0 for ineligible faces."""
    if not elig.any():
        return np.zeros(len(area), np.uint64)
    amax = np.float64(area[elig].max())
    q = np.floor(area.astype(np.float64) / amax * 4294967296.0)
    return np.where(elig, q, 0).astype(np.uint64)


# ---------------------------------------------------------------- random numbers
def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        z = x + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def mulhi64(a, b):
    """The high 64 bits of the 128-bit product of uint64 arrays."""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    m = np.uint64(0xFFFFFFFF)
    s = np.uint64(32)
    a0, a1, b0, b1 = a & m, a >> s, b & m, b >> s
    with np.errstate(over="ignore"):
        p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
        mid = (p00 >> s) + (p01 & m) + (p10 & m)
        return p11 + (p01 >> s) + (p10 >> s) + (mid >> s)


def sample(V, F, n, seed, wrong=None):
    """(points f32 [n,3], faces int32 [n]) of sample_kernel; (NaN, -1) when no face is eligible."""
    V, F = _f(V).reshape(-1, 3), np.asarray(F, np.int64).reshape(-1, 3)
    elig, _, area = face_info(V, F)
    q = weights(area, elig)
    if len(q) == 0 or int(q.sum(dtype=np.uint64)) == 0:
        return np.full((n, 3), np.nan, F32), np.full(n, -1, np.int32)
    P = np.concatenate([[np.uint64(0)], np.cumsum(q, dtype=np.uint64)[:-1]]).astype(np.uint64)
    Q = np.uint64(q.sum(dtype=np.uint64))
    k = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        base = np.uint64(seed) * np.uint64(1 << 40) + np.uint64(3) * k
        x0, x1, x2 = splitmix64(base), splitmix64(base + np.uint64(1)), splitmix64(base + np.uint64(2))
    t = mulhi64(x0, Q)
    face = np.searchsorted(P, t, side="right") - 1
    u1 = (x1 >> np.uint64(40)).astype(F32) * F32(2.0 ** -24)
    u2 = (x2 >> np.uint64(40)).astype(F32) * F32(2.0 ** -24)
    r = u1 if wrong == "nosqrt" else np.sqrt(u1)
    w0, w1, w2 = F32(1) - r, r * (F32(1) - u2), r * u2
    a, b, c = V[F[face, 0]], V[F[face, 1]], V[F[face, 2]]
    p = (w0[:, None] * a + w1[:, None] * b) + w2[:, None] * c
    return p.astype(F32), face.astype(np.int32)


# ---------------------------------------------------------------- distance
def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def _axpy(a, s, b):
    return a + s[..., None] * b


def point_triangle_d2(p, a, b, c, wrong=None):
    """point_triangle_d2 of csrc/mesh_distance.cu on broadcast float32 arrays [..., 3]: Ericson's Voronoi regions in
    the book's order, every operation rounded on its own, the point clamped into the triangle's box, |p - q|^2."""
    p, a, b, c = _f(p), _f(a), _f(b), _f(c)
    p, a, b, c = np.broadcast_arrays(p, a, b, c)
    with np.errstate(all="ignore"):
        ab, ac, ap = b - a, c - a, p - a
        if wrong == "plane":
            n = np.stack([ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1], ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2],
                          ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0]], -1)
            s = _dot(ap, n)
            return (s * s / _dot(n, n)).astype(F32)
        d1, d2 = _dot(ab, ap), _dot(ac, ap)
        bp = p - b
        d3, d4 = _dot(ab, bp), _dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = p - c
        d5, d6 = _dot(ab, cp), _dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        e43, e56 = d4 - d3, d5 - d6
        rem = np.ones(d1.shape, bool)
        regions = []
        for m in ((d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0),
                  (d6 >= 0) & (d5 <= d6), (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)):
            hit = rem & m
            regions.append(hit)
            rem = rem & ~hit
        denom = F32(1) / ((va + vb) + vc)
        cand = [a, b, _axpy(a, d1 / (d1 - d3), ab), c, _axpy(a, d2 / (d2 - d6), ac),
                _axpy(b, e43 / (e43 + e56), c - b), _axpy(_axpy(a, vb * denom, ab), vc * denom, ac)]
        q = cand[-1]
        for m, x in zip(regions[::-1], cand[-2::-1]):
            q = np.where(m[..., None], x, q)
        lo = np.fmin(np.fmin(a, b), c)
        hi = np.fmax(np.fmax(a, b), c)
        q = np.fmin(np.fmax(q, lo), hi)
        e = p - q
        return _dot(e, e).astype(F32)


def region(p, a, b, c):
    """Which Voronoi region Ericson's tests pick (0 A, 1 B, 2 AB, 3 C, 4 AC, 5 BC, 6 face), for test coverage."""
    p, a, b, c = np.broadcast_arrays(_f(p), _f(a), _f(b), _f(c))
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    tests = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)]
    out = np.full(d1.shape, 6)
    for k in range(5, -1, -1):
        out = np.where(tests[k], k, out)
    return out


def closest(points, V, F, chunk=256, wrong=None):
    """Brute force over every eligible face: (distance f32 [n], closest face int32 [n]); min d2, ties to the lowest id
    (highest with wrong="highest"); (+inf, -1) when no face is eligible, (NaN, -1) for a NaN point."""
    V, F = _f(V).reshape(-1, 3), np.asarray(F, np.int64).reshape(-1, 3)
    points = _f(points).reshape(-1, 3)
    elig, _, _ = face_info(V, F)
    ids = np.nonzero(elig)[0]
    n = len(points)
    dist, face = np.full(n, np.inf, F32), np.full(n, -1, np.int32)
    valid = ~np.isnan(points).any(1)
    dist[~valid] = np.nan
    if len(ids) == 0:
        return dist, face
    a, b, c = V[F[ids, 0]], V[F[ids, 1]], V[F[ids, 2]]
    for s in range(0, n, chunk):
        p = points[s:s + chunk]
        d2 = point_triangle_d2(p[:, None, :], a[None], b[None], c[None], wrong=None if wrong == "highest" else wrong)
        if wrong == "highest":
            j = d2.shape[1] - 1 - np.argmin(d2[:, ::-1], axis=1)
        else:
            j = np.argmin(d2, axis=1)
        dd = np.sqrt(d2[np.arange(len(p)), j])
        v = valid[s:s + chunk]
        dist[s:s + chunk][v] = dd[v]
        face[s:s + chunk][v] = ids[j][v]
    return dist, face


def exact_distance(p, a, b, c):
    """fp64 distance from p to triangle abc: the plane distance when the projection lies inside (all three edge
    functions >= 0), else the least of the three segment distances."""
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))

    def seg(x, y):
        d = y - x
        t = np.clip(_dot(p - x, d) / np.maximum(_dot(d, d), 1e-300), 0.0, 1.0)
        e = p - (x + t[..., None] * d)
        return np.sqrt(_dot(e, e))

    n = np.cross(b - a, c - a)
    nn = _dot(n, n)
    s = _dot(p - a, n) / nn
    proj = p - s[..., None] * n
    inside = ((_dot(np.cross(b - a, proj - a), n) >= 0) & (_dot(np.cross(c - b, proj - b), n) >= 0)
              & (_dot(np.cross(a - c, proj - c), n) >= 0))
    plane = np.abs(s) * np.sqrt(nn)
    best = np.minimum(np.minimum(seg(a, b), seg(b, c)), seg(c, a))
    return np.where(inside, np.minimum(plane, best), best)


# ---------------------------------------------------------------- scores
def direction(Vs, Fs, Vt, Ft, n, seed, taus):
    """One direction as the kernel computes it: (out [3] = means of d, d^2, normal term; counts; per-sample dict)."""
    p, f = sample(Vs, Fs, n, seed)
    d, g = closest(p, Vt, Ft)
    _, ns, _ = face_info(Vs, Fs)
    _, nt, _ = face_info(Vt, Ft)
    ok = (f >= 0) & (g >= 0)
    if not ok.all():
        return np.full(3, np.nan), np.full(len(taus), -1, np.int64), dict(points=p, faces=f, distances=d, closest=g)
    nterm = np.abs(_dot(ns[f], nt[g])).astype(F32)
    dd = d.astype(np.float64)
    out = np.array([dd.sum() / n, (dd * dd).sum() / n, nterm.astype(np.float64).sum() / n])
    counts = np.array([(d <= F32(t)).sum() for t in taus], np.int64)
    return out, counts, dict(points=p, faces=f, distances=d, closest=g)


def fscore(p, r):
    return 0.0 if p + r == 0 else 2 * p * r / (p + r)


def scores(fwd, bwd, cf, cb, n):
    """(accuracy, completeness, chamfer_l1, chamfer_l2, normal_consistency, precision, recall, F) from two directions."""
    P = [c / n for c in cf]
    R = [c / n for c in cb]
    return (fwd[0], bwd[0], (fwd[0] + bwd[0]) / 2, (fwd[1] + bwd[1]) / 2, (fwd[2] + bwd[2]) / 2, P, R,
            [fscore(p, r) for p, r in zip(P, R)])


# ---------------------------------------------------------------- test meshes
def random_mesh(nf, seed, decades=6.0, nv=None):
    """nf random triangles with areas spread over `decades` decades: random centres in [-1, 1]^3, edge scale
    10^U(-decades/2, 0), vertices shared by nothing (3 per face)."""
    rng = np.random.default_rng(seed)
    centre = rng.uniform(-1, 1, (nf, 1, 3))
    scale = 10.0 ** rng.uniform(-decades / 2, 0, (nf, 1, 1))
    V = (centre + scale * rng.normal(size=(nf, 3, 3))).reshape(-1, 3).astype(F32)
    F = np.arange(3 * nf, dtype=np.int32).reshape(-1, 3)
    return V, F


def icosphere(subdiv, radius=1.0):
    """Icosahedron subdivided `subdiv` times, vertices projected to the sphere of `radius` (float64 then float32)."""
    t = (1 + 5 ** 0.5) / 2
    V = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
         (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    F = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    V = [np.array(v, np.float64) / np.linalg.norm(v) for v in V]
    for _ in range(subdiv):
        mid = {}

        def m(i, j):
            key = (min(i, j), max(i, j))
            if key not in mid:
                x = V[i] + V[j]
                V.append(x / np.linalg.norm(x))
                mid[key] = len(V) - 1
            return mid[key]

        F = [f for a, b, c in F for f in ((a, m(a, b), m(a, c)), (b, m(b, c), m(a, b)), (c, m(a, c), m(b, c)),
                                         (m(a, b), m(b, c), m(a, c)))]
    return (np.array(V) * radius).astype(F32), np.array(F, np.int32)


def sphere_tessellation_gap(V, F, radius):
    """Largest distance from a point of the icosphere's triangles to the sphere of `radius`: radius minus the smallest
    circumradius-based distance of a face plane from the centre (flat faces lie inside the sphere)."""
    V = np.asarray(V, np.float64)
    a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    n = np.cross(b - a, c - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    plane = np.abs((a * n).sum(1))
    return float(radius - plane.min())
