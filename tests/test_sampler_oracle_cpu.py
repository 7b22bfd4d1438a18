"""The sampler oracle (oracle/sampler.py) against checks that do not restate it, on the edge cases of
tests/sampler_cases.py: float64 directions and slab intervals with derived bounds, the pixel convention through the
ActorsHQ camera model, a scalar march and a per-ray sample emission written from the contract, and named mutants that
these checks must tell apart from the oracle."""
import numpy as np
import pytest

import sampler_cases as SC
from oracle import sampler as S

f32 = np.float32
U = 2.0 ** -24
G3 = 3 * U / (1 - 3 * U)
PIXEL_BOUND = 1e-3
CPU_FAMILIES = {  # family -> (G, grid patterns) for the occupancy checks
    "axis": (33, SC.PATTERNS), "origin": (31, SC.PATTERNS), "graze": (3, ("full", "checker")),
    "miss": (2, ("full",)), "ring": (100, ("corners", "ellipsoid", "checker")), "placed": (128, None),
    "counts": (33, None)}


def _case(name):
    G, pats = CPU_FAMILIES[name]
    return SC.family(name, G, pats) if pats else SC.family(name)


def _rays(case, landscape=None):
    sc = case.scene
    ls = sc["landscape"] if landscape is None else landscape
    return S.ray_directions(sc["inverse_krs"], sc["camera_origins"], ls, case.idx, SC.W, SC.H)


def _bits_equal(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


# ----------------------------------------------------------------------------------------------------------- directions
def direction_bound(T, px, py):
    """Per-component bound on |d_oracle - normalize(v)|, v = px·T0 + py·T1 + T2 in exact arithmetic (T the fp32 table).

    ray_directions rounds v_k = fma(T2k, 1, fma(T1k, py, fl(T0k·px))) three times: |v^_k - v_k| <= e_k = γ3·S_k with
    S_k = |T0k·px| + |T1k·py| + |T2k|.  Normalising an exact vector a instead of b moves component k by at most
    (|a_k - b_k| + |b_k/|b||·|a - b|) / |a|.  The normalisation itself (the fma chain of the dot product, relative γ3;
    sqrt, 1/x and the final multiply, one rounding each) scales v^_k/|v^| by (1 + ε) with |ε| <= 8u.  So
        bound_k = (e_k + |d_k|·|e|) / (|v| - |e|) + 8u·(|v_k| + e_k) / (|v| - |e|),   u = 2^-24, γ3 = 3u / (1 - 3u)."""
    T = T.astype(np.float64)
    v = px[:, None] * T[:, 0] + py[:, None] * T[:, 1] + T[:, 2]
    S_ = np.abs(px[:, None] * T[:, 0]) + np.abs(py[:, None] * T[:, 1]) + np.abs(T[:, 2])
    e = G3 * S_
    nv = np.linalg.norm(v, axis=1, keepdims=True)
    ne = np.linalg.norm(e, axis=1, keepdims=True)
    d = v / nv
    return d, (e + np.abs(d) * ne) / (nv - ne) + 8 * U * (np.abs(v) + e) / (nv - ne) + 1e-15


def _pixels(case):
    sc = case.scene
    img = case.idx // (SC.W * SC.H)
    ls = sc["landscape"][img]
    w, h = np.where(ls, SC.W, SC.H), np.where(ls, SC.H, SC.W)
    return img, case.idx % w, (case.idx // w) % h


@pytest.mark.parametrize("name", list(CPU_FAMILIES))
def test_directions_within_derived_bound(name):
    case = _case(name)
    img, x, y = _pixels(case)
    _, d, _ = _rays(case)
    d64, bound = direction_bound(case.scene["inverse_krs"][img], x + 0.5, y + 0.5)
    ratio = np.abs(d - d64) / bound
    print(f"{name}: {d.shape[0]} rays, largest direction error = {ratio.max():.3f} of the bound")
    assert ratio.max() <= 1.0
    ax = np.abs(d64) == 1.0                                   # the exact axis rays are exact
    assert np.array_equal(d[ax], d64[ax])


# ------------------------------------------------------------------------------------------------------ pixel convention
def pixel_violations(case, landscape=None):
    """Largest distance in pixels between the projection of o + d (t = 1, float64) through the image's float64
    world2pixel matrix and the centre of the pixel the index rule gives (x = idx % w, y = (idx / w) % h, w and h
    swapped for portrait images)."""
    sc = case.scene
    img, x, y = _pixels(case)
    o, d, _ = _rays(case, landscape)
    M = sc["world2pixel"][img]
    ok = np.isfinite(M).all(axis=(1, 2))
    p = np.concatenate([o + d.astype(np.float64), np.ones((o.shape[0], 1))], 1)[ok]
    q = np.einsum("nij,nj->ni", M[ok], p)
    uv = q[:, :2] / q[:, 2:3]
    return np.abs(uv - np.stack([x[ok] + 0.5, y[ok] + 0.5], 1)).max(initial=0.0), int(ok.sum())


@pytest.mark.parametrize("name", list(CPU_FAMILIES))
def test_pixel_convention(name):
    """Bound: f <= 72 px times a direction error below 2e-6 rad (the direction bound, plus the fp32 rounding of the
    ring cameras' tables) is 1.5e-4 px; PIXEL_BOUND = 1e-3 px."""
    case = _case(name)
    err, n = pixel_violations(case)
    print(f"{name}: {n} rays with a camera model, largest pixel error {err:.2e} px")
    assert n > 0 and err <= PIXEL_BOUND


# ----------------------------------------------------------------------------------------------------------- slab test
def expected_slab(o, d, aabb):
    """Float64 slab test with the fp32 kernels' handling of zero direction components stated case by case.

    Nonzero components: t = (bb - o) / d in float64; the oracle's fl(fl(bb - o)·fl(1/d)) is within γ3·|t|, and min
    and max move by at most the largest error among their operands.  A zero component makes 1/d = ±inf, so the axis
    gives ±inf, or NaN where bb - o = 0 (the origin on a face plane).  The glm ternaries min(a,b) = b < a ? b : a and
    max(a,b) = a < b ? b : a return their FIRST operand when either is NaN, which gives:
      * origin strictly inside the slab: the axis does not constrain;
      * strictly outside: rejected;
      * on the lower face of x: rejected (tmin and tmax are NaN);
      * on the lower face of y: the y AND z slabs drop out (max(min_y, min_z) is NaN, and max(min_x, NaN) = min_x);
      * on the lower face of z: the z slab drops out;
      * on the upper face (of an axis that has not dropped out): rejected (tmax = -inf for +0, tmin = +inf for -0).
    Returns (rejected, lo, hi, bound) per ray; lo/hi are NaN for rejected rays."""
    n = o.shape[0]
    o64, d64 = o.astype(np.float64), d.astype(np.float64)
    lo_b, hi_b = aabb[0], aabb[1]
    zero = d == 0
    where = np.full((n, 3), "", object)
    where[zero & (o > lo_b) & (o < hi_b)] = "in"
    where[zero & (o == lo_b)] = "lo"
    where[zero & (o == hi_b)] = "hi"
    where[zero & ((o < lo_b) | (o > hi_b))] = "out"
    dropped = np.zeros((n, 3), bool)
    dropped[where[:, 1] == "lo", 1:] = True
    dropped[(where[:, 2] == "lo") & ~dropped[:, 2], 2] = True
    rejected = where[:, 0] == "lo"
    for k in range(3):
        rejected |= ~dropped[:, k] & np.isin(where[:, k], ["hi", "out"])
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (lo_b.astype(np.float64) - o64) / d64
        t1 = (hi_b.astype(np.float64) - o64) / d64
    use = ~zero & ~dropped
    mn = np.where(use, np.minimum(t0, t1), -np.inf)
    mx = np.where(use, np.maximum(t0, t1), np.inf)
    lo, hi = mn.max(1), mx.min(1)
    err = np.where(use, G3 * np.maximum(np.abs(t0), np.abs(t1)), 0.0)
    bound = err.max(1) + 1e-300
    lo[rejected], hi[rejected] = np.nan, np.nan
    return rejected, lo, hi, bound


def slab_violations(case):
    o, d, _ = _rays(case)
    aabb = case.scene["aabb"]
    tmin, tmax = S.aabb_minmax(o, d, aabb)
    rejected, lo, hi, bound = expected_slab(o, d, aabb)
    kept = tmin < tmax
    bad = rejected & kept
    iv = ~rejected
    assert np.isfinite(lo[iv]).all() and np.isfinite(hi[iv]).all(), "an unbounded ray slipped into the cases"
    bad[iv] |= (np.abs(tmin[iv] - lo[iv]) > bound[iv]) | (np.abs(tmax[iv] - hi[iv]) > bound[iv])
    close = iv & (np.abs(hi - lo) <= 2 * bound)
    bad |= iv & ~close & (kept != (hi > lo))
    return int(bad.sum()), int(close.sum()), int(kept.sum()), int((~kept).sum())


@pytest.mark.parametrize("name", list(CPU_FAMILIES))
def test_slab_test_against_float64(name):
    case = _case(name)
    bad, close, kept, rej = slab_violations(case)
    print(f"{name}: {kept} kept, {rej} rejected, {close} within rounding of tmin == tmax")
    assert bad == 0
    if name == "graze":
        assert close >= 50           # 60 grazing cameras: their first pixel touches the box at one point


def test_face_plane_cases_present():
    """The axis family reaches every row of expected_slab's table, with +0 and -0 components."""
    case = _case("axis")
    o, d, _ = _rays(case)
    aabb = case.scene["aabb"]
    tmin, tmax = S.aabb_minmax(o, d, aabb)
    kept = tmin < tmax
    z = d == 0
    for k in range(3):
        for face, b in (("lo", aabb[0, k]), ("hi", aabb[1, k])):
            on = z[:, k] & (o[:, k] == b)
            assert on.any(), (k, face)
            for neg in (False, True):
                assert (on & (np.signbit(d[:, k]) == neg)).any(), (k, face, neg)
    y_lo = z[:, 1] & (o[:, 1] == aabb[0, 1]) & ~(z[:, 0] & (o[:, 0] == aabb[0, 0]))
    assert (kept & y_lo).any(), "no ray in the lower y face plane kept by the x slab alone"
    assert (~kept & z[:, 0] & (o[:, 0] == aabb[0, 0])).any()


# ---------------------------------------------------------------------------------------------------------------- march
def _tex(grid, p, clamp_hi=None):
    """The texture filter with the upper clamp at `clamp_hi` (G - 1 is the hardware's; G reads an empty layer)."""
    G = grid.shape[0]
    c = G - 1 if clamp_hi is None else clamp_hi
    g = np.zeros((c + 1,) * 3, bool)
    g[:G, :G, :G] = grid > 0
    q = np.floor(((p.astype(f32) * f32(G)).astype(f32) - f32(0.5)).astype(f32) * f32(256.0) + f32(0.5)).astype(np.int64)
    i0, a = q >> 8, q & 255
    occ = np.zeros(p.shape[0], bool)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                w = (((((a[:, 0] if dx else 256 - a[:, 0]) * (a[:, 2] if dz else 256 - a[:, 2]) + 128) >> 8)
                      * (a[:, 1] if dy else 256 - a[:, 1])) + 128) >> 8
                occ |= (w > 0) & g[np.clip(i0[:, 2] + dz, 0, c), np.clip(i0[:, 1] + dy, 0, c), np.clip(i0[:, 0] + dx, 0, c)]
    return occ


def brute_march(o, d, aabb, grid, sequential=True, bisections=5, clamp_hi=None):
    """One ray, from the contract: march t_0 = tmin, t_k+1 = t_k + step (fp32) to the first t_k that is not below the
    box exit or is occupied; if that is before the exit, bisect `bisections` times from -step/2, halving, towards the
    surface; then march back from the exit by t -= step to the first t_k not above tmin or occupied."""
    tmin, tend = (v[0] for v in S.aabb_minmax(o[None], d[None], aabb))
    G = grid.shape[0]
    step = f32(0.5) / f32(G)

    def occ(ts):
        ts = np.asarray(ts, f32)
        with np.errstate(invalid="ignore"):  # rejected rays (tmin NaN) look up NaN once, as the kernel does
            p = (S.fma32(np.broadcast_to(d, (ts.size, 3)), ts[:, None], np.broadcast_to(o, (ts.size, 3))) + f32(0.5))
            return _tex(grid, p.astype(f32), clamp_hi)

    def march(t0, go, sign):
        ts, t, k = [], t0, 0
        while True:
            ts.append(t)
            if not go(t):
                break
            k += 1
            t = f32(t + sign * step) if sequential else f32(S.fma32(f32(k), f32(sign * step), t0))
        ts = np.array(ts, f32)
        stop = ~np.array([go(t) for t in ts]) | occ(ts)
        return ts[np.argmax(stop)]

    tmin = march(tmin, lambda t: t < tend, 1)
    if tmin < tend:
        ref = f32(-step * f32(0.5))
        for _ in range(bisections):
            tmin = f32(tmin + ref)
            mag = f32(abs(ref) * f32(0.5))
            ref = -mag if occ([tmin])[0] else mag
    tmax = march(tend, lambda t: t > tmin, -1)
    return tmin, tmax


def march_mismatches(case, limit=400, **mutation):
    sc = case.scene
    o, d, img = _rays(case)
    sel = np.random.default_rng(3).permutation(o.shape[0])[:limit]
    tmin, tmax = S.occupancy_minmax(o[sel], d[sel], sc["aabb"], sc["grids"], img[sel], sc["G"])
    bad = 0
    for j, r in enumerate(sel):
        a, b = brute_march(o[r], d[r], sc["aabb"], sc["grids"][img[r]], **mutation)
        bad += not (_bits_equal(a, tmin[j]) and _bits_equal(b, tmax[j]))
    return bad


@pytest.mark.parametrize("name", list(CPU_FAMILIES))
def test_march_contract(name):
    case = _case(name)
    assert march_mismatches(case) == 0


def test_placed_first_hits():
    """The placed family's rays stop after the chosen numbers of march moves, counted by the scalar march."""
    case = _case("placed")
    sc = case.scene
    o, d, img = _rays(case)
    nf, nb = SC.march_indices(o, d, sc["aabb"], sc["grids"], img, sc["G"])
    for t in SC.LANE_TARGETS:
        assert (nf == t).any() and (nb == t).any(), t


# -------------------------------------------------------------------------------------------------------------- samples
def emit(mm, o, d, img, grids, step, occupancy, inclusive=False):
    """Per kept ray j, from the contract: candidates t_k = fma(k, step, tmin) for k < int(fl(tmax - tmin)·fl(1/step)),
    the occupied ones in order, written at the exclusive scan of the per-ray counts (the inclusive scan if asked)."""
    inv = f32(1.0) / f32(step)
    per = []
    for j in range(mm.shape[0]):
        cand = max(int(f32(f32(mm[j, 1] - mm[j, 0]) * inv)), 0)
        t = S.fma32(np.arange(cand, dtype=f32), f32(step), mm[j, 0]) if cand else np.zeros(0, f32)
        if occupancy and cand:
            p = (S.fma32(np.broadcast_to(d[j], (cand, 3)), t[:, None], np.broadcast_to(o[j], (cand, 3))) + f32(0.5))
            t = t[S.tex_occupied(grids[img[j]], p.astype(f32))]
        per.append(t)
    counts = np.array([t.size for t in per], np.int64)
    total = int(counts.sum())
    off = np.cumsum(counts) - (0 if inclusive else counts)
    dist, rel = np.zeros(total, f32), np.zeros(total, np.int32)
    for j, t in enumerate(per):
        k = np.arange(off[j], off[j] + t.size)
        k = k[k < total]
        dist[k], rel[k] = t[:k.size], j
    return dist, rel


def sample_mismatches(case, occupancy, inclusive=False):
    sc = case.scene
    bad = 0
    for step in case.steps:
        out = S.get_data(sc["rgba"], sc["light_mask"], sc["frame_numbers"], sc["camera_numbers"], sc["grids"],
                         sc["landscape"], case.idx, sc["inverse_krs"], sc["camera_origins"], sc["aabb"], sc["G"], SC.W,
                         SC.H, step, False, occupancy=occupancy)
        o, d, mm, dist, rel = out[0], out[1], out[5], out[7], out[8]
        img = case.idx[out[6]] // (SC.W * SC.H)
        e_dist, e_rel = emit(mm, o, d, img, sc["grids"], step, occupancy, inclusive)
        bad += not (_bits_equal(dist, e_dist) and np.array_equal(rel, e_rel))
        if not inclusive:  # every distance is a candidate of its ray inside [tmin, tmax), strictly increasing
            assert (dist >= mm[rel, 0]).all() and (dist < mm[rel, 1]).all()
            same = rel[1:] == rel[:-1]
            assert (dist[1:][same] > dist[:-1][same]).all() and (np.diff(rel) >= 0).all()
    return bad


@pytest.mark.parametrize("occupancy", [False, True])
@pytest.mark.parametrize("name", ["axis", "origin", "graze", "ring", "placed", "counts"])
def test_sample_contract(name, occupancy):
    case = _case(name)
    if name == "counts" and not occupancy:
        assert SC.count_check(case) == list(SC.COUNT_TARGETS)
    assert sample_mismatches(case, occupancy) == 0


# -------------------------------------------------------------------------------------------------------------- mutants
def _lookup_points(G, rng):
    faces = np.array([0.0, 1.0], f32)
    near = np.concatenate([faces, np.nextafter(faces, f32(-1)), np.nextafter(faces, f32(2)),
                           rng.uniform(-0.3, 0, 20).astype(f32), rng.uniform(1, 1.3, 20).astype(f32)])
    p = rng.uniform(0, 1, (4000, 3)).astype(f32)
    for k in range(3):
        p[k * 1000:(k + 1) * 1000, k] = rng.choice(near, 1000)
    return p


def lookup_mismatches(clamp_hi_of_G):
    rng = np.random.default_rng(9)
    bad = 0
    for G in (1, 3, 33):
        g = SC.pattern("corners", G)
        p = _lookup_points(G, rng)
        bad += int((_tex(g, p, clamp_hi_of_G(G)) != S.tex_occupied(g, p)).sum())
    return bad


def test_tex_restatement_matches_oracle():
    assert lookup_mismatches(lambda G: G - 1) == 0


def test_bars_see_bugs(monkeypatch):
    """Each named mutant changes at least one output on the edge cases; prints the families that catch it."""
    caught = {m: [] for m in ("glm ternaries -> np.minimum/np.maximum", "t0 + k*step march", "4 bisection steps",
                              "portrait w/h swap dropped", "inclusive sample scan", "filter clamp at G")}
    for name in CPU_FAMILIES:
        case = _case(name)
        with monkeypatch.context() as m:
            m.setattr(S, "_gmin", np.minimum)
            m.setattr(S, "_gmax", np.maximum)
            if slab_violations(case)[0]:
                caught["glm ternaries -> np.minimum/np.maximum"].append(name)
        if march_mismatches(case, 150, sequential=False):
            caught["t0 + k*step march"].append(name)
        if march_mismatches(case, 150, bisections=4):
            caught["4 bisection steps"].append(name)
        if pixel_violations(case, np.ones_like(case.scene["landscape"]))[0] > 0.5:
            caught["portrait w/h swap dropped"].append(name)
        if name != "miss" and sample_mismatches(SC.Case(name, case.scene, case.idx, case.steps[:1]), True, True):
            caught["inclusive sample scan"].append(name)
        if march_mismatches(case, 150, clamp_hi=case.scene["G"]):
            caught["filter clamp at G"].append(name)
    if lookup_mismatches(lambda G: G):
        caught["filter clamp at G"].append("lookup points on and outside the faces")
    for m, fams in caught.items():
        print(f"{m:42s} caught by: {', '.join(fams) if fams else 'NOTHING'}")
    assert all(caught.values()), caught
