"""Geometry scores on the H100 (csrc/mesh_distance.cu, toolbox/geometry_metrics.py): samples and per-sample distances
against the numpy oracle bit for bit, reductions, determinism, analytic geometry, rejection, and evaluate_geometry on
the confined teacher."""
import csv
import math

import numpy as np
import pytest
import torch

import geometry_oracle as O

pytestmark = pytest.mark.gpu

TAUS = (0.001, 0.01, 0.1, 0.5)


def _mesh(V, F, dev):
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    return Mesh(torch.from_numpy(np.ascontiguousarray(V, np.float32)).to(dev),
                torch.from_numpy(np.ascontiguousarray(F, np.int32)).to(dev))


def _run(Vs, Fs, Vt, Ft, n, seed, dev, taus=TAUS):
    from humanrf_b200.toolbox.geometry_metrics import mesh_distance

    out, counts, err, s = mesh_distance(_mesh(Vs, Fs, dev), _mesh(Vt, Ft, dev), n, seed, taus, per_sample=True)
    torch.cuda.synchronize()
    return (out.cpu().numpy(), counts.cpu().numpy(), int(err.cpu()[0]), {k: v.cpu().numpy() for k, v in s.items()})


def _same_bits(x, y):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    return x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))


def _with_degenerate(V, F, rng):
    """F plus zero-area faces: repeated indices, collinear and coincident vertices."""
    nv = len(V)
    extra_v = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2], [0.5, 0.5, 0.5]], np.float32)
    V = np.concatenate([V, extra_v])
    deg = np.array([[nv, nv + 1, nv + 2], [nv, nv, nv + 3], [3, 3, 3], [nv + 3, nv + 3, nv]], np.int32)
    F = np.concatenate([F[:len(F) // 2], deg, F[len(F) // 2:]])
    return V, F


SAMPLE_CASES = {
    "six-decades": lambda rng: O.random_mesh(3001, 0, decades=6) + (5003,),
    "degenerate": lambda rng: _with_degenerate(*O.random_mesh(1000, 1, decades=3), rng) + (4097,),
    "single-face": lambda rng: (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.5]], np.float32),
                                np.array([[0, 1, 2]], np.int32), 777),
    "n1": lambda rng: O.random_mesh(513, 2) + (1,),
}


@pytest.mark.parametrize("case", list(SAMPLE_CASES))
def test_samples_match_oracle_bitwise(cuda, case):
    rng = np.random.default_rng(0)
    V, F, n = SAMPLE_CASES[case](rng)
    for seed in (0, 12345):
        _, _, err, s = _run(V, F, V, F, n, seed, cuda)
        p, f = O.sample(V, F, n, seed)
        assert err == 0
        assert np.array_equal(s["faces"], f)
        assert _same_bits(s["points"], p), int((s["points"] != p).any(1).sum())
        elig, _, _ = O.face_info(V, F)
        assert elig[s["faces"]].all()


def _far_case():
    Vt, Ft = O.random_mesh(3000, 3, decades=2)
    Vs, Fs = O.random_mesh(2000, 4, decades=1)
    Vs = Vs * np.float32(30) + np.float32(50)         # far outside the target's box
    return Vs, Fs, Vt, Ft


def _duplicate_case():
    Vt, Ft = O.random_mesh(1500, 5, decades=2)
    Ft = np.concatenate([Ft, Ft[::-1], Ft[::7]])       # coincident duplicates, later ids
    Vs, Fs = O.random_mesh(2000, 6, decades=2)
    return Vs, Fs, Vt, Ft


DIST_CASES = {
    "random": lambda: O.random_mesh(3000, 7, decades=3) + O.random_mesh(3000, 8, decades=3),
    "far": _far_case,
    "self": lambda: O.random_mesh(3000, 9, decades=3) * 2,
    "duplicates": _duplicate_case,
    "degenerate-target": lambda: O.random_mesh(2000, 10) + _with_degenerate(*O.random_mesh(3000, 11), None),
}


@pytest.mark.parametrize("case", list(DIST_CASES))
def test_distances_match_bruteforce_bitwise(cuda, case):
    Vs, Fs, Vt, Ft = DIST_CASES[case]()
    n = 5000
    out, counts, err, s = _run(Vs, Fs, Vt, Ft, n, 3, cuda)
    d, g = O.closest(s["points"], Vt, Ft)
    assert err == 0
    assert np.array_equal(s["closest"], g), int((s["closest"] != g).sum())
    assert _same_bits(s["distances"], d)
    if case == "self":
        # a sample's distance to its own face: the point's rounding plus the routine's bound (DESIGN §3.11)
        f = Fs[s["faces"]].astype(np.int64)
        A, B, C, P = (np.asarray(x, np.float64) for x in (Vs[f[:, 0]], Vs[f[:, 1]], Vs[f[:, 2]], s["points"]))
        L = np.maximum.reduce([np.linalg.norm(B - A, axis=1), np.linalg.norm(C - A, axis=1),
                               np.linalg.norm(C - B, axis=1)])
        h = np.linalg.norm(np.cross(B - A, C - A), axis=1) / L
        bound = 4 * 2.0 ** -24 * (np.linalg.norm(P - A, axis=1) + L) * (1 + L / h) + 2.0 ** -20 * np.abs(P).max(1)
        assert (s["distances"] <= bound).all()
    if case == "duplicates":
        assert (s["closest"] < 1500).all()
    # reductions: the fp64 sums against an fp64 sum of the per-sample outputs, the counts exactly
    ref, ref_counts, _ = O.direction(Vs, Fs, Vt, Ft, n, 3, TAUS)
    dd = s["distances"].astype(np.float64)
    _, ns, _ = O.face_info(Vs, Fs)
    _, nt, _ = O.face_info(Vt, Ft)
    nterm = np.abs(O._dot(ns[s["faces"]], nt[s["closest"]])).astype(np.float64)
    for k, x in enumerate((dd, dd * dd, nterm)):
        assert abs(out[k] * n - x.sum()) <= n * 2.0 ** -53 * np.abs(x).sum() * 2, (k, out[k], x.sum() / n)
        assert abs(out[k] - ref[k]) <= n * 2.0 ** -53 * np.abs(x).sum() / n * 2
    assert np.array_equal(counts, ref_counts)


def _bench_meshes(dev):
    """The bench model's G = 256 make_scene hull mesh (mesh_bench.py's workload) for two frames."""
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.mesh_extraction import density_lattice, marching_cubes

    model, frames = make_model((50,), seed=123, device=dev)
    hull = torch.from_numpy(np.ascontiguousarray(make_scene(num_images=1, G=256)["grids"][0])).to(dev)
    lat = density_lattice(model, frames[0], hull)
    level = float(torch.median(lat[lat != 0]))
    return (marching_cubes(lat, level, normals=False),
            marching_cubes(density_lattice(model, frames[5], hull), level, normals=False))


def _exact_distance_torch(p, a, b, c):
    """fp64 point-triangle distance on the device for a prefilter: [m,3] points against [F,3] triangles -> [m,F]."""
    p = p[:, None, :]

    def dot(x, y):
        return (x * y).sum(-1)

    def seg(x, y):
        d = y - x
        t = (dot(p - x, d) / dot(d, d).clamp_min(1e-300)).clamp(0, 1)
        return (p - (x + t[..., None] * d)).norm(dim=-1)

    n = torch.linalg.cross(b - a, c - a)
    nn = dot(n, n)
    s = dot(p - a, n) / nn
    proj = p - s[..., None] * n
    inside = ((dot(torch.linalg.cross((b - a).expand_as(proj), proj - a), n) >= 0)
              & (dot(torch.linalg.cross((c - b).expand_as(proj), proj - b), n) >= 0)
              & (dot(torch.linalg.cross((a - c).expand_as(proj), proj - c), n) >= 0))
    best = torch.minimum(torch.minimum(seg(a, b), seg(b, c)), seg(c, a))
    return torch.where(inside, torch.minimum(s.abs() * nn.sqrt(), best), best)


def test_large_marching_cubes_mesh_against_bruteforce(cuda):
    """~2 M faces: 512 random samples checked against every face.  An fp64 prefilter keeps the faces within
    2 * (largest face box diagonal) + 1e-5 of the nearest (the fp32 routine's point stays in its face's box, so no face
    outside can win or tie), then the numpy fp32 routine decides among them."""
    from humanrf_b200.toolbox.geometry_metrics import mesh_distance

    src, dst = _bench_meshes(cuda)
    assert dst.faces.shape[0] > 1_500_000
    n = 200_000
    _, _, err, s = mesh_distance(src, dst, n, 11, TAUS, per_sample=True)
    assert int(err.cpu()[0]) == 0
    Vt, Ft = dst.vertices.cpu().numpy(), dst.faces.cpu().numpy()
    elig, _, _ = O.face_info(Vt, Ft)
    ids = np.nonzero(elig)[0]
    tri = dst.vertices.double()[dst.faces[torch.from_numpy(ids).to(cuda)].long()]       # [E,3,3]
    a, b, c = tri[:, 0][None], tri[:, 1][None], tri[:, 2][None]
    diag = float((tri.amax(1) - tri.amin(1)).norm(dim=-1).max())
    pick = np.random.default_rng(0).choice(n, 512, replace=False)
    pts = s["points"][torch.from_numpy(pick).to(cuda)]
    got_d, got_f = s["distances"].cpu().numpy()[pick], s["closest"].cpu().numpy()[pick]
    for k in range(0, 512, 8):
        d64 = torch.cat([_exact_distance_torch(pts[k:k + 8].double(), a[:, j:j + 262144], b[:, j:j + 262144],
                                               c[:, j:j + 262144]) for j in range(0, len(ids), 262144)], 1)
        dmin = d64.min(1, keepdim=True).values
        cand = (d64 <= dmin + 2 * diag + 1e-5).cpu().numpy()
        for r in range(cand.shape[0]):
            cid = ids[cand[r]]
            p = pts[k + r].cpu().numpy()
            d2 = O.point_triangle_d2(p[None], Vt[Ft[cid, 0]], Vt[Ft[cid, 1]], Vt[Ft[cid, 2]])
            j = int(np.argmin(d2))                 # candidates are in increasing id order: ties to the lowest
            assert got_f[k + r] == cid[j], (k + r, got_f[k + r], cid[j])
            assert _same_bits(got_d[k + r], np.sqrt(d2[j]))


def test_determinism_and_graph_replay(cuda):
    from humanrf_b200.toolbox.geometry_metrics import mesh_distance

    Vs, Fs = O.random_mesh(3000, 12, decades=4)
    Vt, Ft = O.random_mesh(2500, 13, decades=4)
    src, dst = _mesh(Vs, Fs, cuda), _mesh(Vt, Ft, cuda)
    a = mesh_distance(src, dst, 100_003, 5, TAUS, per_sample=True)
    b = mesh_distance(src, dst, 100_003, 5, TAUS, per_sample=True)
    out = torch.empty(3, dtype=torch.float64, device=cuda)
    mesh_distance(src, dst, 100_003, 5, TAUS, out=out)          # warm-up outside capture
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            c = mesh_distance(src, dst, 100_003, 5, TAUS, out=out, per_sample=True)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(0)
    c[3]["distances"].fill_(0)
    g.replay()
    torch.cuda.synchronize()
    for x, y, z in ((a[0], b[0], c[0]), (a[1], b[1], c[1]), (a[2], b[2], c[2])):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)) and torch.equal(x.view(torch.uint8), z.view(torch.uint8))
    for k in a[3]:
        assert torch.equal(a[3][k].view(torch.uint8), b[3][k].view(torch.uint8))
        assert torch.equal(a[3][k].view(torch.uint8), c[3][k].view(torch.uint8))


@pytest.mark.parametrize("delta", [0.01, 0.05])
def test_icospheres(cuda, delta):
    from humanrf_b200.toolbox.geometry_metrics import compare_meshes

    r = 1.0
    V1, F1 = O.icosphere(5, r)
    V2, F2 = O.icosphere(5, r + delta)
    gap = max(O.sphere_tessellation_gap(V1, F1, r), O.sphere_tessellation_gap(V2, F2, r + delta))
    sc = compare_meshes(_mesh(V1, F1, cuda), _mesh(V2, F2, cuda), num_samples=200_000, taus=(delta / 2, 2 * delta))
    for x in (sc.accuracy, sc.completeness):
        assert delta - gap - 1e-6 <= x <= delta + gap + 1e-6, (x, delta, gap)
    assert sc.fscore[1] == 1.0 and sc.fscore[0] == 0.0
    assert sc.normal_consistency >= 1 - 1e-3
    same = compare_meshes(_mesh(V1, F1, cuda), _mesh(V1, F1, cuda), num_samples=100_000, taus=(1e-5,))
    assert same.fscore == (1.0,) and same.precision == (1.0,) and same.recall == (1.0,)
    assert same.normal_consistency >= 1 - 1e-6 and same.accuracy <= 1e-6


def test_rejects_and_nan(cuda):
    from humanrf_b200.toolbox.geometry_metrics import compare_meshes, mesh_distance
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    V, F = O.random_mesh(100, 14)
    good = _mesh(V, F, cuda)
    bad = [Mesh(good.vertices.cpu(), good.faces.cpu()), Mesh(good.vertices.double(), good.faces),
           Mesh(good.vertices, good.faces.long()), Mesh(good.vertices[:, :2].contiguous(), good.faces),
           Mesh(good.vertices.t(), good.faces), "not a mesh"]
    for m in bad:
        with pytest.raises(RuntimeError):
            mesh_distance(m, good, 10, 0)
        with pytest.raises(RuntimeError):
            mesh_distance(good, m, 10, 0)
    for n in (0, -1, 2 ** 31):
        with pytest.raises(RuntimeError):
            mesh_distance(good, good, n, 0)
    with pytest.raises(RuntimeError):
        mesh_distance(good, good, 10, 0, taus=tuple(range(9)))
    # out-of-range indices: NaN, the error word, no fault
    for F_bad in (np.concatenate([F, [[0, 1, 10 ** 6]]]), np.concatenate([F, [[-5, 1, 2]]])):
        for src_bad in (True, False):
            m_bad = _mesh(V, F_bad, cuda)
            out, counts, err, s = mesh_distance(m_bad if src_bad else good, good if src_bad else m_bad, 1000, 0,
                                                per_sample=True)
            torch.cuda.synchronize()
            assert int(err.cpu()[0]) == (1 if src_bad else 2)
            assert torch.isnan(out).all() and (counts == -1).all()
            with pytest.raises(RuntimeError, match="outside the vertex range"):
                compare_meshes(m_bad, good, 1000) if src_bad else compare_meshes(good, m_bad, 1000)
    # empty and all-degenerate meshes: NaN
    empty = Mesh(torch.zeros((0, 3), device=cuda), torch.zeros((0, 3), dtype=torch.int32, device=cuda))
    flat = _mesh(np.zeros((3, 3), np.float32), np.array([[0, 1, 2], [0, 0, 0]], np.int32), cuda)
    for a, b in ((empty, good), (good, empty), (flat, good), (good, flat)):
        out, counts, err, s = mesh_distance(a, b, 100, 0, per_sample=True)
        torch.cuda.synchronize()
        assert int(err.cpu()[0]) == 0 and torch.isnan(out).all() and (counts == -1).all()
        sc = compare_meshes(a, b, 100)
        assert math.isnan(sc.accuracy) and math.isnan(sc.fscore[0])


RADII = np.array([0.2, 0.3, 0.15])


def test_evaluate_geometry_confined_teacher(cuda, tmp_path):
    """The reference OBJs are an icosphere scaled to the teacher's ellipsoid E, in world units.  The learned mesh lies
    within sqrt(3) / scale0 + 1/G of E (§3.6), the reference within its tessellation gap, so both mean distances stay
    below the sum (converted to world units)."""
    from test_learned_occupancy_gpu import _sphere, confined_teacher

    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.geometry_metrics import csv_columns, evaluate_geometry
    from humanrf_b200.toolbox.mesh_extraction import Mesh, scene_normalisation, to_world, write_obj

    m = confined_teacher(cuda)
    G = 64
    ds = SyntheticDataset(G=G)
    ds._grids = {f: _sphere(G) for f in ds.frames}
    offset, scale = scene_normalisation(ds)
    Vu, Fu = O.icosphere(5, 1.0)
    gap = O.sphere_tessellation_gap(Vu, Fu, 1.0) * RADII.max()
    ref = to_world(Mesh(torch.from_numpy((Vu * RADII).astype(np.float32)).to(cuda), torch.from_numpy(Fu).to(cuda)),
                   offset, scale)
    refdir = tmp_path / "ref"
    refdir.mkdir()
    frames = (15, 16)
    for f in frames:
        write_obj(refdir / f"Frame{f:06d}.obj", ref)
    scale0 = float(m.feature_grids[0].layout.scale[0])
    band = (np.sqrt(3) / scale0 + 1 / G + gap) / scale
    taus = (0.005, 0.01, 2 * band)
    scores = evaluate_geometry(m, ds, frames, refdir, tmp_path / "out", 100.0, num_samples=200_000, taus=taus)
    assert [s.frame for s in scores] == list(frames)
    for s in scores:
        assert 0 < s.accuracy <= band and 0 < s.completeness <= band, (s.accuracy, s.completeness, band)
        assert s.normal_consistency > 0.9 and s.fscore[-1] >= 0.999
    rows = list(csv.reader(open(tmp_path / "out" / "geometry.csv")))
    assert rows[0] == csv_columns(taus) and [int(r[0]) for r in rows[1:]] == list(frames)
    assert float(rows[1][1]) == scores[0].accuracy
    avg = list(csv.reader(open(tmp_path / "out" / "geometry_averages.csv")))
    assert avg[0] == rows[0][1:] and float(avg[1][0]) == pytest.approx(np.mean([s.accuracy for s in scores]))
    print(f"confined teacher: accuracy {[s.accuracy for s in scores]} completeness {[s.completeness for s in scores]} "
          f"band {band:.5f} (world units)")
    # a missing reference file is found before any work, and nothing is written
    with pytest.raises(RuntimeError, match="missing reference meshes"):
        evaluate_geometry(m, ds, (15, 17), refdir, tmp_path / "missing", 100.0, num_samples=1000)
    assert not (tmp_path / "missing").exists()
    with pytest.raises(RuntimeError):
        evaluate_geometry(m, ds, (15, 99), refdir, tmp_path / "badframe", 100.0, num_samples=1000)
    # a level above every density: empty meshes, NaN scores, named frames
    with pytest.raises(RuntimeError, match=r"no geometry score for frames \[15, 16\]"):
        evaluate_geometry(m, ds, frames, refdir, tmp_path / "empty", 1e30, num_samples=1000)
    assert not (tmp_path / "empty" / "geometry.csv").exists()
