"""Geometry scores without a GPU: the fp32 closest-point routine of tests/geometry_oracle.py (the kernel's, restated)
against fp64 distances within DESIGN §3.11's bound, the sampling's distribution, the scores on hand cases, read_obj and
the CSV layout, and three deliberately wrong oracles that the GPU bars must reject."""
import csv

import numpy as np
import pytest
import torch
from scipy import stats

import geometry_oracle as O

U = 2.0 ** -24


def _bound(p, a, b, c):
    """DESIGN §3.11: |d_fp32 - d| <= 4 u (R + L)(1 + L / h), R = |p - a|, L the longest edge, h = |n| / L."""
    A, B, C, P = (np.asarray(x, np.float64) for x in (a, b, c, p))
    L = np.maximum.reduce([np.linalg.norm(B - A, axis=-1), np.linalg.norm(C - A, axis=-1),
                           np.linalg.norm(C - B, axis=-1)])
    h = np.linalg.norm(np.cross(B - A, C - A), axis=-1) / L
    return 4 * U * (np.linalg.norm(P - A, axis=-1) + L) * (1 + L / h)


def _check_routine(p, a, b, c):
    p, a, b, c = (np.asarray(x, np.float32) for x in np.broadcast_arrays(p, a, b, c))
    d32 = np.sqrt(O.point_triangle_d2(p, a, b, c).astype(np.float64))
    d64 = O.exact_distance(p, a, b, c)
    err, bound = np.abs(d32 - d64), _bound(p, a, b, c)
    assert (err <= bound).all(), float((err / bound).max())
    return O.region(p, a, b, c)


def test_routine_every_voronoi_region():
    rng = np.random.default_rng(0)
    a, b, c = np.array([0, 0, 0], np.float32), np.array([1, 0, 0], np.float32), np.array([0.3, 0.8, 0], np.float32)
    # one point per region by construction, lifted off the plane
    pts = np.array([[-0.5, -0.5, 0.2], [1.5, -0.3, -0.1], [0.5, -0.5, 0.3], [0.2, 1.5, 0.1], [-0.4, 0.5, -0.2],
                    [1.0, 0.8, 0.4], [0.4, 0.3, 0.5]], np.float32)
    assert list(_check_routine(pts, a, b, c)) == list(range(7))
    p = rng.normal(size=(200000, 3)).astype(np.float32) * 2
    T = rng.normal(size=(200000, 3, 3)).astype(np.float32)
    reg = _check_routine(p, T[:, 0], T[:, 1], T[:, 2])
    assert (np.bincount(reg, minlength=7) > 1000).all()


def test_routine_on_vertices_and_edges_is_exact_there():
    rng = np.random.default_rng(1)
    T = rng.normal(size=(5000, 3, 3)).astype(np.float32)
    for k in range(3):
        d2 = O.point_triangle_d2(T[:, k], T[:, 0], T[:, 1], T[:, 2])
        assert (d2 == 0).all()
    t = rng.uniform(0, 1, (5000, 1))
    for i, j in ((0, 1), (1, 2), (2, 0)):
        p = (T[:, i] + t * (T[:, j] - T[:, i])).astype(np.float32)
        _check_routine(p, T[:, 0], T[:, 1], T[:, 2])


def test_routine_slivers_and_far_points():
    rng = np.random.default_rng(2)
    n = 100000
    a = rng.normal(size=(n, 3))
    b = a + rng.normal(size=(n, 3))
    c = a + (b - a) * rng.uniform(0, 1, (n, 1)) + 10 ** rng.uniform(-6, -2, (n, 1)) * rng.normal(size=(n, 3))
    p = a + 3 * rng.normal(size=(n, 3))
    a, b, c, p = (x.astype(np.float32) for x in (a, b, c, p))
    elig, _, _ = O.face_info(np.stack([a, b, c], 1).reshape(-1, 3), np.arange(3 * n).reshape(-1, 3))
    _check_routine(p[elig], a[elig], b[elig], c[elig])
    _check_routine((a + 1e3 * rng.normal(size=(n, 3))).astype(np.float32), a, b, c)


def test_degenerate_faces_are_ineligible():
    V = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0], [0, 0, 0]], np.float32)
    F = np.array([[0, 1, 2], [0, 1, 3], [0, 0, 3], [0, 4, 3], [0, 1, 5], [-1, 1, 3]], np.int32)
    elig, unit, area = O.face_info(V, F)
    assert list(elig) == [False, True, False, False, False, False]
    assert area[1] == np.float32(0.5) and np.array_equal(unit[1], np.array([0, 0, 1], np.float32))
    assert list(O.weights(area, elig)) == [0, 2 ** 32, 0, 0, 0, 0]


def test_sampling_follows_weights_and_skips_zero_weight_faces():
    V, F = O.random_mesh(40, seed=3, decades=2)
    F = np.concatenate([F, np.array([[0, 0, 1], [5, 5, 5]], np.int32)])     # two degenerate faces
    elig, _, area = O.face_info(V, F)
    q = O.weights(area, elig).astype(np.float64)
    n = 400000
    p, f = O.sample(V, F, n, seed=7)
    assert (f < 40).all() and (f >= 0).all()
    counts = np.bincount(f, minlength=len(F))
    e = q / q.sum() * n
    keep = e > 0
    chi2 = float((((counts - e) ** 2)[keep] / e[keep]).sum())
    dof = int(keep.sum()) - 1
    assert chi2 < stats.chi2.ppf(1 - 1e-6, dof), (chi2, dof)
    assert counts[~keep].sum() == 0
    # points lie on their faces (fp32 barycentric combination: within a few ulps of the plane and inside the box)
    a, b, c = V[F[f, 0]], V[F[f, 1]], V[F[f, 2]]
    assert (O.exact_distance(p, a, b, c) <= 1e-5).all()


def test_splitmix_and_mulhi():
    assert int(O.splitmix64(np.array([0], np.uint64))[0]) == 0xE220A8397B1DCDAF   # SplitMix64's first output for seed 0
    rng = np.random.default_rng(4)
    a = rng.integers(0, 2 ** 63, 1000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    b = rng.integers(0, 2 ** 63, 1000, dtype=np.uint64)
    assert all(int(h) == (int(x) * int(y)) >> 64 for h, x, y in zip(O.mulhi64(a, b), a, b))


def _parallel_squares(delta):
    V = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
    F = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    V2 = V.copy()
    V2[:, 2] = np.float32(delta)
    return V, F, V2, F


@pytest.mark.parametrize("delta", [0.0, 0.25, 0.75])
def test_scores_parallel_squares(delta):
    """Every distance is delta up to the routine's bound (the sample point's in-plane rounding), the normals agree
    exactly, and F is 1 exactly for the thresholds at or above delta."""
    V, F, V2, F2 = _parallel_squares(delta)
    taus = (0.1, 0.5)
    n = 500
    fwd, cf, sf = O.direction(V, F, V2, F2, n, 0, taus)
    bwd, cb, sb = O.direction(V2, F2, V, F, n, 0, taus)
    tol = 4 * U * (2 + 2 ** 0.5) * 3          # R <= |p - a| <= 2, L = sqrt(2), L / h = 2
    for s in (sf, sb):
        assert np.abs(s["distances"].astype(np.float64) - delta).max() <= tol
    acc, comp, l1, l2, nc, P, R, Fs = O.scores(fwd, bwd, cf, cb, n)
    assert abs(acc - delta) <= tol and abs(comp - delta) <= tol and abs(l2 - delta ** 2) <= 3 * tol
    assert nc == 1.0
    assert Fs == [1.0 if delta <= t else 0.0 for t in taus]


def test_f_score_zero_when_nothing_is_close():
    assert O.fscore(0.0, 0.0) == 0.0 and O.fscore(1.0, 1.0) == 1.0 and O.fscore(0.5, 1.0) == pytest.approx(2 / 3)


# ---------------------------------------------------------------- read_obj / write_obj / tables
def _mesh(V, F, colors=None):
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    return Mesh(torch.from_numpy(V), torch.from_numpy(F), None, None if colors is None else torch.from_numpy(colors))


@pytest.mark.parametrize("colors", [False, True])
def test_read_obj_round_trips_write_obj(tmp_path, colors):
    from humanrf_b200.toolbox.geometry_metrics import read_obj
    from humanrf_b200.toolbox.mesh_extraction import write_obj

    rng = np.random.default_rng(5)
    V = (rng.normal(size=(500, 3)) * 10.0 ** rng.uniform(-8, 8, (500, 1))).astype(np.float32)
    F = rng.integers(0, 500, (900, 3)).astype(np.int32)
    col = rng.uniform(0, 1, (500, 3)).astype(np.float32) if colors else None
    write_obj(tmp_path / "m.obj", _mesh(V, F, col))
    m = read_obj(tmp_path / "m.obj", device="cpu")
    assert np.array_equal(m.vertices.numpy().view(np.int32), V.view(np.int32))
    assert np.array_equal(m.faces.numpy(), F) and m.faces.dtype == torch.int32
    assert (m.colors is not None) == colors
    if colors:
        assert np.array_equal(m.colors.numpy(), col)


def test_read_obj_accepts_slash_forms_and_ignores_other_lines(tmp_path):
    from humanrf_b200.toolbox.geometry_metrics import read_obj

    (tmp_path / "m.obj").write_text("# comment\nmtllib x.mtl\no body\nv 0 0 0\nv 1 0 0\nvt 0 0\nvn 0 0 1\nv 0 1 0\n"
                                    "v 1 1 0\ns off\nf 1/1/1 2/1/1 3/1/1\nf 2//1 4//1 3//1\nusemtl m\nf 1/2 2/2 4/2\n")
    m = read_obj(tmp_path / "m.obj", device="cpu")
    assert m.vertices.shape == (4, 3)
    assert m.faces.tolist() == [[0, 1, 2], [1, 3, 2], [0, 1, 3]]


@pytest.mark.parametrize("bad,what", [("f 1 2 3 4", "triangles"), ("f 0 1 2", "outside"), ("f -1 2 3", "outside"),
                                      ("f 1 2 9", "outside"), ("f 1 2", "triangles"), ("f 1 x 2", "integers")])
def test_read_obj_rejects(tmp_path, bad, what):
    from humanrf_b200.toolbox.geometry_metrics import read_obj

    path = tmp_path / "bad.obj"
    path.write_text(f"v 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 0\nf 1 2 3\n{bad}\n")
    with pytest.raises(RuntimeError, match=f"bad.obj:6: .*{what}"):
        read_obj(path, device="cpu")


def test_read_obj_rejects_files_without_faces(tmp_path):
    from humanrf_b200.toolbox.geometry_metrics import read_obj

    path = tmp_path / "empty.obj"
    path.write_text("v 0 0 0\nv 1 0 0\n")
    with pytest.raises(RuntimeError, match="empty.obj: no faces"):
        read_obj(path, device="cpu")


def test_tables_layout(tmp_path):
    from humanrf_b200.toolbox.geometry_metrics import GeometryScore, csv_columns, scores_from, write_geometry_tables

    assert csv_columns((0.005, 0.01)) == ["frame", "accuracy", "completeness", "chamfer_l1", "chamfer_l2",
                                          "normal_consistency", "precision@0.005", "recall@0.005", "fscore@0.005",
                                          "precision@0.01", "recall@0.01", "fscore@0.01"]
    a = scores_from([0.1, 0.02, 0.9], [0.3, 0.1, 0.7], [50, 100], [0, 100], 100, (0.005, 0.01), frame=3)
    assert isinstance(a, GeometryScore)
    assert (a.accuracy, a.completeness, a.chamfer_l1, a.chamfer_l2) == (0.1, 0.3, 0.2, (0.02 + 0.1) / 2)
    assert a.normal_consistency == pytest.approx(0.8)
    assert a.precision == (0.5, 1.0) and a.recall == (0.0, 1.0) and a.fscore == (0.0, 1.0)
    b = scores_from([0.2, 0.05, 0.5], [0.1, 0.01, 0.5], [100, 100], [100, 100], 100, (0.005, 0.01), frame=4)
    write_geometry_tables(tmp_path, [a, b])
    rows = list(csv.reader(open(tmp_path / "geometry.csv")))
    assert rows[0] == csv_columns((0.005, 0.01))
    assert [int(r[0]) for r in rows[1:]] == [3, 4] and float(rows[1][1]) == 0.1 and float(rows[2][9]) == 1.0
    avg = list(csv.reader(open(tmp_path / "geometry_averages.csv")))
    assert avg[0] == rows[0][1:] and float(avg[1][0]) == pytest.approx(0.15)
    nan = scores_from([float("nan")] * 3, [0.1, 0.01, 0.5], [-1], [100], 100, (0.01,))
    assert all(np.isnan(x) for x in (nan.accuracy, nan.precision[0], nan.fscore[0]))


# ---------------------------------------------------------------- wrong oracles fail the GPU bars
def _bitwise_equal(x, y):
    x, y = np.asarray(x), np.asarray(y)
    return x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_wrong_oracles_fail_the_bars():
    """The GPU tests compare per-sample outputs bit for bit; each broken variant changes them on those tests' meshes."""
    V, F = O.random_mesh(300, seed=8, decades=3)
    p, f = O.sample(V, F, 500, seed=1)
    p_bad, f_bad = O.sample(V, F, 500, seed=1, wrong="nosqrt")
    assert np.array_equal(f, f_bad) and not _bitwise_equal(p, p_bad)
    d, g = O.closest(p, V, F)
    d_plane, g_plane = O.closest(p, V, F, wrong="plane")
    assert not (_bitwise_equal(d, d_plane) and _bitwise_equal(g, g_plane))
    # coincident duplicate faces: the tie rule decides the closest face
    Fd = np.concatenate([F, F[::-1]])
    d1, g1 = O.closest(p, V, Fd)
    d2, g2 = O.closest(p, V, Fd, wrong="highest")
    assert _bitwise_equal(d1, d2) and not _bitwise_equal(g1, g2)
    assert (g1 < 300).all()
