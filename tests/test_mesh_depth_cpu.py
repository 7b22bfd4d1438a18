"""Mesh rasterisation and depth scores on the CPU (tests/raster_oracle.py, the restatement of hrf_rasterize_mesh and
hrf_depth_metrics): the projection against the dataset's world2pixel, the tie rule on tilings, fans and closed
meshes, plane depth, visibility ties, the skip and error rules, and the score formulas."""
import numpy as np
import pytest

import raster_oracle as O
from geometry_oracle import icosphere


def _run(V, F, cam, near=0.01, far=100.0, scale=1.0):
    from humanrf_b200.toolbox.mesh_depth import camera_projection

    m, fx, fy, cx, cy = camera_projection(cam, scale)
    return O.rasterize(V, F, m, fx, fy, cx, cy, cam.width, cam.height, near, far)


@pytest.mark.parametrize("W,H,scale", [(96, 72, 1.0), (72, 96, 1.0), (96, 72, 2.5), (4112, 3008, 0.001)])
def test_projection_matches_world2pixel(W, H, scale):
    from humanrf_b200.dataset.cameras import projection_matrix_world2pixel
    from humanrf_b200.toolbox.mesh_depth import camera_projection

    cam = O.look_at(W, H, (0.4, -0.3, 2.5), f=1.1, seed=3)
    rng = np.random.default_rng(0)
    P = (rng.uniform(-0.5, 0.5, (500, 3)) / scale).astype(np.float32)
    m, fx, fy, cx, cy = camera_projection(cam, scale)
    U, Vv, Z, ok = O.project(P, m, fx, fy, cx, cy, 0.01)
    w2p = projection_matrix_world2pixel(W, H, cam.rotation_axisangle, cam.translation, cam.focal_length,
                                        cam.principal_point)
    q = (w2p @ np.concatenate([P.astype(np.float64) * scale, np.ones((len(P), 1))], 1).T).T
    u, v = q[:, 0] / q[:, 2], q[:, 1] / q[:, 2]
    assert ok.all()
    np.testing.assert_allclose(Z, q[:, 2], rtol=1e-14, atol=0)
    # the fixed point is u rounded to 1/256 pixel; the two float64 routes differ by a few ulps of (u, z)
    tol = 1e-12 * max(W, H)
    assert (np.abs(U / 256.0 - u) <= 1 / 512 + tol).all() and (np.abs(Vv / 256.0 - v) <= 1 / 512 + tol).all()


@pytest.mark.parametrize("split", ["main", "anti", "both"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_quad_tiling_covers_every_centre_once(split, seed):
    W, H = 64, 32
    V, F = O.quad_grid(7, 5, W, H, seed, split=split)
    x, y = V[:, 0].astype(np.float64), V[:, 1].astype(np.float64)
    f = F.astype(np.int64)
    area = (x[f[:, 1]] - x[f[:, 0]]) * (y[f[:, 2]] - y[f[:, 0]]) - (y[f[:, 1]] - y[f[:, 0]]) * (x[f[:, 2]] - x[f[:, 0]])
    assert (area > 0).all()                                  # a tiling: no fold-over
    on_centre = ((V[:, 0] - 0.5) % 1 == 0) & ((V[:, 1] - 0.5) % 1 == 0)
    assert on_centre.sum() >= 5
    r = _run(V, F, O.pixel_camera(W, H))
    cx, cy = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    lo, hi = 333 / 256, (W * 256 - 333) / 256,
    inside = (cx > lo) & (cx < W - lo) & (cy > lo) & (cy < H - lo)
    assert (r["hits"][inside] == 1).all(), int((r["hits"][inside] != 1).sum())
    assert (r["hits"][~inside] == 0).all()
    assert (r["mask"][inside] == 255).all() and (r["face"][inside] >= 0).all()
    np.testing.assert_allclose(r["z"][inside], 1.0, rtol=2 ** -23)
    # reversing every face's winding changes no output
    r2 = _run(V, F[:, ::-1].copy(), O.pixel_camera(W, H))
    assert np.array_equal(r2["hits"], r["hits"]) and np.array_equal(r2["face"], r["face"])
    assert np.array_equal(r2["z"].view(np.uint32), r["z"].view(np.uint32))


@pytest.mark.parametrize("n", [3, 4, 5, 7, 12])
def test_fan_covers_its_centre_once(n):
    W = H = 32
    rng = np.random.default_rng(n)
    for trial in range(20):
        c = np.array([15.5, 16.5])
        if trial % 4 == 0 and n >= 4:                        # spokes along the axes through pixel centres
            ang = np.sort(np.concatenate([np.arange(4) * np.pi / 2, rng.uniform(0, 2 * np.pi, n - 4)]))
        else:
            ang = np.sort(rng.uniform(0, 2 * np.pi, n))
            while np.diff(np.concatenate([ang, [ang[0] + 2 * np.pi]])).max() >= np.pi * 0.95:
                ang = np.sort(rng.uniform(0, 2 * np.pi, n))
        rad = rng.uniform(2, 6, n)
        pts = np.round((c + np.stack([np.cos(ang), np.sin(ang)], 1) * rad[:, None]) * 256) / 256
        V = np.concatenate([[c], pts])
        V = np.concatenate([V, np.ones((len(V), 1))], 1).astype(np.float32)
        F = np.array([(0, 1 + k, 1 + (k + 1) % n) for k in range(n)], np.int32)
        flip = rng.random(n) < 0.5                           # mixed windings
        F[flip] = F[flip][:, ::-1]
        r = _run(V, F, O.pixel_camera(W, H))
        assert r["hits"][16, 15] == 1, (n, trial)
        assert r["hits"].max() == 1


def test_closed_icosphere_covers_every_centre_zero_or_two_times():
    Vu, F = icosphere(3)
    for seed in range(4):
        R = O.random_rotation(seed)
        V = ((Vu.astype(np.float64) @ R.T) * 0.4).astype(np.float32)
        cam = O.look_at(80, 60, (0.3, -0.2, 2.0), seed=seed)
        r = _run(V, F, cam)
        assert set(np.unique(r["hits"])) == {0, 2}
        assert ((r["hits"] == 2) == (r["mask"] == 255)).all()
        assert r["skipped"] == 0 and r["error"] == 0


def test_plane_depth_is_the_analytic_depth():
    """A tilted plane whose vertices project onto the fixed-point grid: z at a covered pixel is the plane's depth along
    the pixel ray, within the float64 evaluation and one float32 rounding."""
    W = H = 64
    rng = np.random.default_rng(5)
    uv = np.array([[3.25, 2.5], [60.75, 7.0], [10.5, 61.25], [58.0, 59.5]])
    n, c = np.array([0.3, -0.2, 1.0]), 2.0                   # plane n . X = c
    # X = (u Z, v Z, Z) on the plane: Z = c / (n . (u, v, 1)); exact floats need Z of few bits, so pick Z first
    Z = np.array([2.0, 1.5, 2.5, 1.75])
    P = np.stack([uv[:, 0] * Z, uv[:, 1] * Z, Z], 1)
    # the plane through the first three points
    n = np.cross(P[1] - P[0], P[2] - P[0])
    c = n @ P[0]
    V = P.astype(np.float32)
    assert np.array_equal(V.astype(np.float64), P)
    F = np.array([[0, 1, 2]], np.int32)
    r = _run(V, F, O.pixel_camera(W, H))
    ys, xs = np.nonzero(r["mask"])
    assert len(xs) > 500
    d = np.stack([xs + 0.5, ys + 0.5, np.ones(len(xs))], 1)
    want = c / (d @ n)
    got = r["z"][ys, xs].astype(np.float64)
    assert (np.abs(got - want) <= 2 ** -24 * want + 1e-12 * want).all(), np.abs(got / want - 1).max()
    del rng


def test_equal_depth_goes_to_the_lowest_face_id():
    W = H = 32
    V, F = O.quad_grid(3, 3, W, H, 0, centres=False)
    F2 = np.concatenate([F[::-1], F, F[:, ::-1]])            # three coincident copies; the reversed block first
    r = _run(V, F2, O.pixel_camera(W, H))
    m = r["mask"] == 255
    n = len(F)
    # the lowest id covering a pixel: face k of F appears as ids n - 1 - k, n + k and 2n + k
    r1 = _run(V, F, O.pixel_camera(W, H))
    assert np.array_equal(r["face"][m], n - 1 - r1["face"][m])
    assert (r["hits"][m] == 3).all()


def test_near_far_skipped_and_error():
    W = H = 32
    cam = O.pixel_camera(W, H)
    tri = np.array([[4.5, 4.5, 1], [28.5, 6.5, 1], [8.5, 27.5, 1]], np.float32)
    V = np.concatenate([tri, tri * np.float32(3)])           # z = 1 and z = 3, same pixels
    F = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    r = _run(V, F, cam, far=2.0)
    m = r["mask"] == 255
    assert m.any() and (r["face"][m] == 0).all()
    r = _run(V, F, cam, near=1.5)                            # face 0 has vertices in front of near: skipped
    assert r["skipped"] == 1 and (r["face"][r["mask"] == 255] == 1).all() and r["error"] == 0
    r = _run(V, F, cam, near=0.5, far=0.9)                   # nothing in range: no fragments, but coverage counts
    assert not r["mask"].any() and r["hits"].max() == 2 and (r["z"] == 0).all() and (r["face"] == -1).all()
    bad = np.array([[0, 1, 2], [0, 1, 6], [-1, 1, 2], [3, 4, 5]], np.int32)
    r = _run(V, bad, cam)
    assert r["error"] == 1 and r["skipped"] == 0 and set(np.unique(r["face"])) == {-1, 0}
    # a vertex behind the camera, one far off-screen, a non-finite one: skipped; a zero-area and an off-image face: not
    odd = np.array([[1, 1, -1], [1e7, 1, 1], [np.nan, 1, 1], [40.5, 4.5, 1], [50.5, 4.5, 1], [60.5, 30.5, 1]],
                   np.float32)
    V2 = np.concatenate([tri, odd])
    F2 = np.array([[0, 1, 3], [0, 1, 4], [0, 1, 5], [0, 1, 0], [6, 7, 8], [0, 1, 2]], np.int32)
    r = _run(V2, F2, cam)
    assert r["skipped"] == 3 and r["error"] == 0 and set(np.unique(r["face"])) == {-1, 5}


def test_depth_scores_formulas():
    rng = np.random.default_rng(0)
    n = 5000
    ref = rng.uniform(0.5, 3.0, n).astype(np.float32)
    pred = (ref + rng.normal(0, 0.01, n)).astype(np.float32)
    pm, rm = rng.random(n) < 0.8, rng.random(n) < 0.7
    taus = (0.005, 0.01, 0.02)
    out, counts, err, _ = O.depth_scores(pred, pm, ref, rm, taus)
    B = pm & rm
    d = pred[B].astype(np.float64) - ref[B]
    assert err == 0 and counts[0] == B.sum() and counts[3] == B.sum() and counts[4] == (pm | rm).sum()
    np.testing.assert_allclose(out, [d.mean(), np.abs(d).mean(), np.sqrt((d ** 2).mean()),
                                     (np.abs(d) / ref[B]).mean()], rtol=1e-12)
    assert list(counts[5:]) == [int((np.abs(d) <= t).sum()) for t in taus]
    # NaN rules: empty B, and a non-positive or non-finite z inside B
    out, counts, err, _ = O.depth_scores(pred, pm, ref, np.zeros(n, bool), taus)
    assert np.isnan(out).all() and err == 0 and counts[0] == 0
    for bad in (0.0, -1.0, np.inf, np.nan):
        p2 = pred.copy()
        p2[np.nonzero(B)[0][3]] = bad
        out, _, err, _ = O.depth_scores(p2, pm, ref, rm, taus)
        assert np.isnan(out).all() and err == 1
    p2 = pred.copy()
    p2[np.nonzero(~B)[0][0]] = np.nan                        # outside B: ignored
    assert O.depth_scores(p2, pm, ref, rm, taus)[2] == 0


def test_depth_table_columns(tmp_path):
    import csv

    from humanrf_b200.toolbox.mesh_depth import DepthScore, csv_columns, write_depth_tables

    taus = (0.005, 0.01)
    s = [DepthScore(0, 15, 10, 0.1, 0.2, 0.3, 0.4, taus, (0.5, 0.6), 0.7, 0.8, 0.9),
         DepthScore(2, 16, 20, 0.3, 0.4, 0.5, 0.6, taus, (0.7, 0.8), 0.9, 1.0, 0.5)]
    write_depth_tables(tmp_path, s)
    rows = list(csv.reader(open(tmp_path / "depth.csv")))
    assert rows[0] == csv_columns(taus) == ["camera", "frame", "n", "bias", "mae", "rmse", "absrel", "within@0.005",
                                            "within@0.01", "iou", "precision", "recall"]
    assert rows[1][:3] == ["1", "15", "10"] and rows[2][:3] == ["3", "16", "20"]
    avg = list(csv.reader(open(tmp_path / "depth_averages.csv")))
    assert avg[0] == rows[0][2:] and np.allclose([float(x) for x in avg[1]],
                                                 [15, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 0.7])
