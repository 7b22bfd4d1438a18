"""Mesh rasterisation and depth scores on the H100 (csrc/mesh_raster.cu, toolbox/mesh_depth.py): z, mask, face and hits
against the numpy oracle bit for bit, determinism and graph replay, a 2 M-face marching-cubes mesh, the score
reductions, and evaluate_depth / export_mesh_depth_sequence on the confined teacher."""
import csv

import numpy as np
import pytest
import torch

import raster_oracle as O
from geometry_oracle import icosphere

pytestmark = pytest.mark.gpu


def _mesh(V, F, dev):
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    return Mesh(torch.from_numpy(np.ascontiguousarray(V, np.float32)).to(dev),
                torch.from_numpy(np.ascontiguousarray(F, np.int32)).to(dev))


def _oracle(V, F, cam, near=0.01, far=100.0, scale=1.0):
    from humanrf_b200.toolbox.mesh_depth import camera_projection

    m, fx, fy, cx, cy = camera_projection(cam, scale)
    return O.rasterize(V, F, m, fx, fy, cx, cy, cam.width, cam.height, near, far)


def _gpu(V, F, cam, dev, near=0.01, far=100.0, scale=1.0):
    from humanrf_b200.toolbox.mesh_depth import rasterize_mesh

    r = rasterize_mesh(_mesh(V, F, dev), cam, scale, near, far, hits=True)
    torch.cuda.synchronize()
    return dict(z=r.z.cpu().numpy(), mask=r.mask.cpu().numpy(), face=r.face.cpu().numpy(), hits=r.hits.cpu().numpy(),
                error=int(r.error.cpu()[0]), skipped=int(r.skipped.cpu()[0]))


def _same(a, b):
    for k in ("mask", "face", "hits"):
        assert np.array_equal(a[k], b[k]), (k, int((a[k] != b[k]).sum()))
    assert np.array_equal(a["z"].view(np.uint32), b["z"].view(np.uint32)), int((a["z"] != b["z"]).sum())
    assert a["error"] == b["error"] and a["skipped"] == b["skipped"], (a["error"], b["error"], a["skipped"], b["skipped"])


def _soup(nf, seed, size=(0.02, 0.3), spread=0.5):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-spread, spread, (nf, 1, 3))
    s = 10 ** rng.uniform(np.log10(size[0]), np.log10(size[1]), (nf, 1, 1))
    V = (c + s * rng.normal(size=(nf, 3, 3))).reshape(-1, 3).astype(np.float32)
    return V, np.arange(3 * nf, dtype=np.int32).reshape(-1, 3)


def _case_overlap():
    V, F = _soup(3000, 0)
    F = np.concatenate([F, F[::5], F[::7, ::-1]])               # duplicates, both windings, later ids
    return V, F, O.look_at(97, 61, (0.3, -0.4, 2.2), seed=1), {}


def _case_sizes():
    Vs, Fs = _soup(4000, 1, size=(1e-4, 3e-3))                  # sub-pixel
    Vb, Fb = _soup(12, 2, size=(1.0, 3.0), spread=0.2)          # larger than the image: many chunks each
    return (np.concatenate([Vs, Vb]), np.concatenate([Fs, Fb + len(Vs)]), O.look_at(131, 77, (0.0, 0.2, 2.0), seed=2),
            {})


def _case_border():
    V, F = _soup(2000, 3, size=(0.05, 0.6), spread=1.6)         # straddling the border and off-screen
    V = np.concatenate([V, np.array([[0, 0, 2.1], [0.1, 0, 1.9], [0, 0.1, 2.5]], np.float32)])   # behind / at near
    F = np.concatenate([F, [[len(V) - 3, len(V) - 2, len(V) - 1], [0, 1, len(V) - 2]]])
    return V, F, O.look_at(64, 48, (0.0, 0.0, 2.0), seed=3), dict(near=0.2)


def _case_degenerate():
    V, F = _soup(1500, 4)
    V = np.concatenate([V, np.array([[0, 0, 0], [0.1, 0.1, 0.1], [0.2, 0.2, 0.2]], np.float32)])
    n = len(V)
    deg = np.array([[n - 3, n - 2, n - 1], [5, 5, 5], [7, 7, 9], [0, 1, n], [-1, 2, 3], [2 ** 31 - 1, 0, 1]], np.int32)
    return V, np.concatenate([F[:700], deg, F[700:]]), O.look_at(50, 70, (0.5, 0.1, 1.8), seed=4), {}


def _case_tiny():
    V, F = _soup(200, 5, size=(0.1, 0.8))
    return V, F, O.look_at(1, 1, (0.0, 0.0, 2.0), seed=5), {}


def _case_tiling():
    V, F = O.quad_grid(11, 7, 128, 64, 6)
    return V, F, O.pixel_camera(128, 64), {}


def _case_scale():
    V, F = _soup(1000, 7)
    return (V * np.float32(1000), F, O.look_at(83, 83, (0.1, 0.1, 2.0), seed=6), dict(scale=1e-3, far=2.1))


CASES = {"overlap": _case_overlap, "sizes": _case_sizes, "border": _case_border, "degenerate": _case_degenerate,
         "1x1": _case_tiny, "tiling": _case_tiling, "scale-far": _case_scale}


@pytest.mark.parametrize("case", list(CASES))
def test_matches_oracle_bitwise(cuda, case):
    V, F, cam, kw = CASES[case]()
    got, want = _gpu(V, F, cam, cuda, **kw), _oracle(V, F, cam, **kw)
    _same(got, want)
    print(f"{case}: {len(F)} faces {cam.width}x{cam.height}: covered {int((want['mask'] > 0).sum())}, "
          f"max hits {want['hits'].max()}, skipped {want['skipped']}, error {want['error']}")
    if case == "degenerate":
        assert want["error"] == 1
    if case == "border":
        assert want["skipped"] >= 1
    if case == "tiling":
        assert want["hits"].max() == 1


def test_determinism_and_graph_replay(cuda):
    from humanrf_b200.toolbox.mesh_depth import rasterize_mesh

    V, F, cam, _ = _case_overlap()
    cam = O.look_at(640, 480, (0.3, -0.4, 2.2), seed=1)
    mesh = _mesh(V, F, cuda)
    a = rasterize_mesh(mesh, cam, hits=True)
    b = rasterize_mesh(mesh, cam, hits=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            c = rasterize_mesh(mesh, cam, hits=True)
    torch.cuda.current_stream().wait_stream(s)
    for t in (c.z, c.face, c.hits):
        t.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    for name in ("z", "mask", "face", "hits", "error", "skipped"):
        x, y, z = (getattr(r, name).view(torch.uint8) for r in (a, b, c))
        assert torch.equal(x, y) and torch.equal(x, z), name


def test_bench_mesh_against_oracle(cuda):
    """The bench model's ~2 M-face marching-cubes mesh at 1028x752: seeded pixels against the oracle, and every pixel
    centre covered an even number of times (the mesh is closed)."""
    from test_geometry_metrics_gpu import _bench_meshes

    from humanrf_b200.toolbox.mesh_depth import camera_projection

    mesh, _ = _bench_meshes(cuda)
    assert mesh.faces.shape[0] > 1_500_000
    V, F = mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy()
    for k, pos in enumerate(((2.0, 0.3, 0.4), (-0.5, -1.2, 1.5))):
        cam = O.look_at(1028, 752, pos, f=1.2, seed=k)
        got = _gpu(V, F, cam, cuda)
        assert got["error"] == 0 and got["skipped"] == 0
        assert (got["hits"] % 2 == 0).all(), int((got["hits"] % 2).sum())
        covered = np.nonzero(got["mask"].reshape(-1))[0]
        assert len(covered) > 10_000
        rng = np.random.default_rng(k)
        pix = np.concatenate([rng.choice(covered, 192, replace=False), rng.choice(1028 * 752, 64, replace=False)])
        m, fx, fy, cx, cy = camera_projection(cam)
        z, f, h = O.rasterize_pixels(V, F, m, fx, fy, cx, cy, 1028, 752, pix % 1028, pix // 1028)
        assert np.array_equal(got["face"].reshape(-1)[pix], f)
        assert np.array_equal(got["hits"].reshape(-1)[pix], h)
        assert np.array_equal(got["z"].reshape(-1)[pix].view(np.uint32), z.view(np.uint32))
        print(f"view {k}: {len(F)} faces, covered {len(covered)}, fragments {int(got['hits'].sum())}, "
              f"max hits {got['hits'].max()}")


def test_depth_scores_against_float64(cuda):
    from humanrf_b200.toolbox.mesh_depth import depth_scores

    rng = np.random.default_rng(0)
    taus = (0.001, 0.005, 0.01, 0.02, 0.05, 0.1, 0.2, 0.5)
    for n in (1, 777, 4112 * 3008):
        ref = rng.uniform(0.5, 4.0, n).astype(np.float32)
        pred = (ref + rng.normal(0, 0.02, n)).astype(np.float32)
        pm = (rng.random(n) < 0.8).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)
        rm = rng.random(n) < 0.7
        if n == 1:
            pm[:], rm[:] = 1, True
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(cuda)
        rows = torch.full((3, 4), -1.0, dtype=torch.float64, device=cuda)
        out, counts, err = depth_scores(t(pred), t(pm), t(ref), t(rm), taus, out=rows[1])
        out2, counts2, _ = depth_scores(t(pred), t(pm), t(ref), t(rm), taus)
        torch.cuda.synchronize()
        assert torch.equal(out2.view(torch.uint8), rows[1].view(torch.uint8)) and torch.equal(counts, counts2)
        assert (rows[0] == -1).all() and (rows[2] == -1).all()
        want, want_counts, want_err, sums = O.depth_scores(pred, pm, ref, rm, taus)
        assert int(err.cpu()[0]) == want_err == 0
        assert np.array_equal(counts.cpu().numpy(), want_counts)
        got = out.cpu().numpy()
        B = int(want_counts[0])
        for k in range(4):
            bound = B * 2.0 ** -53 * sums[k] / B * 2
            if k == 2:                     # RMSE: the bound on the mean square, through the square root
                assert abs(got[k] ** 2 - want[k] ** 2) <= bound + 4 * 2.0 ** -53 * want[k] ** 2, (k, got[k], want[k])
            else:
                assert abs(got[k] - want[k]) <= bound + 2.0 ** -53 * abs(want[k]), (k, got[k], want[k])
    # NaN and error rules
    n = 1000
    ref = np.full(n, 2.0, np.float32)
    pred = ref.copy()
    m = np.ones(n, np.uint8)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(cuda)
    out, counts, err = depth_scores(t(pred), t(m), t(ref), t(np.zeros(n, np.uint8)))
    assert torch.isnan(out).all() and int(err.cpu()[0]) == 0 and int(counts[0]) == 0 and int(counts[1]) == n
    for bad in (0.0, -1.0, np.inf, np.nan):
        for side in (0, 1):
            p, r = pred.copy(), ref.copy()
            (p if side == 0 else r)[17] = bad
            out, counts, err = depth_scores(t(p), t(m), t(r), t(m))
            assert torch.isnan(out).all() and int(err.cpu()[0]) == 1 and int(counts[0]) == n
    out, counts, err = depth_scores(t(pred), t(m), t(ref), t(m), taus=(0.0,))
    assert out.cpu().tolist() == [0.0, 0.0, 0.0, 0.0] and counts.cpu().tolist() == [n, n, n, n, n, n]


def test_rejects_bad_inputs(cuda):
    from humanrf_b200.toolbox.mesh_depth import depth_scores, rasterize_mesh
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    V, F = _soup(10, 0)
    good = _mesh(V, F, cuda)
    cam = O.look_at(32, 24, (0, 0, 2.0))
    for m in (Mesh(good.vertices.cpu(), good.faces.cpu()), Mesh(good.vertices.double(), good.faces),
              Mesh(good.vertices, good.faces.long()), "not a mesh"):
        with pytest.raises(RuntimeError):
            rasterize_mesh(m, cam)
    for kw in (dict(near=0.0), dict(near=2.0, far=1.0), dict(far=float("inf")), dict(scale=0.0)):
        with pytest.raises(RuntimeError):
            rasterize_mesh(good, cam, **kw)
    z = torch.ones(100, device=cuda)
    mk = torch.ones(100, dtype=torch.uint8, device=cuda)
    for args in ((z.cpu(), mk, z, mk), (z.double(), mk, z, mk), (z, mk.float(), z, mk), (z, mk, z[:50], mk)):
        with pytest.raises(RuntimeError):
            depth_scores(*args)
    with pytest.raises(RuntimeError):
        depth_scores(z, mk, z, mk, taus=tuple(range(9)))


# ---------------------------------------------------------------------------------------------------- confined scene
def _reference(tmp_path, cuda, frames):
    """The teacher's ellipsoid E as an icosphere in world units, one OBJ per frame; returns the directory and the
    tessellation gap (normalised units)."""
    from test_geometry_metrics_gpu import RADII

    from humanrf_b200.toolbox.mesh_extraction import Mesh, scene_normalisation, to_world, write_obj

    from test_depth_maps_gpu import _loader

    ds, dl = _loader(cuda)
    offset, scale = scene_normalisation(ds)
    Vu, Fu = icosphere(5, 1.0)
    from geometry_oracle import sphere_tessellation_gap

    gap = sphere_tessellation_gap(Vu, Fu, 1.0) * RADII.max()
    ref = to_world(Mesh(torch.from_numpy((Vu * RADII).astype(np.float32)).to(cuda), torch.from_numpy(Fu).to(cuda)),
                   offset, scale)
    refdir = tmp_path / "ref"
    refdir.mkdir()
    for f in frames:
        write_obj(refdir / f"Frame{f:06d}.obj", ref)
    return ds, dl, refdir, gap


def test_evaluate_depth_confined_teacher(cuda, tmp_path):
    """Model depth against the rasterised icosphere of the teacher's ellipsoid E.  The model's surface lies within
    b_m = sqrt(3) / scale0 + 2 step of E along each ray (§3.7's test), the icosphere within its gap g inside E, so both
    surfaces lie in the shell of width b = b_m + g around E's surface; along a ray meeting E's surface at angle theta
    to the normal the shell is at most about b / cos(theta) long, and z <= distance since |v| >= 1.  Checked per pixel
    where cos(theta) >= 0.5 and the view is opaque (bound 2.2 b); and every pixel where the masks differ has a ray passing within b of E."""
    from test_depth_maps_gpu import STEP, _min_distance_along, _ray_directions
    from test_geometry_metrics_gpu import RADII
    from test_learned_occupancy_gpu import confined_teacher

    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid
    from humanrf_b200.toolbox.mesh_depth import csv_columns, depth_scores, evaluate_depth, rasterize_mesh
    from humanrf_b200.toolbox.geometry_metrics import read_obj

    m = confined_teacher(cuda)
    frames = (15, 16)
    ds, dl, refdir, gap = _reference(tmp_path, cuda, frames)
    scene_scale = float(dl.scene_scale)
    scale0 = float(m.feature_grids[0].layout.scale[0])
    b = np.sqrt(3) / scale0 + 2 * STEP + gap                  # normalised units
    band = b / scene_scale                                    # world units
    taus = (0.005, 0.01, 2.2 * band)
    pairs = [(0, 15), (2, 15), (1, 16)]
    scores = evaluate_depth(m, dl, pairs, refdir, tmp_path / "out", taus=taus)
    assert [(s.camera, s.frame) for s in scores] == pairs
    for s in scores:
        assert s.n > 100 and s.mae <= 2.2 * band and s.iou > 0.5, s
        print(f"camera {s.camera} frame {s.frame}: n {s.n} bias {s.bias:.5f} mae {s.mae:.5f} rmse {s.rmse:.5f} "
              f"within {s.within} iou {s.iou:.4f} (band {band:.5f} world units)")
    # per pixel, for one view, through the public pieces evaluate_depth uses
    c, f = 2, 15
    dm = render_depth_map(m, dl, c, f, grid=bake_occupancy_grid(m, f, torch.from_numpy(ds.get_occupancy_grid(f)).to(cuda)))
    ref = rasterize_mesh(read_obj(refdir / f"Frame{f:06d}.obj", device=cuda), ds.cameras[c])
    pm, rm = (dm.alpha >= 0.5).cpu().numpy().reshape(-1), (ref.mask != 0).cpu().numpy().reshape(-1)
    pz, rz = dm.z.double().cpu().numpy().reshape(-1), ref.z.double().cpu().numpy().reshape(-1)
    cam = dl.cameras[c]
    d, _, _ = _ray_directions(dl.all_inverse_krs[c].cpu(), cam.width, cam.height)
    o = dl.all_camera_origins[c].cpu().numpy().astype(np.float64)
    dr, orr = d / RADII, o / RADII                            # ray against E: |(o + t d) / RADII| = 1
    qa, qb, qc = (dr * dr).sum(1), 2 * (dr * orr).sum(1), (orr * orr).sum() - 1
    disc = qb * qb - 4 * qa * qc
    t0 = (-qb - np.sqrt(np.maximum(disc, 0))) / (2 * qa)
    p = o + t0[:, None] * d
    nrm = p / RADII ** 2
    cos = np.abs((nrm * d).sum(1)) / np.linalg.norm(nrm, axis=1)
    B = pm & rm
    solid = dm.alpha.cpu().numpy().reshape(-1) >= 0.99     # where §3.7 pins the rendered distance to the band
    steep = B & solid & (disc > 0) & (cos >= 0.5)
    assert steep.sum() > 100
    err = np.abs(pz - rz)
    assert (err[steep] <= 2.2 * band).all(), (err[steep].max(), band)
    out, counts, _ = depth_scores(dm.z, dm.alpha >= 0.5, ref.z, ref.mask)
    assert int(counts[0]) == B.sum()
    differ = pm != rm
    assert differ.any()
    assert (_min_distance_along(o, d[differ]) <= b).all()
    # the tables
    rows = list(csv.reader(open(tmp_path / "out" / "depth.csv")))
    assert rows[0] == csv_columns(taus)
    assert [(int(r[0]), int(r[1])) for r in rows[1:]] == [(c + 1, f) for c, f in pairs]
    assert int(rows[1][2]) == scores[0].n and float(rows[1][4]) == scores[0].mae
    avg = list(csv.reader(open(tmp_path / "out" / "depth_averages.csv")))
    assert avg[0] == rows[0][2:] and float(avg[1][2]) == pytest.approx(np.mean([s.mae for s in scores]))
    # bad inputs raise before any work, and nothing is written
    for bad_pairs, what in (([(0, 15), (0, 17)], "missing reference meshes"), ([(0, 99)], None), ([(9, 15)], None),
                            ([(-1, 15)], None)):
        with pytest.raises(RuntimeError, match=what):
            evaluate_depth(m, dl, bad_pairs, refdir, tmp_path / "bad")
        assert not (tmp_path / "bad").exists()


def test_export_mesh_depth_sequence(cuda, tmp_path):
    import cv2

    from humanrf_b200.toolbox.geometry_metrics import read_obj
    from humanrf_b200.toolbox.mesh_depth import export_mesh_depth_sequence, rasterize_mesh

    ds, _, refdir, _ = _reference(tmp_path, cuda, (15, 16))
    pairs = [(0, 15), (2, 15), (0, 16)]
    out = tmp_path / "maps"
    paths = export_mesh_depth_sequence(ds.cameras, pairs, refdir, out)
    assert sorted(str(p.relative_to(out)) for p in out.rglob("*") if p.is_file()) == sorted([
        "depths/Cam001/Cam001_depth000015.exr", "depths/Cam001/Cam001_depth000016.exr",
        "depths/Cam003/Cam003_depth000015.exr", "masks/Cam001/Cam001_mask000015.png",
        "masks/Cam001/Cam001_mask000016.png", "masks/Cam003/Cam003_mask000015.png"])
    for (c, f), (dp, mp) in zip(pairs, paths):
        r = rasterize_mesh(read_obj(refdir / f"Frame{f:06d}.obj", device=cuda), ds.cameras[c])
        z = cv2.imread(dp, cv2.IMREAD_UNCHANGED)
        assert z.dtype == np.float32 and np.array_equal(z.view(np.int32), r.z.cpu().numpy().view(np.int32))
        assert (z > 0).any()
        mask = cv2.imread(mp, cv2.IMREAD_UNCHANGED)
        assert mask.dtype == np.uint8 and np.array_equal(mask, r.mask.cpu().numpy())
    for bad in ([(0, 15), (0, 17)], [(5, 15)], [(0, -1)]):
        with pytest.raises(RuntimeError):
            export_mesh_depth_sequence(ds.cameras, bad, refdir, tmp_path / "bad")
        assert not (tmp_path / "bad").exists()
