"""Normal maps on the H100 (TileShardedRenderer.render_range_maps(normals=True), toolbox/normal_maps.py): the affine
teachers of test_position_grad_gpu render a uniform normal, the normals' compositing uses the render's weights, the
colour, alpha and distance maps do not change, and the file export."""
import numpy as np
import pytest
import torch

from test_learned_occupancy_gpu import _sphere
from test_position_grad_gpu import ACC, TEACHERS, affine_teacher, spatial_direction, teacher_angle_bound

pytestmark = pytest.mark.gpu

STEP = 4e-4
W, H, G = 96, 72, 128


def _cams(cuda):
    from humanrf_b200.synthetic_scene import make_scene

    sc = make_scene(num_images=3, width=W, height=H, G=G, portrait_every=3)
    assert list(sc["landscape"]) == [True, True, False]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return sc, t


def _render(m, cuda, k, frame=16, rays_per_batch=2000):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer

    sc, t = _cams(cuda)
    og = OccupanyGrid(G, 1)
    handle = og.add_grid(torch.from_numpy(_sphere(G)).to(cuda))
    r = TileShardedRenderer(m, og, rays_per_batch=rays_per_batch)          # several batches per view
    cam = dict(frame_numbers=torch.tensor([frame], dtype=torch.int32, device=cuda),
               camera_numbers=t(sc["camera_numbers"][k:k + 1]),
               grid_handles=torch.tensor([handle], dtype=torch.int64, device=cuda),
               landscape=t(sc["landscape"][k:k + 1]), inverse_krs=t(sc["inverse_krs"][k:k + 1]),
               camera_origins=t(sc["camera_origins"][k:k + 1]), aabb=t(sc["aabb"]), G=G, width=W, height=H)
    return r, cam


@pytest.mark.parametrize("grid,a,b", TEACHERS, ids=["xyz", "xyt", "yzt", "xzt"])
def test_affine_teacher_normal_map(cuda, grid, a, b):
    """Every sample's normal is -a_s / |a_s| up to the gradient's accumulation bound, so the composited normal (a sum of
    vectors inside that cone) is too, up to the fp32 sum over the ray's samples and the two normalisations."""
    m = affine_teacher(cuda, grid, a, b)
    want = -spatial_direction(grid, a)
    want /= np.linalg.norm(want)
    for k in (0, 2):                                       # a landscape and the portrait camera
        r, cam = _render(m, cuda, k)
        P = W * H
        color, alpha, dist, nrm = r.render_range_maps(cam, 0, P, normals=True)
        nws = r.last_stats["normal_weights_sum"]
        color0, alpha0, dist0 = r.render_range_maps(cam, 0, P)
        assert torch.equal(color, color0) and torch.equal(alpha, alpha0) and torch.equal(dist, dist0)
        assert nrm.shape == (P, 3) and nrm.dtype == torch.float32
        # the normals' compositing runs on the render's weights: the fused-vs-unfused bar of the colour
        assert (nws - alpha).abs().max().item() <= 2e-6
        a_ = alpha.cpu().numpy()
        n_ = nrm.double().cpu().numpy()
        hit = a_ > 0
        assert hit.mean() > 0.05 and (n_[~hit] == 0).all()
        ln = np.linalg.norm(n_[hit], axis=1)
        assert np.abs(ln - 1).max() < 1e-5
        samples_per_ray = int(np.ceil(np.sqrt(3) / STEP))
        bound = teacher_angle_bound(grid, a, b) + (samples_per_ray + 8) * 2.0 ** -23
        ang = np.linalg.norm(n_[hit] - np.outer(n_[hit] @ want, want), axis=1)
        print(f"grid {grid} view {k}: {hit.sum()} pixels, max angle {ang.max():.3e} (bound {bound:.3e})")
        assert (n_[hit] @ want > 0).all() and (ang <= bound).all()


def test_vector_teacher_normal_map(cuda):
    c = 2.0 ** -9
    m = affine_teacher(cuda, 1, None, None, k=1.0, vector_slope=(c, -2.0))
    r, cam = _render(m, cuda, 1, frame=17, rays_per_batch=W * H)   # one batch
    _, alpha, _, nrm = r.render_range_maps(cam, 0, W * H, normals=True)
    hit = (alpha > 0).cpu().numpy()
    n_ = nrm.double().cpu().numpy()[hit]
    assert hit.mean() > 0.05
    scale = float(m.feature_grids[0].layout.scale[0])
    bound = ACC * scale * 2 / (c * 2048) + (int(np.ceil(np.sqrt(3) / STEP)) + 8) * 2.0 ** -23
    assert (n_[:, 2] < 0).all() and (np.abs(n_[:, :2]).max(1) <= bound).all()


def _loader(cuda):
    from test_depth_maps_gpu import _loader as depth_loader

    return depth_loader(cuda)


def test_render_normal_map_camera_frame(cuda):
    """Camera normals are the world normals rotated into the dataset camera's RDF frame, R_c2w^T n."""
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.toolbox.normal_maps import render_normal_map

    grid, a, b = TEACHERS[0]
    m = affine_teacher(cuda, grid, a, b)
    ds, dl = _loader(cuda)
    want = -spatial_direction(grid, a)
    want /= np.linalg.norm(want)
    bound = teacher_angle_bound(grid, a, b) + (int(np.ceil(np.sqrt(3) / STEP)) + 8) * 2.0 ** -23
    for c in (0, 2):
        nm = render_normal_map(m, dl, c, 16)
        cam = ds.cameras[c]
        assert nm.camera.shape == (cam.height, cam.width, 3) and nm.alpha.shape == (cam.height, cam.width)
        hit = (nm.alpha > 0).cpu().numpy()
        assert hit.mean() > 0.02
        R = rotation_from_axisangle(np.asarray(dl.cameras[c].rotation_axisangle, float))
        wc = R.T @ want
        nc = nm.camera.double().cpu().numpy()[hit]
        assert (np.linalg.norm(nc - wc, axis=1) <= 2 * bound + 1e-6).all()
        np.testing.assert_allclose(nm.camera.double().cpu().numpy(),
                                   nm.world.double().cpu().numpy() @ R, atol=1e-6)
        assert (nm.camera.cpu().numpy()[~hit] == 0).all()


def test_export_normal_sequence(cuda, tmp_path):
    import os

    os.environ.setdefault("OPENCV_IO_ENABLE_OPENEXR", "1")
    import cv2

    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid
    from humanrf_b200.toolbox.normal_maps import export_normal_sequence, render_normal_map

    grid, a, b = TEACHERS[1]
    m = affine_teacher(cuda, grid, a, b)
    _, dl = _loader(cuda)
    pairs = [(0, 15), (2, 15), (0, 16)]
    out = tmp_path / "maps"
    paths = export_normal_sequence(m, dl, pairs, out)
    assert sorted(str(p.relative_to(out)) for p in out.rglob("*") if p.is_file()) == sorted([
        "normals/Cam001/Cam001_normal000015.exr", "normals/Cam001/Cam001_normal000016.exr",
        "normals/Cam003/Cam003_normal000015.exr"])
    for (c, f), p in zip(pairs, paths):
        baked = bake_occupancy_grid(m, f, torch.from_numpy(_sphere(64)).to(cuda))
        nm = render_normal_map(m, dl, c, f, grid=baked)
        img = cv2.imread(p, cv2.IMREAD_UNCHANGED)
        ref = nm.camera.cpu().numpy()
        assert img.dtype == np.float32 and img.shape == ref.shape
        rgb = np.ascontiguousarray(img[..., ::-1])            # OpenCV hands back B, G, R
        assert np.array_equal(rgb.view(np.int32), ref.view(np.int32))
        assert (rgb[nm.alpha.cpu().numpy() == 0] == 0).all() and (np.abs(rgb) > 0).any()
    with pytest.raises(RuntimeError):
        export_normal_sequence(m, dl, [(0, 15), (0, 99)], tmp_path / "bad")
    assert not (tmp_path / "bad").exists()


def test_normal_maps_reject_bad_inputs(cuda):
    from humanrf_b200.toolbox.normal_maps import export_normal_sequence, render_normal_map

    grid, a, b = TEACHERS[0]
    m = affine_teacher(cuda, grid, a, b)
    _, dl = _loader(cuda)
    good = torch.from_numpy(_sphere(64)).to(cuda)
    for g in (good.float(), good.cpu(), good[0], good.bool()):
        with pytest.raises(RuntimeError):
            render_normal_map(m, dl, 0, 15, grid=g)
    for c, f in ((0, 99), (0, 14), (7, 15), (-1, 15)):
        with pytest.raises(RuntimeError):
            render_normal_map(m, dl, c, f)
        with pytest.raises(RuntimeError):
            export_normal_sequence(m, dl, [(c, f)], "/nonexistent/never_written")
