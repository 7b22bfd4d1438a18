"""Depth and opacity maps on the H100 (csrc/field_fwd.cu kDepth variants, hrf_render_fused_depth,
volume_rendering.render_with_depth, TileShardedRenderer.render_range_maps, toolbox/depth_maps.py): the fused depth
against float64 compositing of the unfused densities, colour unchanged bit for bit, the geometry of the confined
teacher, and the file export."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import synthetic_rays
from test_depth_maps_cpu import _make_scene_world2pixel
from test_learned_occupancy_gpu import _sphere, confined_teacher
from test_mesh_extraction_gpu import RADII, _ellipsoid_distance

pytestmark = pytest.mark.gpu

STEP = 4e-4


def _ragged_batch(cuda):
    """The ragged batch of test_composite_gpu::test_fused_render_kernel_equals_forward_plus_composite: 0..600 samples per
    ray, every 7th ray empty, rays spanning 2..5 tiles, a tail tile."""
    from helpers import make_pair

    _, m, frames = make_pair((6,), table_std=2.0)
    nr = 150
    b = synthetic_rays(nr, 600, frames, seed=13, ragged=True)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    counts = torch.bincount(b["ri"], minlength=nr)
    assert (counts == 0).any() and (counts > 512).any() and (counts < 128).any()
    return m, g, nr, counts


def _reference_depth(sigma, t, ri, nr):
    """sum_i w_i m_i per ray in float64 from float32 sigma, with the kernel's float32 dt and m_i; also max_i m_i."""
    s = sigma.double().cpu().numpy()
    tf = t.cpu().numpy().astype(np.float32)
    te = tf + np.float32(STEP)
    dt = (te - tf).astype(np.float64)
    mid = (np.float32(0.5) * (tf + te)).astype(np.float64)
    ri = ri.cpu().numpy()
    depth, mmax = np.zeros(nr), np.zeros(nr)
    sdt = s * dt
    for r in range(nr):
        sel = ri == r
        if not sel.any():
            continue
        x = sdt[sel]
        before = np.concatenate([[0.0], np.cumsum(x)[:-1]])
        w = np.exp(-before) * (1 - np.exp(-x))
        depth[r] = (w * mid[sel]).sum()
        mmax[r] = mid[sel].max()
    return depth, mmax


def _features(nat, samples, n, cuda):
    """Composed features of every sample, stored in a shuffled row order: the fused kernel reads them through an index
    as it reads a prune pass's features."""
    _, _, _, saved = nat.forward(samples, 1, want_geo=False, want_feat=True)
    feat = nat.saved_features(saved, n)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(5)).to(cuda)
    shuffled = torch.empty_like(feat)
    shuffled[perm] = feat
    return shuffled, perm.to(torch.int32)


@pytest.mark.parametrize("with_bg", [False, True])
def test_fused_depth_equals_float64_compositing(cuda, with_bg):
    from humanrf_b200.volume_rendering import ray_offsets, render_fused

    m, g, nr, counts = _ragged_batch(cuda)
    n = g["t"].shape[0]
    bg = torch.rand(nr, 3, generator=torch.Generator().manual_seed(1)).to(cuda) if with_bg else None
    nat = m.native()
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"])
    off = ray_offsets(g["ri"], nr)
    sigma, _, _, _ = nat.forward(samples, 1, False, False)
    ref, mmax = _reference_depth(sigma, g["t"], g["ri"], nr)
    feat, src = _features(nat, samples, n, cuda)
    empty = (counts == 0).numpy()
    args = (m, g["o"], g["d"], g["frames"], g["t"], g["ri"], nr, bg)
    for name, reuse in (("encode", None), ("from features", (feat, src, off))):
        col, ws, depth = render_fused(*args, reuse=reuse, want_depth=True)
        col0, ws0 = render_fused(*args, reuse=reuse)
        # colour and weights sum of the depth variant are those of the plain kernel, bit for bit
        assert torch.equal(col, col0) and torch.equal(ws, ws0), name
        d = depth.view(-1).double().cpu().numpy()
        assert depth.shape == (nr, 1) and (d[empty] == 0).all()
        err = np.abs(d - ref)
        # 2e-6 is the fused-vs-unfused colour tolerance (colours <= 1); depth weighs the same weights with m_i <= max m.
        # On an H100 the largest error is 5.1e-7 * max m (__expf weights, float32 segmented sums), 4x inside the bound.
        tol = 2e-6 * mmax
        print(f"{name} bg={with_bg}: max |depth - ref| {err.max():.3e}, max err / max m {(err / np.maximum(mmax, 1e-30)).max():.3e}")
        assert (err <= tol).all(), (name, float((err / np.maximum(mmax, 1e-30)).max()))
        # a live count on the device below the capacity: rays past the cut see no samples
        cut = int(off[100].item())
        count = torch.tensor([cut], dtype=torch.int64, device=cuda)
        off_cut = off.clone()
        off_cut[101:] = cut
        reuse_cut = None if reuse is None else (feat, src, off_cut)
        col2, ws2, depth2 = render_fused(*args, reuse=reuse_cut, count_dev=count, ray_offsets_dev=off_cut, want_depth=True)
        assert torch.equal(col2[:100], col[:100]) and torch.equal(depth2[:100], depth[:100]), name
        assert (ws2.view(-1)[100:] == 0).all() and (depth2.view(-1)[100:] == 0).all(), name


def test_render_with_depth_keeps_render_colour(cuda):
    from helpers import input_batch_of, make_pair
    from humanrf_b200.volume_rendering import prune_samples, render, render_with_depth

    _, m, frames = make_pair((6, 6), table_std=2.0)
    b = synthetic_rays(200, 300, frames, seed=17, ragged=True)
    ib = input_batch_of(b, cuda)
    prune_samples(ib, m, is_training=False)
    bg = torch.rand(200, 3, device=cuda)
    with torch.no_grad():
        a = render(ib, m, bg, is_training=False)
    out, depth = render_with_depth(ib, m, bg)
    assert torch.equal(out.color, a.color) and torch.equal(out.weights_sum, a.weights_sum)
    assert depth.shape == (200, 1) and depth.dtype == torch.float32
    w = out.weights_sum.view(-1)
    dist = depth.view(-1)[w > 1e-3] / w[w > 1e-3]
    assert (dist > 1.0).all() and (dist < 3.0).all()     # origins at |o| = 2, samples inside the unit cube
    assert (depth.view(-1)[w == 0] == 0).all()


def _ray_directions(inverse_kr, w, h):
    T = torch.as_tensor(inverse_kr).double().reshape(3, 3)
    x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    v = np.stack([x, y, np.ones_like(x)], -1).reshape(-1, 3) @ T.numpy()
    return v / np.linalg.norm(v, axis=1, keepdims=True), x.reshape(-1), y.reshape(-1)


def _min_distance_along(o, d, lo=0.0, hi=4.0, iters=60):
    """min over t in [lo, hi] of the distance from o + t d to E (convex along a line outside E): ternary search."""
    a, b = np.full(len(d), lo), np.full(len(d), hi)
    for _ in range(iters):
        m1, m2 = a + (b - a) / 3, b - (b - a) / 3
        f1 = _ellipsoid_distance(o + m1[:, None] * d)
        f2 = _ellipsoid_distance(o + m2[:, None] * d)
        a, b = np.where(f1 > f2, m1, a), np.where(f1 > f2, b, m2)
    return _ellipsoid_distance(o + ((a + b) / 2)[:, None] * d)


def test_confined_teacher_depth_maps(cuda):
    """sigma = 100 e^{12 s} over a +-1 sign grid of the ellipsoid E: the opaque transition lies within one level-0 cell
    diagonal (sqrt(3) / scale0) of E's surface, and a rendered distance is a sample midpoint average over at most a
    couple of steps there (sigma * step goes from 2e-7 to 6.5e3 across the transition), hence the band + 2 step."""
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.depth_maps import pixel_ray_norms

    m = confined_teacher(cuda)
    W, H, G = 96, 72, 128
    sc = make_scene(num_images=3, width=W, height=H, G=G, portrait_every=3)
    cams = _make_scene_world2pixel(3, W, H)
    og = OccupanyGrid(G, 1)
    handle = og.add_grid(torch.from_numpy(_sphere(G)).to(cuda))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    r = TileShardedRenderer(m, og, rays_per_batch=2000)          # several batches per view
    scale0 = float(m.feature_grids[0].layout.scale[0])
    band = np.sqrt(3) / scale0 + 2 * STEP
    for k in range(3):
        w2p, pos, w, h, landscape = cams[k]
        cam = dict(frame_numbers=t(sc["frame_numbers"][k:k + 1]), camera_numbers=t(sc["camera_numbers"][k:k + 1]),
                   grid_handles=torch.tensor([handle], dtype=torch.int64, device=cuda),
                   landscape=t(sc["landscape"][k:k + 1]), inverse_krs=t(sc["inverse_krs"][k:k + 1]),
                   camera_origins=t(sc["camera_origins"][k:k + 1]), aabb=t(sc["aabb"]), G=G, width=W, height=H)
        color, alpha, dist = r.render_range_maps(cam, 0, W * H)
        assert torch.equal(color, r.render_range(cam, 0, W * H))
        alpha, dist = alpha.double().cpu().numpy(), dist.double().cpu().numpy()
        d, px, py = _ray_directions(sc["inverse_krs"][k], w, h)
        o = sc["camera_origins"][k].astype(np.float64)
        solid = alpha >= 0.99
        assert solid.mean() > 0.02 and (dist[alpha == 0] == 0).all()
        p = o + dist[:, None] * d
        dd = _ellipsoid_distance(p[solid])
        assert dd.max() <= band, (k, dd.max(), band)
        # rays that miss E by more than the band carry no sample at all; rays that pass deeper than the band inside E
        # are opaque
        q = lambda x: ((x / RADII) ** 2).sum(1)
        dr, orr = d / RADII, o / RADII
        tstar = -(dr @ orr) / (dr * dr).sum(1)
        pin = o + tstar[:, None] * d
        miss = (q(pin) > 1) & (_min_distance_along(o, d) > band)
        deep = (q(pin) < 1) & (_ellipsoid_distance(pin) > band)
        assert miss.any() and deep.any()
        assert (alpha[miss] == 0).all() and (alpha[deep] >= 0.99).all()
        # reprojection through world2pixel lands on the pixel centre, in row-major order of this view's own width, and
        # its camera z is distance / |v|
        z = dist / pixel_ray_norms(t(sc["inverse_krs"][k]), w, h).cpu().numpy()
        pw = (w2p @ np.concatenate([p, np.ones((len(p), 1))], 1).T).T
        np.testing.assert_allclose(pw[solid, 0] / pw[solid, 2], px[solid], atol=2e-3)
        np.testing.assert_allclose(pw[solid, 1] / pw[solid, 2], py[solid], atol=2e-3)
        np.testing.assert_allclose(pw[solid, 2], z[solid], rtol=1e-5)
        print(f"view {k} ({'landscape' if landscape else 'portrait'} {w}x{h}): solid {solid.sum()}, max distance to E "
              f"{dd.max():.4f} (band {band:.4f}), miss {miss.sum()} deep {deep.sum()}")


def _loader(cuda):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    return ds, DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                  space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=64 * 48, camera_numbers=(0, 1, 2),
                  frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])


def test_render_depth_map_in_world_units(cuda):
    """z reprojects through the dataset camera's (unnormalised) world2pixel onto the pixel centre at that camera z."""
    from humanrf_b200.toolbox.depth_maps import render_depth_map

    m = confined_teacher(cuda)
    ds, dl = _loader(cuda)
    for c in (0, 2):
        dm = render_depth_map(m, dl, c, 16)
        cam = ds.cameras[c]
        assert dm.z.shape == (cam.height, cam.width) and dm.color.shape == (cam.height, cam.width, 3)
        alpha, dist, z = (x.double().cpu().numpy().reshape(-1) for x in (dm.alpha, dm.distance, dm.z))
        solid = alpha >= 0.99
        assert solid.mean() > 0.02 and (z[alpha == 0] == 0).all()
        d, px, py = _ray_directions(dl.all_inverse_krs[c].cpu(), cam.width, cam.height)
        p = cam.translation + dist[:, None] * d
        pw = (cam.projection_matrix_world2pixel() @ np.concatenate([p, np.ones((len(p), 1))], 1).T).T
        np.testing.assert_allclose(pw[solid, 0] / pw[solid, 2], px[solid], atol=2e-3)
        np.testing.assert_allclose(pw[solid, 1] / pw[solid, 2], py[solid], atol=2e-3)
        np.testing.assert_allclose(pw[solid, 2], z[solid], rtol=1e-5)


def test_export_depth_sequence(cuda, tmp_path):
    import cv2

    from humanrf_b200.toolbox.depth_maps import export_depth_sequence, render_depth_map
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid

    m = confined_teacher(cuda)
    ds, dl = _loader(cuda)
    pairs = [(0, 15), (2, 15), (0, 16)]
    out = tmp_path / "maps"
    paths = export_depth_sequence(m, dl, pairs, out, mask_threshold=0.5)
    assert sorted(str(p.relative_to(out)) for p in out.rglob("*") if p.is_file()) == sorted([
        "depths/Cam001/Cam001_depth000015.exr", "depths/Cam001/Cam001_depth000016.exr",
        "depths/Cam003/Cam003_depth000015.exr", "masks/Cam001/Cam001_mask000015.png",
        "masks/Cam001/Cam001_mask000016.png", "masks/Cam003/Cam003_mask000015.png"])
    for (c, f), (dp, mp) in zip(pairs, paths):
        baked = bake_occupancy_grid(m, f, torch.from_numpy(_sphere(64)).to(cuda))
        dm = render_depth_map(m, dl, c, f, grid=baked)
        z = cv2.imread(dp, cv2.IMREAD_UNCHANGED)
        ref = dm.z.cpu().numpy()
        assert z.dtype == np.float32 and np.array_equal(z.view(np.int32), ref.view(np.int32))
        assert (z[dm.alpha.cpu().numpy() == 0] == 0).all() and (z > 0).any()
        mask = cv2.imread(mp, cv2.IMREAD_UNCHANGED)
        assert mask.dtype == np.uint8 and np.array_equal(mask, (dm.alpha.cpu().numpy() >= 0.5).astype(np.uint8) * 255)
    with pytest.raises(RuntimeError):
        export_depth_sequence(m, dl, [(0, 15), (0, 99)], tmp_path / "bad")
    assert not (tmp_path / "bad").exists()


def test_depth_rejects_bad_inputs(cuda):
    from humanrf_b200 import _lib as L
    from humanrf_b200.volume_rendering import ray_offsets, render_with_depth
    from helpers import input_batch_of, make_pair
    from humanrf_b200.toolbox.depth_maps import export_depth_sequence, render_depth_map

    # NULL depth through the C ABI
    m, g, nr, _ = _ragged_batch(cuda)
    nat = m.native()
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"])
    off = ray_offsets(g["ri"], nr)
    col, ws = torch.empty(nr, 3, device=cuda), torch.empty(nr, device=cuda)
    wsp = torch.empty(int(L.lib().hrf_render_fused_workspace_bytes(g["t"].shape[0])), dtype=torch.uint8, device=cuda)
    with pytest.raises(RuntimeError):
        L.check(L.lib().hrf_render_fused_depth(C.byref(nat.field), C.byref(samples), off.data_ptr(), nr, STEP, None, None,
                                               None, col.data_ptr(), ws.data_ptr(), None, wsp.data_ptr(), L.stream()))
    # a CPU batch
    _, m2, frames = make_pair((6,), table_std=2.0)
    b = synthetic_rays(20, 50, frames, seed=3)
    ib = input_batch_of(b, cuda)
    ib.sample_distances = ib.sample_distances.cpu()
    with pytest.raises(RuntimeError):
        render_with_depth(ib, m2, None)
    # grids of the wrong dtype / device / shape, unknown frames and cameras
    mc = confined_teacher(cuda)
    _, dl = _loader(cuda)
    good = torch.from_numpy(_sphere(64)).to(cuda)
    for grid in (good.float(), good.cpu(), good[0], good.bool()):
        with pytest.raises(RuntimeError):
            render_depth_map(mc, dl, 0, 15, grid=grid)
    for c, f in ((0, 99), (0, 14), (7, 15), (-1, 15)):
        with pytest.raises(RuntimeError):
            render_depth_map(mc, dl, c, f)
        with pytest.raises(RuntimeError):
            export_depth_sequence(mc, dl, [(c, f)], "/nonexistent/never_written")
