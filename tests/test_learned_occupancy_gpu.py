"""Learned occupancy grid on the H100 (humanrf_b200/csrc/occupancy_bake.cu, toolbox/learned_occupancy.py):
the fused bake against the same contract built from the public query-form density, against the CPU oracle, and the
user-visible claim: rendering a confined scene with the baked grid gives the same image from far fewer candidates."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from helpers import make_pair
import bake_oracle as O

pytestmark = pytest.mark.gpu

STEP, THRE = 4e-4, 1e-4


def _sphere(G, r=0.42):
    c = (np.arange(G) + 0.5) / G - 0.5
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    return ((x * x + y * y + z * z <= r * r) * 255).astype(np.uint8)


def _psnr(a, b):
    mse = float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))
    return float("inf") if mse == 0 else -10.0 * np.log10(mse)


def _sharp_pair(segs, cuda, cam_emb=0):
    """make_pair's table_std 6 model with the density row of the sigma net scaled by 16 (exact in bf16): densities span
    many decades, so live and dead voxels both occur."""
    om, m, frames = make_pair(segs, table_std=6.0, device=cuda, cam_emb=cam_emb)
    om.w_sigma[1][0] *= 16.0
    with torch.no_grad():
        m.sigma_net.params[32 * 64:32 * 64 + 64] *= 16.0
    return om, m, frames


def unfused_bake(m, frame, hull, step):
    """The contract built from the public API: 8 positions per hull voxel in torch, HumanRF.density (query form),
    per-voxel max, alpha test, max_pool3d dilation, AND with the hull."""
    from humanrf_b200.scene_representation.query_io import QueryInput

    G = hull.shape[0]
    z, y, x = torch.nonzero(hull, as_tuple=True)
    s = torch.arange(8, device=hull.device)
    cols = [(i.to(torch.float32)[:, None] + 0.25 + 0.5 * h.to(torch.float32)[None, :]) / float(G) - 0.5
            for i, h in zip((x, y, z), (s & 1, (s >> 1) & 1, (s >> 2) & 1))]
    pos = torch.stack(cols, -1).reshape(-1, 3).contiguous()
    with torch.no_grad():
        sigma = m.density(QueryInput(is_training=False, positions=pos,
                                     frame_numbers=torch.full((pos.shape[0],), frame, dtype=torch.int32,
                                                              device=hull.device))).density
    msig = sigma.view(-1, 8).amax(1)
    max_sigma = torch.zeros(hull.shape, dtype=torch.float32, device=hull.device)
    max_sigma[z, y, x] = msig
    live = torch.zeros(hull.shape, dtype=torch.bool, device=hull.device)
    live[z, y, x] = (1 - torch.exp(-msig * step)) >= THRE
    dil = Fn.max_pool3d(live.float()[None, None], 3, stride=1, padding=1)[0, 0] > 0
    out = ((hull != 0) & dil).to(torch.uint8) * 255
    return out, max_sigma, live


CASES = [((50,), 64, (15, 64), 0), ((50,), 256, (40,), 0), ((100, 100, 50), 64, (114, 115, 214, 215), 0),
         ((100, 100, 50), 256, (114, 115), 0), ((50,), 64, (15, 30), 2)]


@pytest.mark.parametrize("segs,G,frames,cam_emb", CASES, ids=["seg50-G64", "seg50-G256", "seg100x2-50-G64",
                                                              "seg100x2-50-G256", "seg50-G64-camemb2"])
def test_fused_bake_equals_unfused_bitwise(cuda, segs, G, frames, cam_emb):
    from humanrf_b200.synthetic_scene import ellipsoid_grid
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid

    _, m, _ = _sharp_pair(segs, cuda, cam_emb)
    hull = torch.from_numpy(ellipsoid_grid(G)).to(cuda)
    nh = int((hull != 0).sum())
    for frame in frames:
        # the default step, then a step that puts the threshold at the 99th percentile of the voxel maxima: about 1 %
        # of the voxels stay live, so the dilation decides most of the grid
        for step in (STEP, None):
            if step is None:
                m99 = float(torch.quantile(ms[hull != 0].double(), 0.99))
                step = float(-np.log1p(-THRE) / m99)
            out, ms = bake_occupancy_grid(m, frame, hull, step, return_max_sigma=True)
            ref_out, ref_ms, live = unfused_bake(m, frame, hull, step)
            torch.cuda.synchronize()
            assert out.dtype == torch.uint8 and out.shape == hull.shape and out.device == hull.device
            assert torch.equal(ms.view(torch.int32), ref_ms.view(torch.int32)), "max_sigma differs"
            assert torch.equal(out, ref_out), f"grid differs at {int((out != ref_out).sum())} voxels"
            assert torch.equal(bake_occupancy_grid(m, frame, hull, step), out)
            nl, no = int(live.sum()), int((out != 0).sum())
            print(f"segs={segs} G={G} frame={frame} step={step:g}: hull {nh} live {nl} out {no}")
            if step != STEP:
                assert 0 < nl < nh and no < nh


def test_bake_against_cpu_oracle(cuda):
    """G = 24 against the fp32 CPU restatement: max_sigma within the density tolerance of DESIGN section 1 (rel 4e-2);
    flags may differ only where the oracle's m lies within that band of the threshold (and, for the dilated grid, next
    to such a voxel).  A step of 1e-6 puts the threshold (m = 100) inside this model's density range."""
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid

    om, m, frames = make_pair((50,), table_std=6.0, device=cuda)
    G, step, frame = 24, 1e-6, 20
    hull_np = _sphere(G)
    out, ms = bake_occupancy_grid(m, frame, torch.from_numpy(hull_np).to(cuda), step, return_max_sigma=True)
    ref_out, ref_ms = O.bake_occupancy_grid(om, frame, hull_np, step, THRE)
    out, ms = out.cpu().numpy(), ms.cpu().numpy()
    h = hull_np != 0
    rel = np.abs(ms[h].astype(np.float64) - ref_ms[h]) / np.abs(ref_ms[h])
    assert rel.max() <= 4e-2, rel.max()
    assert (ms[~h] == 0).all()
    m_thr = -np.log1p(-THRE) / step
    band = h & (np.abs(ref_ms.astype(np.float64) - m_thr) <= 4e-2 * m_thr)
    live = h & ((1 - np.exp(-ms * np.float32(step))) >= THRE)
    ref_live = h & ((1 - np.exp(-ref_ms * np.float32(step))) >= THRE)
    assert not ((live != ref_live) & ~band).any()
    near_band = Fn.max_pool3d(torch.from_numpy(band).float()[None, None], 3, 1, 1)[0, 0].numpy() > 0
    assert not ((out != ref_out) & ~near_band).any()
    print(f"hull {h.sum()} live {live.sum()} oracle live {ref_live.sum()} band {band.sum()} "
          f"grid mismatches {(out != ref_out).sum()} max rel {rel.max():.2e}")
    assert 0 < ref_live.sum() < h.sum()


# ---------------------------------------------------------------------------------------------------- confined scene
def confined_teacher(cuda, seed=0):
    """A model whose density is known: feature 0 of the dense level 0 of the xyz grid is +1 at vertices inside the
    ellipsoid E (radii 0.2 / 0.3 / 0.15) and -1 outside, vectors[3] (time) is 1 for feature 0, everything else of the
    tables is zero; the sigma net computes h0 = 12 s(x) (W1[0] = e0, W1[1] = -e0, W2[0] = (12, -12, 0, ...)), so sigma is
    100 e^{+-12} away from E's boundary.  The colour net keeps its random initialisation."""
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    torch.manual_seed(seed)
    frames = tuple(range(15, 21))
    m = HumanRF(sorted_frame_numbers=frames, segment_sizes=(6,), **MODEL_KW)
    with torch.no_grad():
        fg = m.feature_grids[0]
        for g in fg.grids():
            g.zero_()
        lay = fg.layout
        res, off, scale = int(lay.res[0]), int(lay.offset[0]), float(lay.scale[0])
        assert not (lay.hashed_mask & 1) and res ** 3 <= int(lay.size[0])
        i = torch.arange(res, dtype=torch.float64)
        c = (i - 0.5) / scale - 0.5                     # world coordinate of vertex i (tcnn: pos = scale * x + 0.5)
        zz, yy, xx = torch.meshgrid(c, c, c, indexing="ij")
        inside = (xx / 0.2) ** 2 + (yy / 0.3) ** 2 + (zz / 0.15) ** 2 <= 1.0
        iz, iy, ix = torch.meshgrid(torch.arange(res), torch.arange(res), torch.arange(res), indexing="ij")
        idx = (ix + iy * res + iz * res * res).reshape(-1)
        fg.grids()[0].view(-1, 2)[off + idx, 0] = torch.where(inside.reshape(-1), 1.0, -1.0).float()
        fg.vectors.zero_()
        fg.vectors[3, :, 0] = 1.0
        w1, w2 = torch.zeros(64, 32), torch.zeros(16, 64)
        w1[0, 0], w1[1, 0] = 1.0, -1.0
        w2[0, 0], w2[0, 1] = 12.0, -12.0
        m.sigma_net.params.copy_(torch.cat((w1.reshape(-1), w2.reshape(-1))))
    return m.to(cuda)


def test_confined_scene_renders_the_same_from_fewer_candidates(cuda):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid

    m = confined_teacher(cuda)
    W, H, G = 160, 120, 128
    sc = make_scene(num_images=3, width=W, height=H, G=G, portrait_every=0)
    hull = torch.from_numpy(_sphere(G)).to(cuda)
    og = OccupanyGrid(G, 4)
    hull_handle = og.add_grid(hull)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    r = TileShardedRenderer(m, og, rays_per_batch=W * H)
    imgs = {"hull": [], "baked": []}
    cand = {"hull": 0, "baked": 0}
    for k in range(3):
        frame = int(sc["frame_numbers"][k])
        baked = bake_occupancy_grid(m, frame, hull)
        assert int((baked != 0).sum()) < int((hull != 0).sum())
        for kind, handle in (("hull", hull_handle), ("baked", og.add_grid(baked))):
            cam = dict(frame_numbers=t(sc["frame_numbers"][k:k + 1]), camera_numbers=t(sc["camera_numbers"][k:k + 1]),
                       grid_handles=torch.tensor([handle], dtype=torch.int64, device=cuda),
                       landscape=t(sc["landscape"][k:k + 1]), inverse_krs=t(sc["inverse_krs"][k:k + 1]),
                       camera_origins=t(sc["camera_origins"][k:k + 1]), aabb=t(sc["aabb"]), G=G, width=W, height=H)
            imgs[kind].append(r.render_range(cam, 0, W * H).cpu().numpy())
            cand[kind] += r.last_stats["candidate_samples"]
    a, b = np.concatenate(imgs["hull"]), np.concatenate(imgs["baked"])
    psnr = _psnr(b, a)
    print(f"confined scene, 3 x {W}x{H}: candidate samples hull {cand['hull']} baked {cand['baked']} "
          f"({cand['baked'] / cand['hull']:.3f}x), PSNR(baked vs hull) {psnr:.2f} dB, "
          f"object pixels {(a.sum(1) > 0).mean():.2%}")
    assert (a.sum(1) > 0).mean() > 0.02
    assert psnr >= 40.0
    assert cand["baked"] <= 0.5 * cand["hull"]


def test_learned_occupancy_dataset_in_a_test_loader(cuda, monkeypatch):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox import learned_occupancy as LO
    from humanrf_b200.volume_rendering import prune_samples, render

    m = confined_teacher(cuda)
    ds = SyntheticDataset(G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    calls = []
    real_bake = LO.bake_occupancy_grid

    def counting_bake(model, frame, hull, *a, **kw):
        calls.append(int(frame))
        return real_bake(model, frame, hull, *a, **kw)

    monkeypatch.setattr(LO, "bake_occupancy_grid", counting_bake)
    wrapped = LO.LearnedOccupancyDataset(ds, m)
    assert wrapped.frames == ds.frames and wrapped.get_aabb() is ds.get_aabb()
    seq = [(0, 15), (1, 16), (2, 15), (3, 16)]

    def images(dataset):
        dl = DL(dataset=dataset, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=64 * 48, camera_numbers=(0, 1, 2, 3, 4),
                frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=seq)
        out, samples = [], 0
        for b in dl:
            samples += int(b.sample_distances.numel())
            mask = b.ray_masks.view(-1)
            img = torch.zeros((mask.numel(), 3), device=cuda)
            if int(b.num_rays) > 0:
                prune_samples(b, m, is_training=False)
                with torch.no_grad():
                    img[mask] = render(b, m, torch.zeros(3, device=cuda), is_training=False).color
            out.append(img.cpu().numpy())
        return np.concatenate(out), samples

    ref, n_hull = images(ds)
    got, n_baked = images(wrapped)
    assert sorted(calls) == [15, 16], calls                  # each frame baked once, whatever the loader asks
    for f in (15, 16):
        g = wrapped.get_occupancy_grid(f)
        assert isinstance(g, np.ndarray) and g.dtype == np.uint8 and g.shape == (64, 64, 64)
        np.testing.assert_array_equal(g, real_bake(m, f, torch.from_numpy(_sphere(64)).to(cuda)).cpu().numpy())
    assert sorted(calls) == [15, 16]
    psnr = _psnr(got, ref)
    print(f"TEST loader, {len(seq)} images: candidate samples hull {n_hull} baked {n_baked}, PSNR {psnr:.2f} dB")
    assert (ref.sum(1) > 0).mean() > 0.02
    assert psnr >= 40.0 and n_baked < n_hull


def test_bake_rejects_bad_inputs(cuda):
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid

    _, m, frames = make_pair((6,), device=cuda)
    good = torch.from_numpy(_sphere(16)).to(cuda)
    assert bake_occupancy_grid(m, frames[0], good).shape == good.shape
    bad = [good.float(), good.bool(), good[:, :, :8].contiguous(), good[0], good.cpu(), good.transpose(0, 2),
           good.cpu().numpy()]
    for h in bad:
        with pytest.raises(RuntimeError):
            bake_occupancy_grid(m, frames[0], h)
    for f in (frames[0] - 1, frames[-1] + 1, -1, 10 ** 6):
        with pytest.raises(RuntimeError):
            bake_occupancy_grid(m, f, good)
