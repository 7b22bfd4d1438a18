"""The error map on the H100 (humanrf_b200/csrc/error_map.cu, toolbox/error_map.py, DESIGN.md §3.20): accumulate, update
(EMA, weights, scan) and draw bit for bit against tests/error_map_oracle.py, the reset, the state, every refusal, the
loader with and without a map, FusedTrainer with a map against the noise of its own float atomics, and the mechanism
end to end: after training on a scene with one high-frequency region, the share of drawn rays in that region is the one
the oracle predicts from the map read back, and well above the region's pixel share."""
import ctypes as C

import numpy as np
import pytest
import torch

import error_map_oracle as EO

pytestmark = pytest.mark.gpu


def _geometry(landscape, W, H, T, cuda):
    from humanrf_b200 import _lib as L

    ls = torch.tensor(landscape, dtype=torch.bool, device=cuda)
    g = L.ErrorMapGeometry()
    g.landscape_modes, g.num_slots, g.image_width, g.image_height, g.tile = ls.data_ptr(), len(landscape), W, H, T
    return g, ls, EO.Geometry(landscape, W, H, T)


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _accumulate(cuda, g, pixels, color, wsum, rgba, bg, table=None, cams=None, n=None):
    from humanrf_b200 import _lib as L

    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
    s = torch.zeros(n, dtype=torch.int64, device=cuda)
    c = torch.zeros(n, dtype=torch.int32, device=cuda)
    err = torch.zeros(1, dtype=torch.int32, device=cuda)
    ins = [d(color), d(wsum), d(rgba), d(bg), d(pixels)]
    tab, cam = d(table), d(cams)
    L.check(L.lib().hrf_error_map_accumulate(*(L.ptr(t) for t in ins), len(pixels), L.ptr(tab), L.ptr(cam),
                                             0 if table is None else table.shape[0], 0.01, C.byref(g), s.data_ptr(),
                                             c.data_ptr(), err.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    return _u64(s), c.cpu().numpy().view(np.uint32), int(err.cpu()[0])


def _rays(R, rng):
    color, rgba, bg = (rng.uniform(0, 1, (R, k)).astype(np.float32) for k in (3, 4, 3))
    rgba[:, 3] = rng.choice([0.0, 1.0, 0.5], R)
    near = rng.uniform(0, 1, R) < 0.5         # half the rays in the quadratic branch
    color[near] = (rgba[near, :3] * rgba[near, 3:] + bg[near] * (1 - rgba[near, 3:])
                   + rng.normal(0, 3e-3, (near.sum(), 3))).astype(np.float32)
    wsum = rng.uniform(0, 1, R).astype(np.float32)
    return color, wsum, rgba, bg


@pytest.mark.parametrize("response", [False, True])
@pytest.mark.parametrize("spread", ["pool", "one_tile"])
@pytest.mark.parametrize("R", [1, 4096, 65536, (1 << 20) + 3])
def test_accumulate_matches_oracle(cuda, R, spread, response):
    g, _ls, geo = _geometry([True, False, False, True, True], 97, 61, 16, cuda)
    rng = np.random.default_rng(R + 7 * response)
    color, wsum, rgba, bg = _rays(R, rng)
    if spread == "pool":
        pixels = rng.integers(0, geo.B * geo.P, R)
    else:                                       # every ray in one border tile of a portrait slot: contention
        t = 2 * geo.nt - 1
        slot, x0, y0, cw, ch, w = geo.tile_extent(np.array([t]))
        k = rng.integers(0, int(cw[0] * ch[0]), R)
        pixels = int(slot[0]) * geo.P + (int(y0[0]) + k // int(cw[0])) * int(w[0]) + int(x0[0]) + k % int(cw[0])
        assert (geo.tile_of_pixel(pixels) == t).all()
    table = cams = None
    if response:
        table = np.concatenate((rng.uniform(-0.2, 0.2, (6, 3)), rng.uniform(-0.05, 0.05, (6, 3))), 1).astype(np.float32)
        table[0] = 0.0
        cams = rng.integers(-1, 7, R).astype(np.int32)     # out-of-range cameras take the identity
    s, c, err = _accumulate(cuda, g, pixels, color, wsum, rgba, bg, table, cams, geo.num_tiles)
    e = EO.ray_error(color, wsum, rgba, bg, 0.01, table, cams)
    es, ec, eerr = EO.accumulate(geo, pixels, e)
    assert err == 0 == eerr
    assert np.array_equal(c, ec) and np.array_equal(s, es)


def test_out_of_range_pixel_sets_the_error_bit(cuda):
    g, _ls, geo = _geometry([True, False], 33, 20, 8, cuda)
    rng = np.random.default_rng(1)
    color, wsum, rgba, bg = _rays(300, rng)
    pixels = rng.integers(0, geo.B * geo.P, 300)
    pixels[[5, 77]] = [-1, geo.B * geo.P]
    s, c, err = _accumulate(cuda, g, pixels, color, wsum, rgba, bg, n=geo.num_tiles)
    es, ec, _ = EO.accumulate(geo, pixels, EO.ray_error(color, wsum, rgba, bg, 0.01))
    assert err == 1 and int(c.sum()) == 298 and np.array_equal(s, es) and np.array_equal(c, ec)


@pytest.mark.parametrize("shape", [((True, False, False, True, False, True), 97, 61, 16),
                                   ((False, True, True), 37, 23, 7), ((True, False) * 100, 1022, 750, 16)])
def test_update_and_draw_match_oracle(cuda, shape):
    from humanrf_b200 import _lib as L

    landscape, W, H, T = shape
    g, _ls, geo = _geometry(list(landscape), W, H, T, cuda)
    n = geo.num_tiles
    lib = L.lib()
    assert int(lib.hrf_error_map_num_tiles(C.byref(g), 1.0)) == n
    rng = np.random.default_rng(n)
    ema = rng.uniform(0, 0.02, n).astype(np.float32)
    ema[rng.choice(n, n // 10, replace=False)] = 1.0
    R = 50000
    color, wsum, rgba, bg = _rays(R, rng)
    pixels = rng.integers(0, geo.B * geo.P, R)
    e = EO.ray_error(color, wsum, rgba, bg, 0.01)
    es, ec, _ = EO.accumulate(geo, pixels, e)
    ema_dev = torch.from_numpy(ema).to(cuda)
    s_dev = torch.from_numpy(es.view(np.int64)).to(cuda)
    c_dev = torch.from_numpy(ec.view(np.int32)).to(cuda)
    cdf = torch.empty(n, dtype=torch.int64, device=cuda)
    ws = torch.empty(int(lib.hrf_error_map_workspace_bytes(n)), dtype=torch.uint8, device=cuda)
    beta, floor = 0.3, 1e-5
    L.check(lib.hrf_error_map_update(C.byref(g), ema_dev.data_ptr(), s_dev.data_ptr(), c_dev.data_ptr(), beta, floor,
                                     cdf.data_ptr(), ws.data_ptr(), L.stream()))
    new, ecdf = EO.update(geo, ema, es, ec, beta, floor)
    torch.cuda.synchronize()
    assert np.array_equal(ema_dev.cpu().numpy().view(np.uint32), new.view(np.uint32))
    assert np.array_equal(_u64(cdf), ecdf)
    assert int(s_dev.abs().sum()) == 0 and int(c_dev.abs().sum()) == 0
    for seed, counter, R, f in ((3, 0, 100003, 0.25), (2 ** 64 - 1, 12345, 4096, 0.0), (7, 1, 999, 1.0),
                                (9, 2, 1, 0.5)):
        out = torch.empty(R, dtype=torch.int64, device=cuda)
        L.check(lib.hrf_error_map_draw(cdf.data_ptr(), C.byref(g), seed, counter, R, f, out.data_ptr(), L.stream()))
        eo, _ = EO.draw(geo, ecdf, seed, counter, R, f)
        assert np.array_equal(out.cpu().numpy(), eo), (seed, counter, R, f)


# ------------------------------------------------------------------------------------------------ ErrorMap on a loader
def _loader(cuda, batch=4096, mode=None, dataset=None, **kw):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = dataset if dataset is not None else SyntheticDataset(num_cameras=5, frames=range(15, 18))
    mode = DL.Mode.TRAINING if mode is None else mode
    args = dict(max_num_frames_per_batch=2, use_mask=False, filter_light_bloom=False) if mode == DL.Mode.TRAINING \
        else dict(use_mask=False, filter_light_bloom=False, render_sequence=[(0, 15)])
    args.update(kw)
    return DL(dataset=ds, device="cuda", mode=mode, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=batch, camera_numbers=tuple(range(5)),
              frame_numbers=tuple(ds.frames), max_buffer_size=8, **args)


def test_loader_without_a_map_draws_what_it_drew_before(cuda):
    torch.manual_seed(3)
    np.random.seed(3)
    dl = _loader(cuda)
    assert dl.ray_source is None
    torch.manual_seed(11)
    next(dl)
    got = dl.last_ray_indices.clone()
    torch.manual_seed(11)
    exp = torch.randint(0, dl.buffer_size * dl.num_pixels_per_camera, size=(dl.batch_size,), dtype=torch.int64,
                        device=cuda)
    assert torch.equal(got, exp)


def test_loader_with_a_map_draws_the_oracle_and_resets_reloaded_slots(cuda):
    from humanrf_b200.toolbox.error_map import ErrorMap

    np.random.seed(4)
    dl = _loader(cuda, replace_per_next=1)
    em = ErrorMap(dl, tile=8, uniform_fraction=0.3, seed=5, rank=2)
    assert dl.ray_source is em and em.tiles_per_slot == 8 * 6
    geo = EO.Geometry(dl.landscape_mode_cuda.cpu().numpy(), 64, 48, 8)
    with torch.no_grad():
        em.ema.copy_(torch.linspace(0, 0.5, em.num_tiles, device=cuda))
    em.update()
    cdf = EO.cdf_of(geo, em.ema.cpu().numpy(), em.floor)
    it = iter(dl)
    for k, batch in enumerate((4096, 1000)):
        dl.batch_size = batch
        reload_slot = dl.pair_load_index % dl.buffer_size
        before = em.tile_errors()
        next(it)
        after = em.tile_errors()
        assert float(after[reload_slot].min()) == 1.0 == float(after[reload_slot].max())
        keep = [s for s in range(dl.buffer_size) if s != reload_slot]
        assert torch.equal(after[keep], before[keep])
        # the reset writes the EMA only: the draw reads the CDF of the last update
        assert np.array_equal(_u64(em.cdf), cdf)
        exp, _ = EO.draw(geo, cdf, 5 + 2, k, batch, 0.3)
        assert np.array_equal(dl.last_ray_indices.cpu().numpy(), exp)
    assert em.counter == 2
    em.update()
    assert np.array_equal(_u64(em.cdf), EO.cdf_of(geo, em.ema.cpu().numpy(), em.floor))
    dens = em.sampling_density()
    assert dens.shape == (dl.buffer_size, em.tiles_per_slot) and abs(float(dens.sum()) - 1.0) < 1e-12


def test_reset_state_round_trip_and_refusals(cuda):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.error_map import ErrorMap

    np.random.seed(5)
    dl = _loader(cuda)
    with pytest.raises(ValueError, match="TRAINING"):
        ErrorMap(_loader(cuda, mode=DL.Mode.VALIDATION))
    for kw in ({"tile": 0}, {"tile": 2.5}, {"uniform_fraction": 1.01}, {"uniform_fraction": -1e-9}, {"beta": 1.5},
               {"floor": 1e-9}, {"prior": -1.0}, {"rank": -1}):
        with pytest.raises(ValueError):
            ErrorMap(dl, **kw)
    em = ErrorMap(dl, tile=16, seed=9)
    with torch.no_grad():
        em.ema.uniform_(0, 0.1)
    em.update()
    cdf = em.cdf.clone()
    em.reset_slot(3)
    assert float(em.tile_errors()[3].min()) == 1.0 and float(em.tile_errors()[2].max()) < 0.1
    assert torch.equal(em.cdf, cdf)                     # rebuilt by the next update, not by the reset
    em.update()
    with pytest.raises(ValueError):
        em.reset_slot(dl.buffer_size)
    em.draw(100)
    st = em.state_dict()
    assert st["counter"] == 1 and st["seed"] == 9 and st["geometry"] == em.geometry
    other = ErrorMap(_loader(cuda), tile=16)
    other.load_state_dict(st)
    assert torch.equal(other.ema, em.ema) and torch.equal(other.cdf, em.cdf) and other.counter == 1
    assert torch.equal(other.draw(777), em.draw(777))
    for bad in ({**st, "geometry": {**st["geometry"], "tile": 8}}, {**st, "ema": st["ema"][:-1]},
                {**st, "ema": st["ema"].double()}, {**st, "ema": torch.full_like(st["ema"], float("nan"))},
                {**st, "ema": torch.full_like(st["ema"], 2.0)}, {**st, "ema": torch.full_like(st["ema"], -1e-3)},
                {**st, "counter": -1}, {**st, "counter": 1.5}, {k: v for k, v in st.items() if k != "ema"},
                {k: v for k, v in st.items() if k != "seed"}, {k: v for k, v in st.items() if k != "counter"},
                {**st, "geometry": None}, [("ema", st["ema"])]):
        with pytest.raises(ValueError):
            other.load_state_dict(bad)
    assert torch.equal(other.ema, em.ema)
    # a pool whose total weight could overflow 64 bits
    with pytest.raises(ValueError, match="overflow"):
        ErrorMap(dl, tile=16, prior=2.0 ** 40)
    with pytest.raises(ValueError, match="overflow"):
        ErrorMap(dl, tile=16, floor=1e12)
    # an out-of-range pixel from a step is reported
    em.error.fill_(1)
    with pytest.raises(RuntimeError):
        em.state_dict()


def _fixed_batch(cuda, R=4096):
    from humanrf_b200.synthetic import synthetic_rays

    b = synthetic_rays(R, 32, list(range(15, 21)), seed=4)
    return {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba")}


def test_trainer_with_a_map_refuses_bad_pixels(cuda):
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.toolbox.error_map import ErrorMap
    from humanrf_b200.training import FusedTrainer

    np.random.seed(6)
    em = ErrorMap(_loader(cuda), tile=16)
    g = _fixed_batch(cuda)
    m, _ = make_model((6,), seed=1, device=cuda)
    with pytest.raises(ValueError, match="rank"):
        FusedTrainer(m, error_map=ErrorMap(_loader(cuda), rank=1))
    tr = FusedTrainer(m, error_map=em)
    args = (g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], 4096)
    with pytest.raises(ValueError, match="pixels"):
        tr.step(*args)
    with pytest.raises(ValueError, match="entries"):
        tr.step(*args, pixels=torch.zeros(4095, dtype=torch.int64, device=cuda))


def test_trainer_update_is_the_one_without_a_map(cuda):
    """For a fixed batch, loss, sample count and parameters with a map differ from a run without one no more than two
    runs without one differ from each other (the order of the float atomics in the loss and the gradient scatter)."""
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.toolbox.error_map import ErrorMap
    from humanrf_b200.training import FusedTrainer

    np.random.seed(7)
    dl = _loader(cuda)
    g = _fixed_batch(cuda)
    pixels = torch.randint(0, dl.buffer_size * dl.num_pixels_per_camera, (4096,), device=cuda)

    def run(em):
        m, _ = make_model((6,), seed=1, device=cuda)
        tr = FusedTrainer(m, error_map=em)
        out = []
        for _ in range(3):
            loss = tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], 4096, return_loss=True,
                           pixels=pixels if em is not None else None)
            out.append((loss, int(tr.last["samples"])))
        return out, torch.cat([p.detach().reshape(-1) for p in m.hot_parameters()])

    (a, pa), (b, pb) = run(None), run(None)
    em = ErrorMap(dl, tile=16)
    (c, pc) = run(em)
    assert int(em.tile_count.abs().sum()) == 0 and float(em.ema.min()) < 1.0      # the map was fed and updated
    assert a[0][1] == c[0][1]                           # the first step prunes from identical parameters
    for (la, na), (lb, nb), (lc, nc) in zip(a, b, c):
        assert abs(lc - la) <= 4 * abs(lb - la) + 1e-5 * abs(la)
        assert abs(nc - na) <= 4 * abs(nb - na) + 2
    noise = float((pb - pa).norm())
    assert float((pc - pa).norm()) <= 4 * noise + 1e-6 * float(pa.norm())


# ------------------------------------------------------------------------------------------------ mechanism
class _PatchDataset:
    """SyntheticDataset whose images are flat grey except one high-frequency region: a random-pixel patch in the
    top-left 24 x 16 pixels of every camera."""

    REGION = (24, 16)

    def __init__(self):
        from humanrf_b200.synthetic_scene import SyntheticDataset

        self.base = SyntheticDataset(num_cameras=5, frames=range(15, 16))
        self.frames = self.base.frames

    def __getattr__(self, name):
        return getattr(self.base, name)

    def get_rgb(self, camera_number, frame_number, normalize=True):
        rgb = np.full((48, 64, 3), 0.5, np.float32)
        rng = np.random.default_rng(camera_number)
        w, h = self.REGION
        rgb[:h, :w] = rng.integers(0, 256, (h, w, 3)) / np.float32(255)
        return rgb

    def get_mask(self, camera_number, frame_number, normalize=True):
        return np.ones((48, 64, 1), np.float32)


def test_map_draws_the_hard_region_as_the_oracle_predicts(cuda):
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.toolbox.error_map import ErrorMap
    from humanrf_b200.training import FusedTrainer

    torch.manual_seed(0)
    np.random.seed(0)
    dl = _loader(cuda, dataset=_PatchDataset(), max_num_frames_per_batch=1)
    em = ErrorMap(dl, tile=8, uniform_fraction=0.25, beta=0.5, seed=1)
    m, _ = make_model((1,), seed=1, device=cuda)
    tr = FusedTrainer(m, error_map=em)
    for _ in range(150):
        ib = next(dl)
        px = dl.last_ray_indices[ib.ray_masks.view(-1)]
        tr.step(ib.ray_origins.contiguous(), ib.ray_directions.contiguous(), ib.frame_numbers.view(-1).contiguous(),
                ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous(), ib.rgba.contiguous(),
                ib.num_rays, pixels=px)
    em.check()
    geo = EO.Geometry(dl.landscape_mode_cuda.cpu().numpy(), 64, 48, 8)
    ema = em.tile_errors().view(-1).cpu().numpy()
    cdf = EO.cdf_of(geo, ema, em.floor)
    assert np.array_equal(_u64(em.cdf), cdf)
    idx = np.arange(geo.B * geo.P)
    _, x, y = EO.sampler_pixel_xy(geo, idx)
    region_tiles = np.unique(geo.tile_of_pixel(idx[(x < 24) & (y < 16)]))
    R = 1 << 20
    predicted = float(EO.target_probabilities(geo, cdf, em.uniform_fraction, R)[region_tiles].sum())
    share = 24 * 16 / (64 * 48)
    drawn = em.draw(R).cpu().numpy()
    _, x, y = EO.sampler_pixel_xy(geo, drawn)
    observed = float(((x < 24) & (y < 16)).mean())
    sigma = np.sqrt(predicted * (1 - predicted) / R)
    print(f"region pixel share {share:.4f}; predicted draw share {predicted:.4f} ({predicted / share:.2f}x), "
          f"observed {observed:.4f}")
    assert abs(observed - predicted) < 5 * sigma
    assert predicted > 2.0 * share


# ------------------------------------------------------------------------------------------------ the loss kernels' term
@pytest.mark.parametrize("response", [False, True])
def test_ray_error_is_the_loss_kernels_term(cuda, response):
    """e_r is the term the loss kernels sum.  One ray per launch, bce_weight = 0, and two of the three channels exactly
    on their target (x = 0, so they add +0): the kernel's loss is then fl(h inv3r) with inv3r = fl(1/3) for the one
    remaining channel's Huber value h, which pins the oracle's h (and through test_accumulate_matches_oracle the error
    map kernel's e_r) to hrf_train_loss and hrf_train_loss_response as compiled, in both Huber branches."""
    from humanrf_b200 import _lib as L

    lib = L.lib()
    rng = np.random.default_rng(11 + response)
    inv3 = np.float32(1.0) / np.float32(3.0)
    n_quad = 0
    for i in range(64):
        color, wsum, rgba, bg = _rays(1, rng)
        k = i % 3
        table = cams = None
        if response:
            table = np.zeros((2, 6), np.float32)
            table[1, k], table[1, 3 + k] = rng.uniform(-0.2, 0.2), rng.uniform(-0.05, 0.05)
            cams = np.array([1], np.int32)
        m = rgba[:, 3]
        for j in range(3):
            if j != k:    # x = color - gt = 0 exactly, and the identity response there
                color[:, j] = EO.target(m, rgba[:, j], bg[:, j], response)
        if i % 2:          # the quadratic branch
            color[:, k] = (color[:, k] + np.float32(rng.uniform(-5e-3, 5e-3))).astype(np.float32)
            if response:
                table[1, k] = table[1, 3 + k] = 0.0
        h = EO.ray_error(color, wsum, rgba, bg, 0.01, table, cams)
        n_quad += int(h[0] < 0.5 * 0.01 * 0.01)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
        c_, w_, r_, b_ = d(color), d(wsum), d(rgba), d(bg)
        dc, dw, loss = torch.empty((1, 3), device=cuda), torch.empty(1, device=cuda), torch.zeros(1, device=cuda)
        if response:
            tab, cam = d(table), d(cams)
            grad, count = torch.empty((2, 6), device=cuda), torch.empty(2, dtype=torch.int32, device=cuda)
            err = torch.zeros(1, dtype=torch.int32, device=cuda)
            ws = torch.empty(int(lib.hrf_train_loss_response_workspace_bytes(2)), dtype=torch.uint8, device=cuda)
            L.check(lib.hrf_train_loss_response(c_.data_ptr(), w_.data_ptr(), r_.data_ptr(), b_.data_ptr(),
                                                cam.data_ptr(), 1, tab.data_ptr(), 2, 0.01, 0.0, None, dc.data_ptr(),
                                                dw.data_ptr(), loss.data_ptr(), grad.data_ptr(), count.data_ptr(),
                                                err.data_ptr(), ws.data_ptr(), L.stream()))
        else:
            L.check(lib.hrf_train_loss(c_.data_ptr(), w_.data_ptr(), r_.data_ptr(), b_.data_ptr(), 1, 0.01, 0.0, None,
                                       dc.data_ptr(), dw.data_ptr(), loss.data_ptr(), L.stream()))
        torch.cuda.synchronize()
        exp = np.array([h[0] * inv3], np.float32)
        assert loss.cpu().numpy().view(np.uint32)[0] == exp.view(np.uint32)[0], (i, float(loss), float(exp[0]))
    assert 0 < n_quad < 64
