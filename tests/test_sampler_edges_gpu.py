"""The sm_90a sampler (csrc/sampler.cu) on the edge cases of tests/sampler_cases.py: all four entry points bit for bit
against oracle/sampler.py with a CPU- and a GPU-resident pool and light-bloom filtering off and on; the contract on the
kernels' own outputs (offsets, sentinel, ordering); the occupancy lookup at every grid size; the ring's limits; and a
call whose sample total lies between 2^31 and 2^32."""
import ctypes as C

import numpy as np
import pytest
import torch

import sampler_cases as SC
from oracle import sampler as S

pytestmark = pytest.mark.gpu
NAMES = ["origins", "directions", "rgba", "frame_numbers", "camera_numbers", "minmaxes", "ray_mask", "distances", "rel"]
CONFIGS = {  # family -> [(G, grid patterns)], None: the family's own grids.  The oracle's march costs a full pass over
    # each image's grid per step, so G = 257 and 512 are left to the lookup test.
    "axis": [(33, SC.PATTERNS), (3, ("checker", "full"))],
    "origin": [(31, SC.PATTERNS), (1, ("full",)), (100, ("corners", "ellipsoid"))],
    "graze": [(2, ("full",)), (33, ("checker", "full"))],
    "miss": [(100, ("full",))],
    "ring": [(128, ("ellipsoid", "checker", "corners")), (33, ("shell", "full"))],
    "placed": [None],
    "counts": [None],
}
BOTH_OUTCOMES = ("axis", "origin", "graze", "ring")


class Sampler:
    """One scene on the device: its grids in a ring, its tables and pools."""

    def __init__(self, cuda, sc):
        from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

        self.sc, self.cuda = sc, cuda
        self.og = OccupanyGrid(sc["G"], len(sc["grids"]))
        self.handles = torch.tensor([self.og.add_grid(torch.from_numpy(g).to(cuda)) for g in sc["grids"]],
                                    dtype=torch.int64, device=cuda)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        self.dev = [t(sc[k]) for k in ("frame_numbers", "camera_numbers")] + [self.handles, t(sc["landscape"])]
        self.cam = [t(sc["inverse_krs"]), t(sc["camera_origins"]), t(sc["aabb"])]
        self.pool = {False: (torch.from_numpy(sc["rgba"]), torch.from_numpy(sc["light_mask"]))}
        self.pool[True] = tuple(x.to(cuda) for x in self.pool[False])

    def run(self, idx, occupancy, samples, bloom, pool_gpu, step):
        from humanrf_b200.dataset import ray_sampler_native as rs

        fn = getattr(rs, f"get_{'samples' if samples else 'rays'}_{'occupancy' if occupancy else 'aabb'}_minmax")
        rgba, lm = self.pool[pool_gpu]
        out = fn(rgba, lm, *self.dev, torch.from_numpy(idx).to(self.cuda), *self.cam, self.sc["G"], SC.W, SC.H, step,
                 bloom)
        return [o.cpu().numpy() for o in out]

    def offsets(self, idx, occupancy, step, bloom):
        """sample_offsets [n_kept + 1] and counters straight from hrf_sampler_rays (GPU pool)."""
        from humanrf_b200 import _lib as L

        rgba, lm = self.pool[True]
        R = idx.shape[0]
        p = L.SamplerParams()
        p.frame_numbers, p.camera_numbers = self.dev[0].data_ptr(), self.dev[1].data_ptr()
        p.grid_handles, p.landscape_modes = self.handles.data_ptr(), self.dev[3].data_ptr()
        p.inverse_krs, p.camera_origins, p.aabb = (x.data_ptr() for x in self.cam)
        p.light_mask = lm.view(torch.uint8).data_ptr() if bloom else None
        p.rgba_pool = rgba.data_ptr()
        p.grid_resolution, p.image_width, p.image_height = self.sc["G"], SC.W, SC.H
        p.step, p.occupancy, p.want_samples, p.filter_light_bloom = step, int(occupancy), 1, int(bloom)
        d = self.cuda
        ri = torch.from_numpy(idx).to(d)
        f = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=d)
        bufs = [f(R, dt=torch.bool), f(R, 3), f(R, 3), f(R, 4), f(R, dt=torch.int32), f(R, dt=torch.int32), f(R, 2),
                f(R, dt=torch.int64)]
        offs = torch.full((R + 1,), -7, dtype=torch.int32, device=d)
        counters = torch.zeros(2, dtype=torch.int64, device=d)
        ws_bytes = int(L.lib().hrf_sampler_workspace_bytes(R))
        ws = f(ws_bytes, dt=torch.uint8)
        L.check(L.lib().hrf_sampler_rays(C.byref(p), ri.data_ptr(), R, *(b.data_ptr() for b in bufs), offs.data_ptr(),
                                         counters.data_ptr(), ws.data_ptr(), ws_bytes, L.stream()))
        n, total = (int(v) for v in counters.cpu())
        return offs[:n + 1].cpu().numpy(), n, total


def oracle(sc, idx, occupancy, bloom, step):
    return S.get_data(sc["rgba"], sc["light_mask"], sc["frame_numbers"], sc["camera_numbers"], sc["grids"],
                      sc["landscape"], idx, sc["inverse_krs"], sc["camera_origins"], sc["aabb"], sc["G"], SC.W, SC.H,
                      step, bloom, occupancy=occupancy)


def _same(got, exp, what):
    for name, g, e in zip(NAMES, got, exp):
        assert g.shape == e.shape, (what, name, g.shape, e.shape)
        if g.dtype == np.float32:
            np.testing.assert_array_equal(g.view(np.int32), e.view(np.int32), err_msg=f"{what}: {name}")
        else:
            np.testing.assert_array_equal(g, e, err_msg=f"{what}: {name}")


def check_all(cuda, sc, idx, steps, what, tally=None, modes=((False, True), (True, True)), blooms=(False, True)):
    s = Sampler(cuda, sc)
    empty = [np.zeros(0, np.float32), np.zeros(0, np.int32)]
    for occupancy, want in modes:
        for bloom in blooms:
            for step in steps:
                exp = oracle(sc, idx, occupancy, bloom, step)
                if tally is not None:
                    tally[0] += int(exp[6].sum())
                    tally[1] += int((~exp[6]).sum())
                for pool_gpu in (False, True):
                    tag = f"{what} occ={occupancy} bloom={bloom} step={step:.3g} pool_gpu={pool_gpu}"
                    _same(s.run(idx, occupancy, False, bloom, pool_gpu, step), list(exp[:7]) + empty, tag + " rays")
                    if want:
                        _same(s.run(idx, occupancy, True, bloom, pool_gpu, step), exp, tag + " samples")
                if want:
                    check_contract(s, idx, occupancy, bloom, step, exp)
    return s


def check_contract(s, idx, occupancy, bloom, step, exp):
    """On the kernel's own outputs: offsets start at 0, never decrease, end in the sentinel = the sample total, and
    match rel; rel is sorted and in range; distances strictly increase within a ray and lie in [tmin, tmax)."""
    offs, n, total = s.offsets(idx, occupancy, step, bloom)
    mm, dist, rel = exp[5], exp[7], exp[8]
    assert n == mm.shape[0] and total == dist.size
    assert offs[0] == 0 and offs[n] == total and (np.diff(offs) >= 0).all()
    np.testing.assert_array_equal(offs, np.searchsorted(rel, np.arange(n + 1)))
    assert (np.diff(rel) >= 0).all() and (rel.size == 0 or (rel[0] >= 0 and rel[-1] < n))
    same = rel[1:] == rel[:-1]
    assert (dist[1:][same] > dist[:-1][same]).all()
    assert (dist >= mm[rel, 0]).all() and (dist < mm[rel, 1]).all()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_families_bit_exact(cuda, name):
    tally = [0, 0]
    for cfg in CONFIGS[name]:
        case = SC.family(name) if cfg is None else SC.family(name, cfg[0], cfg[1])
        if name == "counts":
            assert SC.count_check(case) == list(SC.COUNT_TARGETS)
        check_all(cuda, case.scene, case.idx, case.steps, f"{name} G={case.scene['G']}", tally)
    print(f"{name}: {tally[0]} rays kept, {tally[1]} rejected (over all grids, modes and bloom settings)")
    if name in BOTH_OUTCOMES:
        assert tally[0] > 0 and tally[1] > 0
    if name == "miss":
        assert tally[0] == 0


def test_batches_at_chunk_seams(cuda):
    for what, sc, idx, small in SC.batches():
        if small:
            check_all(cuda, sc, idx, (SC.STEP,), what)
        else:  # 2^20 + 3 rays: the rays entry points, and samples at a coarse step
            check_all(cuda, sc, idx, (0.1,), what, modes=((False, True), (True, False)), blooms=(True,))
        print(f"{what}: {idx.size} rays")
    sc = SC.batches()[0][1]
    masked = dict(sc, light_mask=np.ones_like(sc["light_mask"]))
    idx = np.arange(3 * 1024 + 7, dtype=np.int64) % sc["light_mask"].size
    s = check_all(cuda, masked, idx, (SC.STEP,), "every ray light-masked", blooms=(True,))
    assert s.run(idx, True, True, True, True, SC.STEP)[0].shape[0] == 0


def _lookup_points(G, grid, rng):
    """Voxel-centre planes of occupied voxels, 1/256 sub-steps and their fp32 neighbours (as the texture probe builds
    them), points on the faces of [0, 1]^3 and just past them, and points outside on both sides."""
    zz, yy, xx = np.nonzero(grid)
    if zz.size == 0:
        zz = yy = xx = np.zeros(1, np.int64)
    sel = rng.integers(0, zz.size, 60000)
    base = (np.stack([xx[sel], yy[sel], zz[sel]], 1) + 0.5) / G
    sub = rng.integers(-300, 301, base.shape) / (256.0 * G)
    jit = rng.integers(-3, 4, base.shape) * np.spacing(np.float32(base))
    near = (base + sub + jit).astype(np.float32)
    faces = np.array([0.0, 1.0], np.float32)
    edge = np.concatenate([faces, np.nextafter(faces, np.float32(-1)), np.nextafter(faces, np.float32(2))])
    onf = rng.uniform(0, 1, (30000, 3)).astype(np.float32)
    for k in range(3):
        onf[k * 10000:(k + 1) * 10000, k] = rng.choice(edge, 10000)
    out = rng.uniform(-0.3, 1.3, (30000, 3)).astype(np.float32)
    out[:15000, 0] = rng.uniform(-0.3, -1e-3, 15000)
    out[15000:, 2] = rng.uniform(1 + 1e-3, 1.3, 15000)
    return np.concatenate([near, onf, out])


@pytest.mark.parametrize("G", SC.GRID_SIZES)
def test_lookup_every_grid_size(cuda, G):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    rng = np.random.default_rng(G)
    pats = ("corners", "checker", "ellipsoid") if G >= 257 else SC.PATTERNS
    og = OccupanyGrid(G, len(pats))
    for p in pats:
        grid = SC.pattern(p, G)
        h = og.add_grid(torch.from_numpy(grid).to(cuda))
        pts = _lookup_points(G, grid, rng)
        got = og.lookup(h, torch.from_numpy(pts).to(cuda)).cpu().numpy()
        exp = S.tex_occupied(grid, pts)
        bad = np.nonzero(got != exp)[0]
        assert bad.size == 0, f"G={G} {p}: {bad.size} of {pts.shape[0]} differ, first p*G = {pts[bad[0]] * G}"


def test_ring_limits(cuda):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    with pytest.raises(RuntimeError, match="above 1024"):
        OccupanyGrid(1025, 1)
    G = 7
    og = OccupanyGrid(G, 3)
    rng = np.random.default_rng(4)
    grids = [((rng.random((G, G, G)) < 0.3) * 255).astype(np.uint8) for _ in range(7)]
    h = [og.add_grid(torch.from_numpy(g).to(cuda)) for g in grids]
    assert len(set(h[:3])) == 3 and h[3:] == h[:3] + h[:1]          # slots reused in order
    pts = _lookup_points(G, grids[6], rng)
    for slot, last in ((0, 6), (1, 4), (2, 5)):                     # each slot holds the grid written last
        got = og.lookup(h[slot], torch.from_numpy(pts).to(cuda)).cpu().numpy()
        np.testing.assert_array_equal(got, S.tex_occupied(grids[last], pts))


def test_sample_total_past_int32_is_refused(cuda):
    """About 10^6 candidates per ray in aabb mode and a total strictly between 2^31 and 2^32, computed from the
    oracle's count formula before any GPU call.  The rays pass writes per-ray values only, so the samples kernel never
    runs with wrapped offsets; the call must fail with a message naming the total and the cap."""
    case = SC.family("counts")
    sc = case.scene
    pix = np.unique(case.idx)
    step = 1e-6
    o, d, _ = S.ray_directions(sc["inverse_krs"], sc["camera_origins"], sc["landscape"], pix, SC.W, SC.H)
    tmin, tmax = S.aabb_minmax(o, d, sc["aabb"])
    assert (tmin < tmax).all()
    per = (np.float32(tmax - tmin) * (np.float32(1.0) / np.float32(step))).astype(np.float32).astype(np.int64)
    assert 8e5 < per.min() and per.max() < 1.2e6
    R = int(3.2e9 // per.mean())
    idx = np.resize(pix, R)
    total = int(np.resize(per, R).sum())
    assert 2 ** 31 < total < 2 ** 32, total
    s = Sampler(cuda, sc)
    with pytest.raises(RuntimeError, match=rf"{total} samples .*2147483647"):
        s.run(idx, False, True, False, True, step)
    got = s.run(idx, False, False, False, True, step)                 # the rays entry point is unaffected
    assert got[0].shape[0] == R
    check_all(cuda, sc, case.idx, (SC.STEP,), "after the refused call", modes=((False, True),), blooms=(False,))
