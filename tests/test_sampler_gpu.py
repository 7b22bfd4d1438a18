"""Bit-exact parity of the sm_90a sampler (csrc/sampler.cu) with oracle/sampler.py, which restates
ray_sampler.cu:11-194,196-325 in canonical IEEE float32 arithmetic, for all four entry points, a
CPU- and a GPU-resident image pool, landscape/portrait images, light-bloom filtering."""
import numpy as np
import pytest
import torch

from oracle import sampler as S
from scene import make_scene

pytestmark = pytest.mark.gpu
NAMES = ["origins", "directions", "rgba", "frame_numbers", "camera_numbers", "minmaxes", "ray_mask", "distances", "rel"]


def _run(cuda, sc, idx, occupancy, samples, bloom, pool_gpu, step=4e-4):
    from humanrf_b200.dataset import ray_sampler_native as rs
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    og = OccupanyGrid(sc["G"], len(sc["grids"]))
    handles = [og.add_grid(torch.from_numpy(g).to(cuda)) for g in sc["grids"]]
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rgba, lm = torch.from_numpy(sc["rgba"]), torch.from_numpy(sc["light_mask"])
    if pool_gpu:
        rgba, lm = rgba.to(cuda), lm.to(cuda)
    fn = getattr(rs, f"get_{'samples' if samples else 'rays'}_{'occupancy' if occupancy else 'aabb'}_minmax")
    out = fn(rgba, lm, t(sc["frame_numbers"]), t(sc["camera_numbers"]), torch.tensor(handles, dtype=torch.int64, device=cuda),
             t(sc["landscape"]), torch.from_numpy(idx).to(cuda), t(sc["inverse_krs"]), t(sc["camera_origins"]),
             t(sc["aabb"]), sc["G"], sc["width"], sc["height"], step, bloom)
    torch.cuda.synchronize()
    exp = S.get_data(sc["rgba"], sc["light_mask"], sc["frame_numbers"], sc["camera_numbers"], sc["grids"], sc["landscape"],
                     idx, sc["inverse_krs"], sc["camera_origins"], sc["aabb"], sc["G"], sc["width"], sc["height"],
                     step, bloom, occupancy=occupancy, samples=samples)
    del og
    return [o.cpu().numpy() for o in out], exp


@pytest.mark.parametrize("occupancy", [True, False])
@pytest.mark.parametrize("samples", [True, False])
def test_all_entry_points_bit_exact(cuda, occupancy, samples):
    sc = make_scene()
    rng = np.random.default_rng(5)
    idx = rng.integers(0, len(sc["grids"]) * sc["width"] * sc["height"], 3000).astype(np.int64)
    step = 4e-4 if occupancy else 2e-3
    for pool_gpu in (False, True):
        got, exp = _run(cuda, sc, idx, occupancy, samples, True, pool_gpu, step)
        for name, g, e in zip(NAMES, got, exp):
            assert g.shape == e.shape, (name, g.shape, e.shape)
            np.testing.assert_array_equal(g, e, err_msg=f"{name} pool_gpu={pool_gpu}")
        assert got[7].dtype == np.float32 and got[8].dtype == np.int32 and got[6].dtype == bool
    if samples:
        assert got[7].size > 0


def test_contiguous_pixel_range_and_empty(cuda):
    sc = make_scene(num_images=1, portrait_every=0)
    idx = np.arange(1000, 3048, dtype=np.int64)                     # validation/test style range (data_loader.py:578-580)
    got, exp = _run(cuda, sc, idx, True, True, False, True)
    for name, g, e in zip(NAMES, got, exp):
        np.testing.assert_array_equal(g, e, err_msg=name)
    got, exp = _run(cuda, sc, np.zeros(0, np.int64), True, True, False, True)
    assert got[0].shape == (0, 3) and got[7].shape == (0,)
    # rays that miss everything: a corner pixel range on a tight grid
    sc["grids"] = [np.zeros_like(sc["grids"][0])]
    got, exp = _run(cuda, sc, np.arange(0, 64, dtype=np.int64), True, True, False, True)
    assert got[0].shape[0] == 0 and not got[6].any() and got[7].size == 0


def test_wrong_resolution_raises(cuda):
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    og = OccupanyGrid(32, 2)
    with pytest.raises(RuntimeError, match="correct resolution"):
        og.add_grid(torch.zeros(16, 16, 16, dtype=torch.uint8, device=cuda))
    with pytest.raises(RuntimeError, match="expected device"):
        og.add_grid(torch.zeros(32, 32, 32, dtype=torch.uint8))
    h = [og.add_grid(torch.zeros(32, 32, 32, dtype=torch.uint8, device=cuda)) for _ in range(3)]
    assert h[0] == h[2] and h[0] != h[1]          # ring overwrite policy, occupancy_grid.cu:65-66
