"""Learned occupancy grid (include/humanrf_b200.h, hrf_bake_occupancy): the contract on the CPU oracle, small grids."""
import numpy as np
import pytest
import torch

from oracle import field as F
import bake_oracle as O

STEP, THRE = 4e-4, 1e-4


def _sphere(G, r=0.42):
    c = (np.arange(G) + 0.5) / G - 0.5
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    return ((x * x + y * y + z * z <= r * r) * 255).astype(np.uint8)


@pytest.fixture(scope="module")
def sharp_model():
    """table_std 6 and a density row scaled by 16: densities span many decades, so live and dead voxels both occur."""
    om = F.make_model((50,), seed=123, table_init="trained", bf16=True, table_std=6.0)
    om.w_sigma[1][0] *= 16.0
    return om


def _live(hull, max_sigma, step=STEP):
    return (hull != 0) & ((1 - np.exp(-max_sigma.astype(np.float32) * np.float32(step))) >= THRE)


@pytest.mark.parametrize("step", [STEP, 4e-6])
def test_bake_is_hull_subset_and_dead_voxels_have_no_live_neighbour(sharp_model, step):
    G = 16
    hull = _sphere(G)
    out, ms = O.bake_occupancy_grid(sharp_model, 15, hull, step, THRE)
    assert out.dtype == np.uint8 and set(np.unique(out)) <= {0, 255}
    assert not ((out != 0) & (hull == 0)).any()
    assert (ms[hull == 0] == 0).all() and (ms[hull != 0] > 0).all()
    live = _live(hull, ms, step)
    assert 0 < live.sum() <= (hull != 0).sum()
    assert ((out != 0) | ~live).all()             # every live voxel is kept
    p = np.pad(live, 1)
    for z, y, x in zip(*np.nonzero((hull != 0) & (out == 0))):
        assert not p[z:z + 3, y:y + 3, x:x + 3].any()
    if step != STEP:
        assert live.sum() < (hull != 0).sum() and (out == 0).sum() > (hull == 0).sum()


def test_bake_of_an_empty_hull_is_empty(sharp_model):
    out, ms = O.bake_occupancy_grid(sharp_model, 15, np.zeros((8, 8, 8), np.uint8), STEP, THRE)
    assert not out.any() and not ms.any()


def test_position_formula_numpy_equals_torch():
    """The float32 sub-sample positions of the oracle equal the torch expression the GPU test builds them with."""
    for G in (1, 7, 16, 24, 64, 256, 1000):
        idx = np.arange(G)
        x, y, z = idx, idx[::-1].copy(), (idx * 7) % G
        ref = O.bake_positions(x, y, z, G)
        s = torch.arange(8)
        cols = []
        for i, h in zip((x, y, z), (s & 1, (s >> 1) & 1, (s >> 2) & 1)):
            ti = torch.from_numpy(i).to(torch.float32)[:, None]
            cols.append((ti + 0.25 + 0.5 * h.to(torch.float32)[None, :]) / float(G) - 0.5)
        got = torch.stack(cols, -1).numpy()
        assert got.dtype == np.float32
        np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))
