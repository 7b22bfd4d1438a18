"""The training occupancy oracle (tests/training_occupancy_oracle.py) against independent restatements: the dilation
against scipy, the compaction against np.flatnonzero, the points against float64, the bound update and the alpha test
on hand-made values.  Each named mutant of the oracle fails at least one of these checks."""
import numpy as np
import pytest
from scipy import ndimage

import training_occupancy_oracle as O

F32 = np.float32


def _hull(G, seed, density=0.4):
    rng = np.random.default_rng(seed)
    return np.where(rng.random((G, G, G)) < density, 255, 0).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ checks
def check_dilation(mutant=None):
    for G, seed in ((1, 0), (5, 1), (12, 2), (17, 3)):
        hull = _hull(G, seed, 0.6)
        lv = (np.random.default_rng(seed + 10).random((G, G, G)) < 0.05) & (hull != 0)
        ref = ndimage.binary_dilation(lv, structure=np.ones((3, 3, 3), bool)) & (hull != 0)
        assert np.array_equal(O.dilate(lv, hull, mutant), ref), (G, seed)


def check_compaction():
    for G, seed, d in ((1, 0, 1.0), (1, 0, 0.0), (7, 1, 0.3), (33, 2, 0.05), (16, 3, 1.0)):
        hull = _hull(G, seed, d)
        ids = O.compact(hull)
        assert ids.dtype == np.int32
        assert np.array_equal(ids, np.flatnonzero(hull.reshape(-1)).astype(np.int32))


def check_points(mutant=None):
    for G in (1, 33, 64, 256, 1024):
        rng = np.random.default_rng(G)
        ids = np.unique(rng.integers(0, G ** 3, 4000)).astype(np.int32)
        x, y, z = ids % G, (ids // G) % G, ids // (G * G)
        p = O.points(ids, G, seed=7, frame=21, counter=3, mutant=mutant)
        us = O.fractions(ids, O.key(7, 21, 3))
        for a, (i, u) in enumerate(zip((x, y, z), us)):
            # the fractions are exact 24-bit numbers in [0, 1)
            assert np.all(u >= 0) and np.all(u < 1) and np.array_equal(np.ldexp(np.floor(np.ldexp(u.astype(np.float64), 24)), -24), u)
            exact = (i + u.astype(np.float64)) / G - 0.5
            # float64 restatement of the three roundings: each is within half an ulp of its float32 result
            s = F32(i.astype(np.float64) + u)                  # fl(i + u)
            q = F32(s.astype(np.float64) / G)                  # fl(s / G)
            r = F32(q.astype(np.float64) - 0.5)                # fl(q - 0.5)
            assert np.array_equal(p[:, a], r), (G, a)
            bound = 4 * np.spacing(np.float32(1.0)) * np.maximum(np.abs(exact) + 0.5, 1.0 / G)
            assert np.all(np.abs(p[:, a].astype(np.float64) - exact) <= bound)
            # inside the voxel: p + 0.5 in [i / G, (i + 1) / G] (rounding may land on the upper face)
            q64 = p[:, a].astype(np.float64) + 0.5
            assert np.all(q64 >= i / G - 1e-7) and np.all(q64 <= (i + 1) / G + 1e-7)
    # a later refresh evaluates other points of the same voxel
    ids = np.arange(0, 64 ** 3, 97, dtype=np.int32)
    a = O.points(ids, 64, 7, 21, 0, mutant)
    b = O.points(ids, 64, 7, 21, 1, mutant)
    assert np.mean(np.all(a == b, axis=1)) < 0.01


def check_update(mutant=None):
    inf = np.inf
    bound = np.array([inf, inf, 1.0, 1.0, 1.0, 2.0, 3.0], F32)
    sigma = np.array([0.3, np.nan, 0.9, 0.2, inf, 0.1, np.nan], F32)
    exp = np.array([0.3, inf, 0.9, 0.5, inf, 1.0, inf], F32)
    got = O.update(bound, sigma, 0.5, mutant)
    assert np.array_equal(got, exp), got
    # decay 1 keeps the running maximum
    assert np.array_equal(O.update(np.array([2.0], F32), np.array([1.0], F32), 1.0, mutant), np.array([2.0], F32))


def _exact_threshold_bound(step, thre):
    """A float32 bound whose float32 alpha equals `thre` exactly."""
    b = F32(-np.log1p(-float(thre)) / float(step))
    for _ in range(20000):
        for c in (b, np.nextafter(b, F32(0))):
            alpha = F32(1.0) - np.exp((-c * F32(step)).astype(F32)).astype(F32)
            if alpha == F32(thre):
                return c
        b = np.nextafter(b, F32(np.inf)) if alpha < F32(thre) else np.nextafter(b, F32(0))
    raise AssertionError("no exact threshold bound")


def check_live(mutant=None):
    step, thre = F32(4e-4), F32(1678 * 2.0 ** -24)      # a threshold float32 alpha can equal exactly
    b = _exact_threshold_bound(step, thre)
    got = O.live(np.array([b, np.inf, 0.0, 1e6], F32), step, thre, mutant)
    assert got.tolist() == [True, True, False, True], got
    # the default threshold: a never-evaluated voxel is live, an empty one dead
    assert O.live(np.array([np.inf, 0.0], F32), mutant=mutant).tolist() == [True, False]


CHECKS = {"dilation": check_dilation, "points": check_points, "update": check_update, "live": check_live}


# ------------------------------------------------------------------------------------------------ tests
def test_dilation_matches_scipy():
    check_dilation()


def test_compaction_matches_flatnonzero():
    check_compaction()


def test_points_match_float64_restatement():
    check_points()


def test_bound_update():
    check_update()


def test_alpha_test():
    check_live()


def test_slot_bit_layout():
    rng = np.random.default_rng(4)
    for G in (1, 3, 4, 33):
        g = np.where(rng.random((G, G, G)) < 0.5, 255, 0).astype(np.uint8)
        w = O.pack_bits(g)
        assert w.shape == ((G ** 3 + 31) // 32,)
        bits = ((w[:, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1)
        assert np.array_equal(bits[:G ** 3] != 0, g.reshape(-1) != 0) and not bits[G ** 3:].any()


def test_grid_of_a_never_evaluated_frame_is_its_hull():
    hull = _hull(9, 5, 0.3)
    ids = O.compact(hull)
    g = O.grid(ids, np.full(ids.size, np.inf, F32), 9)
    assert np.array_equal(g != 0, hull != 0)


def test_splitmix64_known_values():
    assert int(O.splitmix64(np.uint64(0))) == 0xE220A8397B1DCDAF
    assert int(O.splitmix64(O.GOLDEN)) == 0x6E789E6AA1B965F4


@pytest.mark.parametrize("mutant,check", [("decay_after_max", "update"), ("six", "dilation"), ("leave_hull", "dilation"),
                                          ("no_counter", "points"), ("gt", "live"), ("inf_dead", "live")])
def test_named_mutants_fail(mutant, check):
    assert mutant in O.MUTANTS
    with pytest.raises(AssertionError):
        CHECKS[check](mutant)
