"""The error map's numpy oracle (tests/error_map_oracle.py) against independent restatements and statistical properties,
and the named mutants each of these checks must reject: the tile mapping against the sampler's own pixel coordinates,
border tiles' pixel counts, the draw's landing pixels, the CDF search, the EMA of unsampled tiles, the uniform share,
and the tile histogram of many draws against the target distribution (chi-square, p > 1e-4 for the oracle, < 1e-12 for
a mutant).  Also the hash, the 64-bit high product, the fixed-point sums and the refusals of ErrorMap."""
import math

import numpy as np
import pytest
from scipy import stats

import error_map_oracle as EO

MUTANTS = ("orientation", "npix", "lower_bound", "ema_unsampled", "uniform_ceil")


def _geo():
    # W, H not multiples of T; landscape and portrait slots
    return EO.Geometry([True, False, True, False], 37, 23, 8)


def _concentrated_ema(geo, rng):
    ema = rng.uniform(1e-4, 2e-3, geo.num_tiles).astype(np.float32)
    ema[rng.choice(geo.num_tiles, 6, replace=False)] = 0.05
    return ema


# ------------------------------------------------------------------------------------------------ checks
def check_tile_mapping(mutant=None) -> bool:
    """Every pool pixel's tile from the sampler's (x, y), and every tile's pixel count, equal the oracle's."""
    geo = _geo()
    idx = np.arange(geo.B * geo.P)
    slot, x, y = EO.sampler_pixel_xy(geo, idx)
    width = np.where(geo.landscape[slot], geo.W, geo.H)
    expect = slot * geo.nt + (y // geo.T) * (-(-width // geo.T)) + x // geo.T
    if not np.array_equal(geo.tile_of_pixel(idx, mutant), expect):
        return False
    return np.array_equal(np.bincount(expect, minlength=geo.num_tiles), geo.npix(mutant))


def check_draw_lands_in_tile(mutant=None) -> bool:
    geo = _geo()
    cdf = EO.cdf_of(geo, _concentrated_ema(geo, np.random.default_rng(1)), 1e-5, mutant)
    out, tiles = EO.draw(geo, cdf, 11, 3, 20000, 0.25, mutant)
    if out.min() < 0 or out.max() >= geo.B * geo.P:
        return False
    imp = tiles >= 0
    return np.array_equal(geo.tile_of_pixel(out[imp]), tiles[imp])


def check_cdf_search(mutant=None) -> bool:
    """Every integer target in [0, total) of a small CDF lands in the tile whose half-open interval holds it."""
    cdf = np.cumsum(np.array([3, 1, 4, 1, 5, 9, 2, 6], np.uint64), dtype=np.uint64)
    targets = np.arange(int(cdf[-1]), dtype=np.uint64)
    t = EO.pick_tile(cdf, targets, mutant)
    lo = np.concatenate(([0], cdf[:-1].astype(np.int64)))[np.minimum(t, len(cdf) - 1)]
    return bool((t < len(cdf)).all() and (lo <= targets.astype(np.int64)).all()
                and (targets.astype(np.int64) < cdf.astype(np.int64)[np.minimum(t, len(cdf) - 1)]).all())


def check_ema_keeps_unsampled(mutant=None) -> bool:
    geo = _geo()
    rng = np.random.default_rng(2)
    ema = rng.uniform(0, 1, geo.num_tiles).astype(np.float32)
    pixels = rng.integers(0, geo.B * geo.P, 40)
    sums, counts, _ = EO.accumulate(geo, pixels, rng.uniform(0, 0.02, 40).astype(np.float32))
    new, _ = EO.update(geo, ema, sums, counts, 0.5, 1e-5, mutant)
    cold = counts == 0
    return bool(cold.any() and np.array_equal(new[cold].view(np.uint32), ema[cold].view(np.uint32))
                and (new[~cold] != ema[~cold]).all())


def check_uniform_share(mutant=None) -> bool:
    """The leading rays that are the uniform draw are exactly floor(f R) (f R not an integer; the map is concentrated,
    so an importance ray all but never repeats the uniform pixel of its hash)."""
    geo = _geo()
    cdf = EO.cdf_of(geo, _concentrated_ema(geo, np.random.default_rng(3)), 1e-5)
    R, f = 1001, 0.3
    out, _ = EO.draw(geo, cdf, 5, 0, R, f, mutant)
    uniform = EO.umulhi(EO.hashes(5, 0, np.arange(R), 0), np.uint64(geo.B * geo.P)).astype(np.int64)
    lead = int(np.argmin(out == uniform)) if not (out == uniform).all() else R
    return lead == math.floor(f * R)


def check_histogram(mutant=None) -> bool:
    """Tiles of 2^20 rays drawn over 16 counters against the target probabilities: chi-square p > 1e-4."""
    geo = _geo()
    cdf_true = EO.cdf_of(geo, _concentrated_ema(geo, np.random.default_rng(4)), 1e-5)
    cdf = EO.cdf_of(geo, _concentrated_ema(geo, np.random.default_rng(4)), 1e-5, mutant)
    R, f = 65536, 0.25
    hist = np.zeros(geo.num_tiles)
    for c in range(16):
        out, _ = EO.draw(geo, cdf, 9, c, R, f, mutant)
        if out.min() < 0 or out.max() >= geo.B * geo.P:
            return False
        hist += np.bincount(geo.tile_of_pixel(out), minlength=geo.num_tiles)
    p = EO.target_probabilities(geo, cdf_true, f, R) * hist.sum()
    return stats.chisquare(hist, p).pvalue > 1e-4


CHECKS = (check_tile_mapping, check_draw_lands_in_tile, check_cdf_search, check_ema_keeps_unsampled,
          check_uniform_share, check_histogram)


@pytest.mark.parametrize("check", CHECKS, ids=lambda c: c.__name__)
def test_oracle_passes(check):
    assert check()


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_is_rejected(mutant):
    failed = [c.__name__ for c in CHECKS if not c(mutant)]
    assert failed, f"no check rejects the {mutant!r} mutant"


def test_histogram_rejects_a_wrong_distribution_strongly():
    """The chi-square check has the power it claims: the npix mutant's histogram is far outside (p < 1e-12)."""
    geo = _geo()
    cdf = EO.cdf_of(geo, np.ones(geo.num_tiles, np.float32), 1e-5, "npix")
    out, _ = EO.draw(geo, cdf, 9, 0, 1 << 20, 0.0, "npix")
    out = out[(out >= 0) & (out < geo.B * geo.P)]
    hist = np.bincount(geo.tile_of_pixel(out), minlength=geo.num_tiles)
    p = geo.npix() / (geo.B * geo.P) * hist.sum()
    assert stats.chisquare(hist, p).pvalue < 1e-12


def test_prior_draws_uniformly_by_pixel_count():
    """At a uniform EMA every tile weighs exactly EMA npix 2^24: the draw density per pixel is the same everywhere."""
    geo = _geo()
    w = EO.weights(geo, np.ones(geo.num_tiles, np.float32), 1e-5)
    assert np.array_equal(w, geo.npix().astype(np.uint64) << np.uint64(24))


# ------------------------------------------------------------------------------------------------ arithmetic
def test_splitmix64_known_values():
    # SplitMix64 seeded with 0: its first outputs are s(0), s(golden), ...
    assert int(EO.splitmix64(np.uint64(0))) == 0xE220A8397B1DCDAF
    assert int(EO.splitmix64(EO.GOLDEN)) == 0x6E789E6AA1B965F4


def test_umulhi_matches_python_integers():
    rng = np.random.default_rng(5)
    a = rng.integers(0, 2 ** 63, 2000, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, 2000, dtype=np.uint64)
    b = rng.integers(0, 2 ** 63, 2000, dtype=np.uint64)
    b[:4] = [0, 1, 2 ** 63, 2 ** 64 - 1]
    got = EO.umulhi(a, b)
    assert [int(x) for x in got] == [(int(x) * int(y)) >> 64 for x, y in zip(a, b)]


def test_fixed_point_sums_are_exact_and_capped():
    geo = _geo()
    rng = np.random.default_rng(6)
    e = rng.uniform(0, 0.03, 5000).astype(np.float32)
    e[:4] = [1.0, 2.0, np.nan, 0.0]
    q = EO.quantise(e)
    assert list(q[:4]) == [2 ** 32 - 1, 2 ** 32 - 1, 2 ** 32 - 1, 0]
    assert [int(x) for x in q[4:50]] == [min(round(float(x) * 2 ** 32), 2 ** 32 - 1) for x in e[4:50]]
    pixels = np.concatenate((rng.integers(0, geo.B * geo.P, 4999), [geo.B * geo.P]))
    sums, counts, err = EO.accumulate(geo, pixels, e)
    assert err == 1 and int(counts.sum()) == 4999
    t = geo.tile_of_pixel(pixels[:-1])
    for tile in np.unique(t)[:20]:
        assert int(sums[tile]) == sum(int(x) for x in q[:-1][t == tile])


def test_scan_is_exact_at_full_actorshq_scale_bound():
    """The reference's default pool at full ActorsHQ resolution fits the 2^63 bound with room to spare at T = 1."""
    for T in (1, 16, 32):
        geo = EO.Geometry([True] * 200, 4088, 3000, T)
        assert geo.max_total(1.0) < 2.0 ** 63
    assert EO.Geometry([True] * 200, 4088, 3000, 16).num_tiles == 200 * 256 * 188


def test_ray_error_is_the_loss_kernels_huber_sum():
    """Away from rounding ties, e_r is the Huber loss summed over the channels (float64 restatement)."""
    rng = np.random.default_rng(7)
    R = 4000
    color, rgba, bg = (rng.uniform(0, 1, (R, k)).astype(np.float32) for k in (3, 4, 3))
    rgba[:, 3] = rng.choice([0.0, 1.0, 0.5], R)
    e = EO.ray_error(color, None, rgba, bg, 0.01)
    gt = rgba[:, :3].astype(np.float64) * rgba[:, 3:] + bg * (1 - rgba[:, 3:].astype(np.float64))
    x = np.abs(color - gt)
    h = np.where(x < 0.01, 0.5 * x * x, 0.01 * (x - 0.005)).sum(1)
    assert np.allclose(e, h, rtol=1e-5, atol=1e-9)
    # through the response kernel's rounding of gt: the identity is the same value up to that rounding, and an
    # out-of-range camera takes the identity bit for bit
    table = np.zeros((3, 6), np.float32)
    table[1] = [0.1, -0.1, 0.05, 0.02, 0.0, -0.01]
    w = rng.uniform(0, 1, R).astype(np.float32)
    ident = EO.ray_error(color, w, rgba, bg, 0.01, table, np.zeros(R, np.int64))
    assert np.allclose(ident, h, rtol=1e-5, atol=1e-9)
    cams = rng.choice([-1, 0, 3, 7], R)
    assert np.array_equal(EO.ray_error(color, w, rgba, bg, 0.01, table, cams).view(np.uint32), ident.view(np.uint32))


def test_refusals_need_no_device():
    from humanrf_b200.dataset.data_loader import DataLoader
    from humanrf_b200.toolbox.error_map import ErrorMap

    class _Loader:
        mode = DataLoader.Mode.VALIDATION

    with pytest.raises(ValueError, match="TRAINING"):
        ErrorMap(_Loader())
    _Loader.mode = DataLoader.Mode.TRAINING
    for kw, msg in (({"tile": 0}, "tile"), ({"uniform_fraction": 1.5}, "uniform_fraction"),
                    ({"uniform_fraction": -0.1}, "uniform_fraction"), ({"beta": 0.0}, "beta"),
                    ({"floor": 0.0}, "floor"), ({"prior": float("nan")}, "prior")):
        with pytest.raises(ValueError, match=msg):
            ErrorMap(_Loader(), **kw)
