"""The held-out response fit's float64 oracle (tests/response_fit_oracle.py) without a GPU: its closed-form solve against
numpy.linalg.lstsq on the augmented least-squares system, its closed-form residuals against a direct evaluation, four
wrong models the same check must reject, and ``held_out_fit_pairs``."""
import math

import numpy as np
import pytest

import response_fit_oracle as FO

LAM = 1e-6


def _view(P, seed, gain=(0.9, 1.1, 0.95), offset=(0.03, -0.02, 0.01), noise=2e-3):
    """A render (f, a) and an 8-bit image of g f + a b (+ noise) with a 60 % mask; background pixels are random."""
    rng = np.random.default_rng(seed)
    a = np.where(rng.uniform(0, 1, P) < 0.7, 1.0, rng.uniform(0, 1, P)).astype(np.float32)
    f = (rng.uniform(0.05, 0.85, (P, 3)) * a[:, None]).astype(np.float32)
    y = np.asarray(gain) * f + a[:, None] * np.asarray(offset) + rng.normal(0, noise, (P, 3))
    gt = np.rint(np.clip(y, 0, 1) * 255).astype(np.uint8)
    mask = (rng.uniform(0, 1, P) < 0.6).astype(np.uint8)
    gt[mask == 0] = rng.integers(0, 256, ((mask == 0).sum(), 3))     # outside the mask: unrelated colours
    return f, a, gt, mask


def _lstsq(f, a, gt, mask, lam):
    """Per channel, the least-squares solution of the augmented system [f a; sqrt(lam n) 0; 0 sqrt(lam n)] (g, b) =
    [y / 255; sqrt(lam n); 0] over the masked pixels."""
    m = mask != 0
    n = int(m.sum())
    r = math.sqrt(lam * n)
    out = np.zeros((3, 2))
    for k in range(3):
        A = np.concatenate((np.stack((f[m, k].astype(np.float64), a[m].astype(np.float64)), 1), [[r, 0.0], [0.0, r]]))
        rhs = np.concatenate((gt[m, k] / 255.0, [r, 0.0]))
        out[k] = np.linalg.lstsq(A, rhs, rcond=None)[0]
    return out


def _oracle_fit(f, a, gt, mask, lam=LAM):
    row, _, _ = FO.moments(f, a, gt, mask)
    gains, offs, report, status = FO.solve(row[None], [0], lam, 1)
    return np.stack((gains[0], offs[0]), 1), report[0], int(status[0])


def _agrees(gb, ref):
    return bool(np.all(np.abs(gb - ref) <= 1e-9 * np.maximum(np.abs(ref), 1e-3)))


@pytest.mark.parametrize("P,seed", [(500, 0), (20000, 1), (3001, 2)])
def test_oracle_solve_matches_lstsq(P, seed):
    f, a, gt, mask = _view(P, seed)
    for lam in (LAM, 1e-2):
        gb, _, st = _oracle_fit(f, a, gt, mask, lam)
        assert st == FO.OK
        assert _agrees(gb, _lstsq(f, a, gt, mask, lam)), (gb, _lstsq(f, a, gt, mask, lam))
    gb, _, _ = _oracle_fit(f, a, gt, mask)
    assert np.allclose(gb[:, 0], (0.9, 1.1, 0.95), atol=0.02) and np.allclose(gb[:, 1], (0.03, -0.02, 0.01), atol=0.01)


def test_oracle_residuals_match_direct_evaluation():
    f, a, gt, mask = _view(40000, 3)
    gb, report, _ = _oracle_fit(f, a, gt, mask)
    n = int(report[0])
    assert n == int(mask.sum())
    ident = FO.direct_sse(f, a, gt, mask, np.ones(3), np.zeros(3))
    fit = FO.direct_sse(f, a, gt, mask, gb[:, 0], gb[:, 1])
    # the expanded forms cancel: their error is a few ulps of the largest expanded term (S_ff, S_yy ~ n)
    assert np.allclose(report[1:4], ident, rtol=0, atol=1e-12 * n)
    assert np.allclose(report[4:7], fit, rtol=0, atol=1e-12 * n)
    assert (report[4:7] < report[1:4]).all()
    # the fit minimises the data term up to the ridge: no nearby (g, b) does better by more than the ridge's pull
    for d in ((1e-4, 0), (-1e-4, 0), (0, 1e-4), (0, -1e-4)):
        assert (FO.direct_sse(f, a, gt, mask, gb[:, 0] + d[0], gb[:, 1] + d[1]) >= fit - 2 * LAM * n).all()


def _wrong(f, a, gt, mask, which):
    """lstsq fits of four wrong models on the same data."""
    m = np.ones_like(mask) if which == "unmasked" else mask
    n = int((m != 0).sum())
    r = math.sqrt(LAM * n)
    out = np.zeros((3, 2))
    for k in range(3):
        sel = m != 0
        off_col = np.ones(sel.sum()) if which == "offset_unweighted" else a[sel].astype(np.float64)
        A = np.concatenate((np.stack((f[sel, k].astype(np.float64), off_col), 1), [[r, 0.0], [0.0, r]]))
        y = gt[sel, k].astype(np.float64) / (1.0 if which == "no_255" else 255.0)
        rhs = np.concatenate((y, [0.0 if which == "ridge_to_zero" else r, 0.0]))
        out[k] = np.linalg.lstsq(A, rhs, rcond=None)[0]
    return out


@pytest.mark.parametrize("which", ["unmasked", "offset_unweighted", "ridge_to_zero", "no_255"])
def test_wrong_models_are_rejected(which):
    # a ridge toward 0 moves the gain by about lambda n / S_ff (5e-6 here), far above the check's 1e-9
    f, a, gt, mask = _view(8000, 4)
    gb, _, _ = _oracle_fit(f, a, gt, mask)
    assert _agrees(gb, _lstsq(f, a, gt, mask, LAM))
    assert not _agrees(_wrong(f, a, gt, mask, which), gb), which


def test_held_out_fit_pairs_never_returns_a_scored_pair_and_spreads_evenly():
    from humanrf_b200.toolbox.camera_response import held_out_fit_pairs

    frames = list(range(15, 115))
    hero = [(126, f) for f in frames[::3]]
    landscape = [(v, f) for v, f in zip([0, 63, 97] * 40, frames[::5])]
    score = hero + landscape
    pairs = held_out_fit_pairs(score, frames, per_camera=8)
    assert not set(pairs) & set(score)
    cams = list(dict.fromkeys(c for c, _ in pairs))
    assert cams == [126, 0, 63, 97]
    for c in cams:
        got = [f for cc, f in pairs if cc == c]
        spare = [f for f in frames if (c, f) not in set(score)]
        want = [spare[i] for i in np.round(np.linspace(0, len(spare) - 1, 8)).astype(int)]
        assert got == want and len(got) == 8
        gaps = np.diff([spare.index(f) for f in got])
        assert gaps.max() - gaps.min() <= 1                   # evenly spread over the spare frames
        assert got[0] == spare[0] and got[-1] == spare[-1]


def test_held_out_fit_pairs_with_few_spare_frames():
    from humanrf_b200.toolbox.camera_response import held_out_fit_pairs

    frames = [15, 16, 17, 18, 19]
    score = [(3, 15), (3, 17), (3, 19), (5, 16)]
    pairs = held_out_fit_pairs(score, frames, per_camera=8)
    assert [f for c, f in pairs if c == 3] == [16, 18]             # fewer spare frames than asked: all of them
    assert [f for c, f in pairs if c == 5] == [15, 17, 18, 19]
    assert held_out_fit_pairs([(1, f) for f in frames], frames) == []   # scored on every frame: nothing to fit on
    assert held_out_fit_pairs(score, frames, per_camera=1) == [(3, 16), (5, 15)]
    with pytest.raises(ValueError):
        held_out_fit_pairs(score, frames, per_camera=0)
