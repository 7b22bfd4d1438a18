"""The colour-response oracle (tests/response_oracle.py) against float64 torch autograd of the pixel model
pred = g fg + w b + (1 - w) bg (fg = color - (1 - w) bg, g = e^gamma), through hrf_train_loss's Huber + BCE loss:
loss, d_color, d_wsum and the per-camera gradient of (gamma, b).  The same check must reject four wrong models:
d_color without g, d_wsum without the response term, the offset not weighted by w, and the gain applied to the
background.  Also the step and the data-parallel reduction of the oracle against torch.optim.Adam.  No GPU."""
import numpy as np
import pytest
import torch

import response_oracle as RO

DELTA, BCE_W = 0.01, 1e-3


def _batch(R, C_, seed):
    rng = np.random.default_rng(seed)
    color = rng.uniform(0, 1, (R, 3))
    w = np.where(rng.uniform(0, 1, R) < 0.8, rng.uniform(0.01, 0.99, R), rng.choice([0.0, 1.0], R))
    rgba = rng.uniform(0, 1, (R, 4))
    rgba[:, 3] = rng.choice([0.0, 1.0, 0.3], R)
    bg = rng.uniform(0, 1, (R, 3))
    near = rng.uniform(0, 1, R) < 0.5          # both Huber branches
    color[near] = rgba[near, :3] * rgba[near, 3:] + bg[near] * (1 - rgba[near, 3:]) + rng.normal(0, 3e-3, (near.sum(), 3))
    cams = rng.integers(0, C_, R)
    params = np.concatenate((rng.uniform(-0.2, 0.2, (C_, 3)), rng.uniform(-0.05, 0.05, (C_, 3))), 1)
    return color, w, rgba, bg, cams, params


def _autograd(color, w, rgba, bg, cams, params):
    """Loss and gradients of the pixel model by torch autograd in float64 (the table's em = expm1(gamma) and b, as
    float64 of the float32 table the kernel reads)."""
    table = RO.table_of(params).astype(np.float64)
    gamma = torch.tensor(np.log1p(table[:, :3]), requires_grad=True)
    off = torch.tensor(table[:, 3:], requires_grad=True)
    c = torch.tensor(color, requires_grad=True)
    wt = torch.tensor(w, requires_grad=True)
    bgt, rg = torch.tensor(bg), torch.tensor(rgba)
    idx = torch.tensor(cams)
    W = wt[:, None]
    fg = c - (1 - W) * bgt
    pred = torch.exp(gamma[idx]) * fg + W * off[idx] + (1 - W) * bgt
    m = rg[:, 3:]
    gt = rg[:, :3] * m + bgt * (1 - m)
    pc = torch.clamp(wt, 0, 1)
    bce = -(m[:, 0] * torch.log(pc + 1e-10) + (1 - m[:, 0]) * torch.log(1 - pc + 1e-10))
    loss = torch.nn.HuberLoss(delta=DELTA)(pred, gt) + BCE_W * bce.mean()
    loss.backward()
    return (float(loss.detach()), c.grad.numpy(), wt.grad.numpy(), torch.cat((gamma.grad, off.grad), 1).numpy(), table)


def _check(model, seed=0, R=3000, C_=7):
    color, w, rgba, bg, cams, params = _batch(R, C_, seed)
    loss, dc, dw, grad, table = _autograd(color, w, rgba, bg, cams, params)
    ref = RO.loss_and_grads(color, w, rgba, bg, cams, table.astype(np.float32), DELTA, BCE_W, model=model)
    close = lambda a, b: np.allclose(a, b, rtol=1e-9, atol=1e-15)   # noqa: E731
    return {"loss": abs(ref["loss"] - loss) <= 1e-12 * abs(loss), "d_color": close(ref["d_color"], dc),
            "d_wsum": close(ref["d_wsum"], dw), "grad": close(ref["grad"], grad)}


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_autograd(seed):
    assert _check(RO.pixel_model, seed) == {"loss": True, "d_color": True, "d_wsum": True, "grad": True}


def _dcolor_without_gain(color, w, bg, em, b):
    pred, g, dw, dgamma, db = RO.pixel_model(color, w, bg, em, b)
    return pred, np.ones_like(g), dw, dgamma, db


def _dwsum_without_response(color, w, bg, em, b):
    pred, g, dw, dgamma, db = RO.pixel_model(color, w, bg, em, b)
    return pred, g, np.zeros_like(dw), dgamma, db


def _offset_not_weighted(color, w, bg, em, b):
    W = w[:, None]
    fg = color - (1 - W) * bg
    pred = color + em * fg + b
    return pred, 1 + em, em * bg, (1 + em) * fg, np.ones_like(pred)


def _gain_on_background(color, w, bg, em, b):
    W = w[:, None]
    pred = (1 + em) * color + W * b
    return pred, 1 + em, b + 0 * bg, (1 + em) * color, np.broadcast_to(W, pred.shape)


@pytest.mark.parametrize("mutant, caught_by", [
    (_dcolor_without_gain, {"d_color"}),
    (_dwsum_without_response, {"d_wsum"}),
    (_offset_not_weighted, {"loss", "d_color", "d_wsum", "grad"}),
    (_gain_on_background, {"loss", "d_color", "d_wsum", "grad"}),
], ids=["dcolor_without_g", "dwsum_without_response", "offset_not_weighted", "gain_on_background"])
def test_mutants_are_rejected(mutant, caught_by):
    res = _check(mutant)
    failed = {k for k, ok in res.items() if not ok}
    assert failed, "the mutant passed"
    assert caught_by <= failed, (failed, caught_by)


def test_identity_is_exact_in_the_oracle():
    color, w, rgba, bg, cams, _ = _batch(500, 3, 5)
    ref = RO.loss_and_grads(color, w, rgba, bg, cams, np.zeros((3, 6), np.float32))
    assert np.array_equal(ref["pred"], color)
    assert np.array_equal(ref["d_wsum"], ref["dw_bce"] + 0.0)


def test_bad_camera_takes_identity_and_leaves_the_sums():
    color, w, rgba, bg, cams, params = _batch(400, 3, 6)
    cams[5], cams[9] = 3, -1
    table = RO.table_of(params)
    ref = RO.loss_and_grads(color, w, rgba, bg, cams, table)
    assert np.array_equal(ref["pred"][[5, 9]], color[[5, 9]]) and ref["count"].sum() == 398
    keep = np.ones(400, bool)
    keep[[5, 9]] = False
    sub = RO.loss_and_grads(color[keep], w[keep], rgba[keep], bg[keep], cams[keep], table)
    assert np.allclose(ref["grad"] * 400, sub["grad"] * 398, rtol=1e-12, atol=1e-18)


def test_adam_oracle_matches_torch():
    rng = np.random.default_rng(3)
    C_, lr = 4, 2e-3
    st = {"params": np.zeros((C_, 6)), "m": np.zeros((C_, 6)), "v": np.zeros((C_, 6)), "steps": np.zeros(C_, np.int64)}
    ref = [torch.zeros(6, dtype=torch.float64, requires_grad=True) for _ in range(C_)]
    opts = [torch.optim.Adam([p], lr=lr, betas=(0.9, 0.99), eps=1e-15) for p in ref]
    fixed = np.array([True, False, False, False])
    for _ in range(6):
        g = rng.standard_normal((C_, 6)) * 1e-3
        count = rng.integers(0, 2, C_)
        RO.adam(st, g, count, fixed, lr)
        for c in range(C_):
            if count[c] and not fixed[c]:
                ref[c].grad = torch.from_numpy(g[c])
                opts[c].step()
    for c in range(C_):
        assert np.allclose(st["params"][c], ref[c].detach().numpy(), rtol=1e-12, atol=1e-20)


def test_ranked_step_at_one_rank_is_the_single_rank_step():
    rng = np.random.default_rng(8)
    g = rng.standard_normal((5, 6)).astype(np.float32)
    n = np.array([0, 3, 1, 0, 2])
    fixed = np.zeros(5, bool)
    a = {"params": np.zeros((5, 6)), "m": np.zeros((5, 6)), "v": np.zeros((5, 6)), "steps": np.zeros(5, np.int64)}
    b = {k: v.copy() for k, v in a.items()}
    RO.ranked_step(a, [g], [n], [0], fixed, 1e-3)
    RO.adam(b, g.astype(np.float64), n, fixed, 1e-3)
    for k in a:
        assert np.array_equal(a[k], b[k])
    _, _, after = RO.ranked_step(a, [g, g], [n, n], [0, 1], fixed, 1e-3)
    assert after == [2, 1]
