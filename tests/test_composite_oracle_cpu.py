"""The float64 compositing reference of tests/composite_oracle.py on the CPU: its analytic backward against torch
autograd, its forward against oracle/rendering.py, the +inf convention, and that each deliberately wrong fp32
restatement of the kernels lands outside the error bound on the GPU test's inputs while the faithful one stays inside."""
import numpy as np
import pytest
import torch

import composite_oracle as O
from oracle import rendering as R


def _small(seed=3, with_inf=False):
    rng = np.random.default_rng(seed)
    counts = np.array([0, 1, 5, 40, 33, 0, 70, 2])
    R_ = counts.shape[0]
    off = np.concatenate(([0], np.cumsum(counts)))
    n = int(off[-1])
    sigma = (rng.random(n) ** 2 * 2000).astype(np.float32)
    if with_inf:
        sigma[off[3] + 7] = np.inf
    t = (rng.uniform(0.5, 7.5, n)).astype(np.float32)
    return dict(sigma=sigma, rgb=rng.random((n, 3)).astype(np.float32), t=t, off=off, num_rays=R_,
                ri=O.ray_of(off), bg=rng.random((R_, 3)).astype(np.float32),
                dcolor=rng.standard_normal((R_, 3)).astype(np.float32), dwsum=rng.standard_normal(R_).astype(np.float32))


@pytest.mark.parametrize("with_bg", [False, True])
def test_backward_matches_autograd(with_bg):
    B = _small()
    bg = B["bg"] if with_bg else None
    F = O.Forward(B["sigma"], B["rgb"], B["t"], B["off"], O.STEP, bg)
    G = O.Backward(F, B["rgb"], bg, B["dcolor"], B["dwsum"])
    s = torch.tensor(B["sigma"], dtype=torch.float64, requires_grad=True)
    c = torch.tensor(B["rgb"], dtype=torch.float64, requires_grad=True)
    dt = torch.tensor(O.dt32(B["t"], O.STEP), dtype=torch.float64)
    sdt = s * dt
    ri = torch.tensor(B["ri"])
    T = torch.exp(-R._exclusive_by_ray(sdt, ri, "sum"))
    w = T * (1 - torch.exp(-sdt))
    col = R.accumulate(w, ri, c, B["num_rays"])
    ws = R.accumulate(w, ri, None, B["num_rays"])
    if with_bg:
        col = col + torch.tensor(bg, dtype=torch.float64) * (1 - ws)
    loss = (col * torch.tensor(B["dcolor"], dtype=torch.float64)).sum() + (ws[:, 0] * torch.tensor(B["dwsum"], dtype=torch.float64)).sum()
    loss.backward()
    np.testing.assert_allclose(G.d_sigma, s.grad.numpy(), rtol=1e-9, atol=1e-12 * np.abs(s.grad.numpy()).max())
    np.testing.assert_allclose(G.d_rgb, c.grad.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(F.color, col.detach().numpy(), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("with_bg", [False, True])
def test_forward_matches_oracle_rendering(with_bg):
    B = O.ray_batch(num_rays=300, max_random=300, seed=4)
    fin = np.isfinite(B["sigma"])
    B["sigma"][~fin] = 1e4               # oracle/rendering's cumsum-difference form cannot take +inf
    bg = B["bg"] if with_bg else None
    F = O.Forward(B["sigma"], B["rgb"], B["t"], B["off"], O.STEP, bg)
    ri = torch.tensor(B["ri"])
    col, ws = R.render(torch.tensor(B["t"]),   # fp32 t: the oracle forms dt in fp32 as the kernels do
                        torch.tensor(B["sigma"]).double(), torch.tensor(B["rgb"]).double(),
                       ri, B["num_rays"], None if bg is None else torch.tensor(bg).double(), step=float(np.float32(O.STEP)))
    np.testing.assert_allclose(F.color, col.numpy(), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(F.wsum, ws.numpy()[:, 0], rtol=1e-9, atol=1e-12)
    # the kernels' dt differs from step once t is large: (t + step) - t rounds in fp32
    assert (O.dt32(B["t"], O.STEP) != np.float32(O.STEP)).mean() > 0.5


def test_inf_density_is_an_opaque_sample():
    """nerfacc's running sum renders sigma = +inf as opaque: weight T there, 0 behind it, nothing NaN; the gradient of
    the opaque sample and of every sample behind it is 0."""
    B = _small(with_inf=True)
    k = B["off"][3] + 7
    b, e = B["off"][3], B["off"][4]
    F = O.Forward(B["sigma"], B["rgb"], B["t"], B["off"], O.STEP, B["bg"])
    G = O.Backward(F, B["rgb"], B["bg"], B["dcolor"], B["dwsum"])
    for name in ("weights", "color", "wsum", "depth"):
        assert np.isfinite(getattr(F, name)).all(), name
        assert np.isfinite(getattr(F, name + "_err")).all(), name
    assert F.weights[k] == F.T[k] > 0 and (F.weights[k + 1:e] == 0).all() and F.T[k + 1] == 0
    np.testing.assert_allclose(F.wsum[3], 1.0, rtol=1e-15)
    assert np.isfinite(G.d_sigma).all() and (G.d_sigma[k:e] == 0).all()
    assert (G.d_sigma[b:k] != 0).all() and (G.d_rgb[k + 1:e] == 0).all()
    # the dead samples' allowance is the suffix cancellation noise alone: (2 chunks + 14) u sum |g w| times dt
    sgw = np.abs(G.g[b:e] * F.w[b:e]).sum()
    np.testing.assert_allclose(G.d_sigma_err[k + 1:e], F.dt[k + 1:e] * (2 * 2 + 14) * O.U * sgw, rtol=1e-6)
    # the fp32 restatements do not NaN either
    w32, c32, ws32 = O.kernel_forward32(B["sigma"], B["rgb"], B["t"], B["off"], O.STEP, B["bg"])
    assert np.isfinite(c32).all() and w32[k] > 0 and (w32[k + 1:e] == 0).all()


def test_thresholds_hit_exactly_are_not_ambiguous():
    """sigma = 0 gives alpha = 0 and T = 1 exactly: with eps = 1 and thre = 0 the reference must decide, not shrug."""
    off = np.array([0, 4, 9])
    sigma = np.array([0, 0, 3, 0, 0, 0, 0, 0, 1e3], np.float32)
    keep, amb, _ = O.visibility(sigma, off, O.STEP, eps=1.0, thre=0.0)
    assert not amb[[0, 1, 2, 4, 5, 6, 7, 8]].any()
    np.testing.assert_array_equal(keep, [1, 1, 1, 0, 1, 1, 1, 1, 1])


FAITHFUL = {}


def _gpu_inputs():
    if "B" not in FAITHFUL:
        FAITHFUL["B"] = O.ray_batch()
    return FAITHFUL["B"]


def _ratio(B, mutant):
    """error / bound of the fp32 restatement (mutant = None: the faithful one) on the GPU test's batch."""
    a = (B["sigma"], B["rgb"], B["t"], B["off"], O.STEP)
    if mutant == "scan_without_block_carry":
        keep, _, _ = O.visibility(B["sigma"], B["off"], O.STEP)
        ref = O.kept_offsets(keep, B["off"])
        got = O.scan32(np.diff(ref), mutant)
        return float(np.sum(got != ref)) * np.inf if (got != ref).any() else 0.0
    if mutant == "d_sigma_without_dt" or mutant == "backward":
        F = O.Forward(*a, B["bg"])
        G = O.Backward(F, B["rgb"], B["bg"], B["dcolor"], B["dwsum"])
        ds, drgb = O.kernel_backward32(*a, B["bg"], B["dcolor"], B["dwsum"], None if mutant == "backward" else mutant)
        return max(O.ratio(ds, G.d_sigma, G.d_sigma_err), O.ratio(drgb, G.d_rgb, G.d_rgb_err))
    if mutant in ("fixup_without_T", "fused"):
        F = O.Forward(*a, B["bg"], kernel="fused")
        c, ws, dep = O.fused_forward32(*a, B["bg"], None if mutant == "fused" else mutant)
        return max(O.ratio(c, F.color, F.color_err), O.ratio(ws, F.wsum, F.wsum_err), O.ratio(dep, F.depth, F.depth_err))
    F = O.Forward(*a, B["bg"])
    w, c, ws = O.kernel_forward32(*a, B["bg"], mutant)
    return max(O.ratio(w, F.weights, F.weights_err), O.ratio(c, F.color, F.color_err), O.ratio(ws, F.wsum, F.wsum_err))


@pytest.mark.parametrize("which", [None, "backward", "fused"])
def test_faithful_restatements_stay_inside_the_bound(which):
    B = _gpu_inputs()
    r = _ratio(B, which)
    keep, _, _ = O.visibility(B["sigma"], B["off"], O.STEP)
    assert (O.scan32(np.diff(O.kept_offsets(keep, B["off"]))) == O.kept_offsets(keep, B["off"])).all()
    print(f"faithful {which or 'forward'}: largest error / bound {r:.3g}")
    assert r <= 1.0


@pytest.mark.parametrize("mutant", O.MUTANTS)
def test_every_mutant_lands_outside_the_bound(mutant):
    B = _gpu_inputs()
    r = _ratio(B, mutant)
    print(f"mutant {mutant}: largest error / bound {r:.3g}")
    assert r > 1.0
