"""The rounding-faithful MLP reference (tests/mlp_oracle.py) checked on its own, without a GPU.

Bars and where they come from:
* rounding off: the hand-written backward is the exact derivative of the float64 MLP, so it equals torch autograd of the
  same float64 function up to float64 summation order: 1e-12 relative to each tensor's largest entry.
* rounding on, against oracle.field.OracleModel(bf16=True) (fp32 accumulation in torch's order, bf16 at the same
  points): on samples the reference calls non-ambiguous the bf16 geometry features are identical and sigma / rgb are
  within the reference's own derived bounds (sigma_tol, rgb_tol: accumulation bound + exp bound); ambiguous samples
  within their propagated deviation bounds (D_geo, sigma_dev, rgb_dev).
* the classifier: every sample of the dyadic generator is exact; an accumulation whose terms span more than 24 bits is
  not; a value on a bf16 tie with a non-zero error bound is ambiguous.
"""
import numpy as np
import pytest
import torch

import mlp_oracle as M
from oracle import field as OF


def _float64_mlp(feat, dirs, cams, emb, P, scale, K):
    """Plain float64 torch forward of both MLPs (no rounding): the function the reference's rounding-off mode
    differentiates by hand."""
    T = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in P.items()}
    f = torch.tensor(feat, dtype=torch.float64, requires_grad=True)
    em = torch.tensor(np.asarray(emb, np.float64), requires_grad=True) if emb is not None else None
    hs = torch.relu(f @ T["W1s"].t())
    o = hs @ T["W2s"].t()
    sigma = torch.exp(o[:, 0]) * scale
    sh, _ = M.sh4(dirs)
    parts = [torch.tensor(sh), o[:, 1:16]]
    n = feat.shape[0]
    if em is not None:
        c = torch.tensor(cams)
        rows = torch.zeros((n, em.shape[1]), dtype=torch.float64)
        ok = c >= 0
        rows = rows.index_put((ok.nonzero()[:, 0],), em[c[ok]])
        parts.append(rows)
    width = sum(p.shape[1] for p in parts)
    parts.append(torch.ones((n, K - width), dtype=torch.float64))
    cin = torch.cat(parts, 1)
    h1 = torch.relu(cin @ T["W1c"].t())
    h2 = torch.relu(h1 @ T["W2c"].t())
    rgb = torch.sigmoid((h2 @ T["W3c"].t())[:, :3])
    return T, f, em, o, sigma, rgb


@pytest.mark.parametrize("K", [32, 48])
@pytest.mark.parametrize("upstream", ["sigma", "rgb", "geo", "all"])
def test_backward_equals_autograd_without_rounding(K, upstream):
    rng = np.random.default_rng(7 + K)
    n, E, C = 300, (2 if K == 48 else 0), 5
    P = {k: rng.uniform(-1, 1, s) * np.sqrt(6 / sum(s)) for k, s in
         dict(W1s=(64, 32), W2s=(16, 64), W1c=(64, K), W2c=(64, 64), W3c=(16, 64)).items()}
    feat = rng.standard_normal((n, 32)) * 0.5
    dirs = rng.standard_normal((n, 3))
    dirs = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True)).astype(np.float32)
    cams = rng.integers(-1, C, n) if E else None
    emb = rng.standard_normal((C, E)).astype(np.float32) if E else None
    d_sigma = rng.standard_normal(n) * 1e-2 if upstream in ("sigma", "all") else None
    d_rgb = rng.standard_normal((n, 3)) if upstream in ("rgb", "all") else None
    d_geo = rng.standard_normal((n, 15)).astype(np.float32) if upstream in ("geo", "all") else None

    F = M.Forward(feat, dirs, cams, emb, P, 100.0, K, rounding=False)
    B = M.Backward(F, d_sigma, d_rgb, d_geo, 100.0, num_cameras=C)
    T, f, em, o, sigma, rgb = _float64_mlp(feat, dirs, cams, emb, P, 100.0, K)
    np.testing.assert_allclose(F.sigma, sigma.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(F.rgb, rgb.detach().numpy(), rtol=1e-12)
    o.retain_grad()
    loss = torch.zeros((), dtype=torch.float64)
    if d_sigma is not None:
        loss = loss + (sigma * torch.tensor(d_sigma)).sum()
    if d_rgb is not None:
        loss = loss + (rgb * torch.tensor(d_rgb)).sum()
    if d_geo is not None:
        loss = loss + (o[:, 1:16] * torch.tensor(d_geo.astype(np.float64))).sum()
    loss.backward()

    def close(got, ref, what):
        ref = ref.detach().numpy() if torch.is_tensor(ref) else ref
        scale = max(np.abs(ref).max(), 1e-300)
        err = np.abs(got - ref).max() / scale
        assert err <= 1e-12, (what, err)

    ref_mlp = M.d_mlp_layout(*[(T[k].grad if T[k].grad is not None else torch.zeros_like(T[k])).detach().numpy()
                               for k in ("W1s", "W2s", "W1c", "W2c", "W3c")])
    close(B.d_mlp, ref_mlp, "d_mlp")
    close(B.dfeat, f.grad, "d features")
    close(B.gs_exact[:, 1:], o.grad[:, 1:16], "d geo")
    close(B.gs_exact[:, 0], o.grad[:, 0], "d h0")
    if E:
        close(B.d_emb, em.grad if em.grad is not None else np.zeros_like(B.d_emb), "d embedding")
    assert (B.d_mlp[-(16 * 64) + 3 * 64:] == 0).all()   # padded colour outputs 3..15


@pytest.mark.parametrize("cam_emb", [0, 2])
def test_forward_matches_bf16_oracle(cam_emb):
    """Rounding on: the reference's forward against OracleModel(bf16=True) sigma / colour heads."""
    K = 32 if cam_emb == 0 else 48
    om = OF.make_model((6,), seed=3, bf16=True, camera_embedding_dim=cam_emb)
    rng = np.random.default_rng(11)
    n = 2000
    feat = M.bf16(rng.standard_normal((n, 32)) * 0.7)
    dirs = rng.standard_normal((n, 3))
    dirs = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True)).astype(np.float32)
    cams = rng.integers(0, 160, n) if cam_emb else None
    sp = torch.cat([w.reshape(-1) for w in om.w_sigma]).numpy()
    cp = torch.cat([w.reshape(-1) for w in om.w_color]).numpy()
    P = M.split_params(sp, cp, K)
    emb = om.camera_embeddings.numpy() if cam_emb else None
    F = M.Forward(feat, dirs, cams, emb, P, om.density_scale, K)
    with torch.no_grad():
        sig, geo = om.sigma_head(torch.tensor(feat, dtype=torch.float32))
        rgb = om.color_head(torch.from_numpy(dirs), geo, torch.tensor(cams) if cam_emb else None)
    geo_bits = M.bf16(geo.double().numpy())
    amb = F.amb
    ex, tight, na = F.classes()
    print(f"K={K}: exact {ex} tight {tight} ambiguous {na}")
    assert (geo_bits[~F.amb_geo] == F.geo[~F.amb_geo, 1:]).all()
    assert (np.abs(geo_bits - F.geo[:, 1:]) <= F.D_geo[:, 1:]).all()
    ok, rep = M.compare_rows(sig.double().numpy(), F.sigma, F.sigma_tol, np.zeros(n, bool), F.amb_geo, F.sigma_dev)
    print("sigma", rep)
    assert ok
    ok, rep = M.compare_rows(rgb.double().numpy(), F.rgb, F.rgb_tol, np.zeros(n, bool), amb, F.rgb_dev)
    print("rgb", rep)
    assert ok


def test_dyadic_generator_is_exact():
    rng = np.random.default_rng(5)
    n, K = 2048, 32
    sp, cp = M.dyadic_params(rng, K)
    P = M.split_params(sp, cp, K)
    F = M.Forward(M.dyadic_features(rng, n), M.axis_directions(rng, n), None, None, P, 100.0, K)
    assert F.exact_geo.all() and F.exact.all(), F.classes()
    _, _, d_geo = M.dyadic_upstream(rng, n)
    B = M.Backward(F, None, None, d_geo, 100.0)
    assert B.exact.all(), B.classes()
    assert B.d_mlp_exact.all()


def test_classifier_rejects_broken_premise_and_ties():
    # terms 1 and 2^-30: not representable together in fp32
    X = np.array([[1.0, 2.0 ** -30]])
    W = np.array([[1.0, 1.0]])
    assert not M.Dense(X, W).exact.any()
    assert M.Dense(np.array([[1.0, 2.0 ** -20]]), W).exact.all()
    # a value on a bf16 tie (1 + 2^-8 lies halfway between 1 and 1 + 2^-7)
    v = np.array([1.0 + 2.0 ** -8, 1.0 + 2.0 ** -9])
    _, amb = M.round_amb(v, np.array([1e-9, 1e-9]))
    assert amb.tolist() == [True, False]
    assert M.bf16(np.array([1.0 + 2.0 ** -8]))[0] == 1.0 and M.bf16(np.array([1.0 + 3 * 2.0 ** -8]))[0] == 1.0 + 2.0 ** -6
    assert M.mask_amb(np.array([1e-9, 1e-3]), np.array([1e-8, 1e-8])).tolist() == [True, False]
    # the rounding agrees with torch's bf16 conversion (RN-even) on fp32 values
    x = np.random.default_rng(0).standard_normal(100000).astype(np.float32)
    assert (M.bf16(x.astype(np.float64)) == torch.from_numpy(x).bfloat16().double().numpy()).all()
    assert (M.valuation(np.array([3.0, 0.75, 2.0 ** -30, 0.0])) == np.array([0, -2, -30, M.BIG])).all()
