"""The float64 position-gradient reference (tests/position_grad_oracle.py) on its own: autograd through the float64
trilinear weights and vector lerps against central finite differences, and its composed features against
OracleModel.features."""
import numpy as np
import pytest
import torch

import position_grad_oracle as P
from oracle import field as ofield

H = 1e-9


def _model(segment_sizes=(50,), seed=7):
    """A HumanRF-shaped CPU stand-in: the oracle's tables rounded to bf16 (as the kernels read them)."""
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    frames = tuple(range(15, 15 + sum(segment_sizes)))
    om = ofield.make_model(segment_sizes, frames, seed=seed, table_std=2.0)
    m = HumanRF(sorted_frame_numbers=frames, segment_sizes=tuple(segment_sizes), **MODEL_KW)
    with torch.no_grad():
        for s, fg in enumerate(m.feature_grids):
            for k, g in enumerate(fg.grids()):
                r = om.segments[s].grids[k].to(torch.bfloat16).to(torch.float32)
                om.segments[s].grids[k] = r
                g.copy_(r.reshape(-1))
            fg.vectors.copy_(om.segments[s].vectors)
    return om, m, frames


def _points(rng, n, frames, segs, f2s, f2t, margin):
    """Random points in the unit cube further than `margin` (u units) from every cell face and vector-tap kink."""
    out_p, out_f = [], []
    while sum(len(p) for p in out_p) < n:
        p = rng.uniform(-0.499, 0.499, (4 * n, 3)).astype(np.float32)
        f = rng.choice(np.asarray(frames), 4 * n).astype(np.int32)
        ok = P.face_distance(p, f, f2s, f2t, segs) > margin
        out_p.append(p[ok])
        out_f.append(f[ok])
    return np.concatenate(out_p)[:n], np.concatenate(out_f)[:n]


@pytest.mark.parametrize("segment_sizes", [(50,), (100, 100, 50)])
def test_oracle_matches_central_differences(segment_sizes):
    om, m, frames = _model(segment_sizes)
    segs = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    rng = np.random.default_rng(3)
    n = 400
    pos, fr = _points(rng, n, frames, segs, f2s, f2t, 1e3 * H)
    dF = torch.from_numpy(rng.standard_normal((n, 32)))
    u32, _ = P._normalised(pos, fr, f2s, f2t)
    u = torch.from_numpy(u32.astype(np.float64))
    g = P.position_grad(segs, f2s, f2t, pos, fr, dF, exact32=False, u_override=u)

    def phi(uu):
        out = torch.zeros(n, dtype=torch.float64)
        seg = f2s[fr]
        for s, sd in enumerate(segs):
            sel = torch.from_numpy(np.nonzero(seg == s)[0])
            if len(sel):
                out[sel] = (P._features_seg(sd, uu[sel], False) * dF[sel]).sum(1)
        return out

    fd = torch.zeros((n, 3), dtype=torch.float64)
    for d in range(3):
        up, dn = u.clone(), u.clone()
        up[:, d] += H
        dn[:, d] -= H
        fd[:, d] = (phi(up) - phi(dn)) / (2 * H)
    # inside a cell the features are linear along each axis: the difference quotient is exact up to float64 rounding of
    # phi, about 2^-52 * sum|terms| / H
    S = P.bound_terms(segs, f2s, f2t, pos, fr, dF)
    err = (g - fd).abs()
    scale = S.sum(1, keepdim=True) * 2.0 ** -52 * 64 / H + S * 1e-9
    print(f"max |autograd - fd| {err.max():.3e}, max |g| {g.abs().max():.3e}")
    assert (err <= scale).all()
    assert g.abs().max() > 1.0


def test_oracle_features_match_oracle_model():
    om, m, frames = _model((100, 100, 50), seed=11)
    segs = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    rng = np.random.default_rng(5)
    n = 3000
    pos = rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)
    pos[:8] = np.array([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5], [0.5, -0.5, 0.25], [0, 0, 0],
                        [0.4999, -0.4999, 0.1], [0.25, 0.25, 0.25], [-0.125, 0.375, 0.5], [0.5, 0.5, -0.5]], np.float32)
    fr = rng.choice(np.asarray(frames), n).astype(np.int32)
    fr[-5:] = [frames[0] - 1, 0, 114, 115, 214]
    ours = P.features(segs, f2s, f2t, pos, fr, exact32=True)
    with torch.no_grad():
        ref = om.features(torch.from_numpy(pos), torch.from_numpy(fr)).double()
    # float32 precision of the oracle model: its blends and compositions run in fp32
    err = (ours - ref).abs()
    tol = 1e-5 * (ours.abs() + ref.abs()) + 1e-6
    print(f"max |float64 - OracleModel| {err.max():.3e}")
    assert (err <= tol).all()
    assert ours.abs().max() > 0.1
    # frames the table maps to no segment compose to 0
    assert (ours[-5:-3] == 0).all() and (ours[-3:] != 0).any(1).all()


def test_exact32_mode_differs_only_by_float32_offsets():
    """The kernel-faithful mode moves each fractional offset by at most one float32 rounding of pos."""
    _, m, frames = _model((50,))
    segs = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    rng = np.random.default_rng(9)
    n = 500
    pos, fr = _points(rng, n, frames, segs, f2s, f2t, 1e-4)
    dF = torch.from_numpy(rng.standard_normal((n, 32)))
    a = P.position_grad(segs, f2s, f2t, pos, fr, dF, exact32=True)
    b = P.position_grad(segs, f2s, f2t, pos, fr, dF, exact32=False)
    S = P.bound_terms(segs, f2s, f2t, pos, fr, dF)
    # frac moves by <= ulp(2048) = 2^-12 at the finest level: a relative change of the terms of at most 2^-12 / 1e-4 * 2
    assert ((a - b).abs() <= S * 2.0 ** -12 / 1e-4 * 4).all()
    assert (a - b).abs().max() > 0     # the two modes are not the same function
