"""The float64 references of the ray-form gradients (tests/ray_grad_oracle.py) on their own.  CPU only."""
import numpy as np
import torch

import ray_grad_oracle as RG
from oracle import field as ofield


def _dirs(rng, n):
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d[:8] = np.eye(3)[rng.integers(0, 3, 8)] * rng.choice([-1.0, 1.0], (8, 1))   # axis-aligned directions too
    return d.astype(np.float32)


def test_sh_jacobian_matches_autograd_of_oracle_sh4():
    rng = np.random.default_rng(0)
    d = _dirs(rng, 500)
    v = RG.sh_xyz(d)
    J, Jm = RG.sh4_jacobian(v)
    x = torch.from_numpy(v).requires_grad_(True)
    # oracle/field.sh4 maps its input through ((d + 1) * 0.5) * 2 - 1, the identity in float64 up to rounding
    sh = ofield.sh4(x)
    ref = np.stack([torch.autograd.grad(sh[:, j].sum(), x, retain_graph=True)[0].numpy() for j in range(16)], 1)
    assert np.abs(J - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    assert (np.abs(J) <= Jm + 1e-15).all()
    assert (J[:, 0] == 0).all()


def test_sh_jacobian_matches_central_differences():
    rng = np.random.default_rng(1)
    v = rng.uniform(-1, 1, (300, 3))
    J, _ = RG.sh4_jacobian(v)
    h = 1e-6
    for a in range(3):
        e = np.zeros(3)
        e[a] = h
        num = (ofield.sh4(torch.from_numpy(v + e)).numpy() - ofield.sh4(torch.from_numpy(v - e)).numpy()) / (2 * h)
        assert np.abs(J[:, :, a] - num).max() < 1e-7


def test_direction_grad_is_the_contraction():
    rng = np.random.default_rng(2)
    d = _dirs(rng, 64)
    dc = rng.standard_normal((64, 16))
    x = torch.from_numpy(RG.sh_xyz(d)).requires_grad_(True)
    (ref,) = torch.autograd.grad((ofield.sh4(x) * torch.from_numpy(dc)).sum(), x)
    np.testing.assert_allclose(RG.direction_grad(d, dc), ref.numpy(), rtol=1e-12, atol=1e-12)
    b = RG.direction_grad_bound(d, dc, np.zeros_like(dc))
    assert (b > 0).all() and (b < 1e-4 * (np.abs(dc).sum(1, keepdims=True) * 10)).all()


def test_ray_gradients_restatement():
    """Against a per-ray python loop; rays with 0 and 1 samples and a long one."""
    rng = np.random.default_rng(3)
    counts = np.array([0, 1, 5, 0, 300, 2, 1, 0])
    off = np.concatenate([[0], np.cumsum(counts)])
    n = off[-1]
    dp, dd = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
    t = rng.uniform(1, 3, n)
    rd = rng.standard_normal((len(counts), 3))
    d_o, d_d, d_t, S_o, S_d = RG.ray_gradients(dp, dd, t, rd, off)
    for r in range(len(counts)):
        s = slice(off[r], off[r + 1])
        np.testing.assert_allclose(d_o[r], dp[s].sum(0), atol=1e-12)
        np.testing.assert_allclose(d_d[r], (t[s, None] * dp[s] + dd[s]).sum(0), atol=1e-12)
        np.testing.assert_allclose(d_t[s], dp[s] @ rd[r], atol=1e-12)
        assert (S_o[r] >= np.abs(d_o[r])).all() and (S_d[r] >= np.abs(d_d[r])).all()
        if counts[r] == 0:
            assert (d_o[r] == 0).all() and (d_d[r] == 0).all()
    d_o2, d_d2, *_ = RG.ray_gradients(dp, None, t, rd, off)
    np.testing.assert_allclose(d_d2, d_d - np.stack([dd[off[r]:off[r + 1]].sum(0) for r in range(len(counts))]), atol=1e-12)


def test_refinement_rays_match_the_sampler_formula():
    """pixel_rays (torch, from the pose increment) against oracle/sampler.ray_directions on the synthetic cameras, at
    omega = 0 (the loader's own table, bit for bit) and at a small rotation (the table the refinement hands the
    sampler)."""
    from oracle import sampler as osamp

    from humanrf_b200.synthetic_scene import make_scene
    from humanrf_b200.toolbox.camera_refinement import pixel_rays, view_table

    sc = make_scene(num_images=4, width=96, height=72, portrait_every=0)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(4)
    for k in range(4):
        for omega in (np.zeros(3), np.array([0.01, -0.02, 0.005])):
            table = view_table(torch.from_numpy(sc["inverse_krs"][k]), torch.from_numpy(omega))
            if not omega.any():
                assert torch.equal(table, torch.from_numpy(sc["inverse_krs"][k]))
            pix = torch.from_numpy(np.concatenate([[0, W - 1, W * H - 1], rng.integers(0, W * H, 2000)]))
            o, d = pixel_rays(table, torch.from_numpy(sc["camera_origins"][k]), pix, W)
            ro, rd, _ = osamp.ray_directions(table.numpy()[None], sc["camera_origins"][k][None], np.array([True]),
                                             pix.numpy(), W, H)
            assert np.array_equal(o.numpy(), ro)
            # in units of 2^-24 (an ulp of the unit vector's length): v's components cancel, so a small component of d
            # carries the rounding of the large ones
            err = np.abs(d.numpy().astype(np.float64) - rd) / 2.0 ** -24
            assert err.max() <= 8, err.max()


def test_axisangle_round_trip():
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.toolbox.camera_refinement import axisangle_of

    for w in (np.array([0.1, -0.2, 0.3]), np.array([1e-9, 0, 0]), np.array([0, 3.0, 0.1]), np.zeros(3)):
        assert np.abs(axisangle_of(rotation_from_axisangle(w)) - w).max() < 1e-12
