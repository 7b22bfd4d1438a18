"""Float64 references for the ray-form gradients: the SH4 Jacobian (what hrf_field_backward_mlp_dirs contracts dCin
columns 0..15 with), hrf_ray_gradients restated in numpy, and the whole render() backward through OracleModel +
oracle/rendering.render under autograd.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np
import torch

import position_grad_oracle as P
from oracle import rendering as R

A, B, C, E, F, G, H, K, M = (0.48860251190291987, 1.0925484305920792, 0.94617469575755997, 0.54627421529603959,
                             0.59004358992664352, 2.8906114426405538, 0.45704579946446572, 0.3731763325901154,
                             1.4453057213202769)


def sh_xyz(d):
    """The fp32 x, y, z sh4 evaluates (field_common.cuh: ((d + 1) * 0.5) * 2 - 1 in fp32), as float64 [N,3]."""
    d = np.asarray(d, np.float32)
    return (((d + np.float32(1)) * np.float32(0.5)) * np.float32(2) - np.float32(1)).astype(np.float64)


def sh4_jacobian(v):
    """dSH_j / d(x, y, z) at v [N,3] float64: [N,16,3]; also the same with every monomial in absolute value (for the
    fp32 bound)."""
    v = np.asarray(v, np.float64)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    o = np.zeros_like(x)
    J = np.zeros((v.shape[0], 16, 3))
    Jm = np.zeros_like(J)
    rows = {
        1: ((o, -A + o, o), (o, A + o, o)),
        2: ((o, o, A + o), (o, o, A + o)),
        3: ((-A + o, o, o), (A + o, o, o)),
        4: ((B * y, B * x, o), (B * abs(y), B * abs(x), o)),
        5: ((o, -B * z, -B * y), (o, B * abs(z), B * abs(y))),
        6: ((o, o, 2 * C * z), (o, o, 2 * C * abs(z))),
        7: ((-B * z, o, -B * x), (B * abs(z), o, B * abs(x))),
        8: ((2 * E * x, -2 * E * y, o), (2 * E * abs(x), 2 * E * abs(y), o)),
        9: ((-6 * F * x * y, 3 * F * (y * y - x * x), o), (6 * F * abs(x * y), 3 * F * (y * y + x * x), o)),
        10: ((G * y * z, G * x * z, G * x * y), (G * abs(y * z), G * abs(x * z), G * abs(x * y))),
        11: ((o, H * (1 - 5 * z * z), -10 * H * y * z), (o, H * (1 + 5 * z * z), 10 * H * abs(y * z))),
        12: ((o, o, K * (15 * z * z - 3)), (o, o, K * (15 * z * z + 3))),
        13: ((H * (1 - 5 * z * z), o, -10 * H * x * z), (H * (1 + 5 * z * z), o, 10 * H * abs(x * z))),
        14: ((2 * M * x * z, -2 * M * y * z, M * (x * x - y * y)), (2 * M * abs(x * z), 2 * M * abs(y * z), M * (x * x + y * y))),
        15: ((3 * F * (y * y - x * x), 6 * F * x * y, o), (3 * F * (y * y + x * x), 6 * F * abs(x * y), o)),
    }
    for j, (val, mag) in rows.items():
        for a in range(3):
            J[:, j, a] = val[a]
            Jm[:, j, a] = mag[a]
    return J, Jm


def direction_grad(d, dcin16):
    """d_dir [N,3] = sum_j dcin16[:, j] dSH_j/d(x,y,z), float64, at the kernel's fp32 x, y, z."""
    J, _ = sh4_jacobian(sh_xyz(d))
    return np.einsum("nj,nja->na", np.asarray(dcin16, np.float64), J)


def direction_grad_bound(d, dcin16, dcin16_dev):
    """Entrywise bound on |kernel - direction_grad(d, dcin16)|: the dCin deviation bound propagated through |J|, plus
    the fp32 evaluation of J and of the 16-term contraction (at most 64 roundings of 2^-24 of sum |dcin_j| |J|_j)."""
    J, Jm = sh4_jacobian(sh_xyz(d))
    return (np.einsum("nj,nja->na", np.asarray(dcin16_dev, np.float64), np.abs(J))
            + 64 * 2.0 ** -24 * np.einsum("nj,nja->na", np.abs(np.asarray(dcin16, np.float64)), Jm))


def ray_gradients(d_pos, d_dir, t, ray_dirs, offsets):
    """hrf_ray_gradients in float64: (d_o [R,3], d_d [R,3], d_t [N], S_o, S_d) with S the sums of |terms| per entry."""
    d_pos, t, ray_dirs = (np.asarray(a, np.float64) for a in (d_pos, t, ray_dirs))
    d_dir = np.zeros_like(d_pos) if d_dir is None else np.asarray(d_dir, np.float64)
    off = np.asarray(offsets, np.int64)
    Rn = len(off) - 1
    ri = np.repeat(np.arange(Rn), np.diff(off))
    d_o, d_d, S_o, S_d = (np.zeros((Rn, 3)) for _ in range(4))
    np.add.at(d_o, ri, d_pos)
    np.add.at(S_o, ri, np.abs(d_pos))
    np.add.at(d_d, ri, t[:, None] * d_pos + d_dir)
    np.add.at(S_d, ri, np.abs(t[:, None] * d_pos) + np.abs(d_dir))
    d_t = (d_pos * ray_dirs[ri]).sum(1)
    return d_o, d_d, d_t, S_o, S_d


def _features_autograd(segs, f2s, f2t, u3, frames):
    """Composed features [N,32] float64 of normalised positions u3 [N,3] (float64, may require grad); 0 rows for
    samples whose frame has no segment."""
    fr = np.asarray(frames, np.int64)
    ok = (fr >= 0) & (fr < len(f2s))
    seg = np.where(ok, f2s[np.clip(fr, 0, len(f2s) - 1)], -1)
    tl = torch.from_numpy(np.where(ok, f2t[np.clip(fr, 0, len(f2t) - 1)], 0).astype(np.float32).astype(np.float64))
    u = torch.cat([u3, tl[:, None]], 1)
    out = torch.zeros((u.shape[0], 32), dtype=torch.float64)
    for s, sd in enumerate(segs):
        m = torch.from_numpy(np.nonzero(seg == s)[0])
        if len(m):
            out = out.index_put((m,), P._features_seg(sd, u[m], True))
    return out


def render_oracle(om, segs, f2s, f2t, o, d, t, ri, ray_frames, n_rays, bg, c_color, c_wsum, step=4e-4):
    """Gradients of loss = sum(color c_color) + sum(wsum c_wsum) with respect to (o, d, t, bg) through the float64
    features (autograd through the trilinear weights and vector lerps), the oracle MLPs with the kernels' bf16 rounding
    points (straight-through), SH4 of each sample's ray direction and oracle/rendering.render."""
    o_ = torch.from_numpy(np.asarray(o, np.float64)).requires_grad_(True)
    d_ = torch.from_numpy(np.asarray(d, np.float64)).requires_grad_(True)
    t_ = torch.from_numpy(np.asarray(t, np.float64)).requires_grad_(True)
    bg_ = torch.from_numpy(np.asarray(bg, np.float64)).requires_grad_(True)
    ri_ = torch.from_numpy(np.asarray(ri, np.int64))
    fr = np.asarray(ray_frames, np.int64)[np.asarray(ri, np.int64)]
    p = o_[ri_] + t_[:, None] * d_[ri_]
    feats = _features_autograd(segs, f2s, f2t, p + 0.5, fr)
    sigma, geo = om.sigma_head(om._q(feats.float()))
    rgb = om.color_head(d_[ri_].float(), geo)
    color, wsum = R.render(t_.float(), sigma, rgb, ri_, n_rays, background=None, step=step)
    color = color.double() + bg_ * (1.0 - wsum.double())
    loss = (color * torch.from_numpy(c_color)).sum() + (wsum.double() * torch.from_numpy(c_wsum)).sum()
    return [g.numpy() for g in torch.autograd.grad(loss, (o_, d_, t_, bg_))]
