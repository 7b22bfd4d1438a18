"""Float64 references for per-camera pose refinement in the train step (hrf_camera_pose_grad, hrf_camera_pose_step):
the SO(3) exponential and its left Jacobian, the per-camera sums with their fp32 accumulation bound, per-camera Adam,
and the sampler table of a rotated view.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np


def skew(w):
    w = np.asarray(w, np.float64)
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def _coeffs(th):
    """sin t / t, (1 - cos t) / t^2, (t - sin t) / t^3, by their series below t = 1e-2."""
    t2 = th * th
    if th < 1e-2:
        return (1 - t2 / 6 * (1 - t2 / 20 * (1 - t2 / 42)), 0.5 * (1 - t2 / 12 * (1 - t2 / 30 * (1 - t2 / 56))),
                (1 - t2 / 20 * (1 - t2 / 42 * (1 - t2 / 72))) / 6)
    return np.sin(th) / th, (1 - np.cos(th)) / t2, (th - np.sin(th)) / (t2 * th)


def so3_exp(w):
    K = skew(w)
    a, b, _ = _coeffs(float(np.linalg.norm(w)))
    return np.eye(3) + a * K + b * (K @ K)


def left_jacobian(w):
    """J_l(w) = I + (1 - cos t)/t^2 [w]x + (t - sin t)/t^3 [w]x^2; the identity at w = 0."""
    K = skew(w)
    _, b, c = _coeffs(float(np.linalg.norm(w)))
    return np.eye(3) + b * K + c * (K @ K)


def pose_grad(d_origins, d_ray_directions, ray_directions, cameras, omega):
    """(grad [C,6], count [C], bound [C,6]): grad = (J_l(omega_c)^T sum d x g_d, sum g_o) in float64 of the kernel's own
    fp32 inputs; bound = the fp32 error bound n 2^-23 sum|terms| per entry (cross products' own rounding included),
    carried through |J_l^T| for the rotation part, plus the final rounding."""
    g_o, g_d, d = (np.asarray(a, np.float64).reshape(-1, 3) for a in (d_origins, d_ray_directions, ray_directions))
    cam = np.asarray(cameras, np.int64).reshape(-1)
    omega = np.asarray(omega, np.float64).reshape(-1, 3)
    C = omega.shape[0]
    cross = np.cross(d, g_d)
    # |dy gz| + |dz gy| etc.: the magnitude the fp32 cross product and the sum see
    cabs = np.stack([np.abs(d[:, 1] * g_d[:, 2]) + np.abs(d[:, 2] * g_d[:, 1]),
                     np.abs(d[:, 2] * g_d[:, 0]) + np.abs(d[:, 0] * g_d[:, 2]),
                     np.abs(d[:, 0] * g_d[:, 1]) + np.abs(d[:, 1] * g_d[:, 0])], 1)
    S, A = np.zeros((C, 6)), np.zeros((C, 6))
    np.add.at(S, cam, np.concatenate([cross, g_o], 1))
    np.add.at(A, cam, np.concatenate([cabs, np.abs(g_o)], 1))
    n = np.bincount(cam, minlength=C)[:C]
    out, bound = S.copy(), np.zeros((C, 6))
    u = 2.0 ** -23
    for c in range(C):
        J = left_jacobian(omega[c])
        out[c, :3] = J.T @ S[c, :3]
        e = (n[c] + 2) * u * A[c]
        bound[c, :3] = np.abs(J).T @ e[:3] + 1e-15 * np.abs(J).T @ A[c, :3]
        bound[c, 3:] = e[3:]
    bound += 2.0 ** -24 * np.abs(out)
    return out, n.astype(np.int32), bound


def adam(state, grad, count, fixed, lr, betas=(0.9, 0.99), eps=1e-15):
    """torch.optim.Adam per camera on params [C,6] = (omega, tau): only cameras with count > 0 that are not fixed move,
    each with its own step counter.  state = dict(params, m, v, steps) of float64 / int arrays, updated in place."""
    b1, b2 = betas
    for c in range(len(count)):
        if count[c] == 0 or fixed[c]:
            continue
        state["steps"][c] += 1
        k = state["steps"][c]
        g = np.asarray(grad[c], np.float64)
        state["m"][c] = b1 * state["m"][c] + (1 - b1) * g
        state["v"][c] = b2 * state["v"][c] + (1 - b2) * g * g
        denom = np.sqrt(state["v"][c]) / np.sqrt(1 - b2 ** k) + eps
        state["params"][c] -= lr / (1 - b1 ** k) * state["m"][c] / denom
    return state


def view_table(inverse_kr, omega):
    """float64 (exp([omega]x) M)^T with M = inverse_kr^T: the sampler table before its one rounding."""
    M = np.asarray(inverse_kr, np.float32).astype(np.float64).reshape(3, 3).T
    return (so3_exp(omega) @ M).T
