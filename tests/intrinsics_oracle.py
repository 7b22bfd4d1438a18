"""Float64 references for per-camera intrinsics refinement in the train step (hrf_camera_calib_grad,
hrf_camera_calib_step): the intrinsics gradient from the rays' directions, g_d and the cameras' rotations with its fp32
bound, B = K0 A K0^-1 and the refined sampler table, per-camera Adam over two learning rates, and the RMS reprojection
error the recovery tests score cameras with.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np

import pose_oracle as PO


def intrinsics_grad(d_ray_directions, ray_directions, cameras, alpha, rotations):
    """(grad [C,4], count [C], bound [C,4]): d(loss)/d(alpha_x, alpha_y, beta_x, beta_y) in float64 of the kernel's own
    fp32 inputs.  q = R'^T d, h = R'^T (g_d - d (d . g_d)); grad = (-sum q_x h_x, -sum q_y h_y, -e^-ax sum q_z h_x,
    -e^-ay sum q_z h_y).  bound = (n + 12) 2^-23 sum|terms| per entry, |terms| from the magnitudes each fp32 product and
    sum of a ray's term sees (12 covers the roundings of one ray's term: d.g_d, the projection, two mat-vecs, the
    product), times e^-alpha for beta, plus the final rounding."""
    g_d, d = (np.asarray(a, np.float64).reshape(-1, 3) for a in (d_ray_directions, ray_directions))
    cam = np.asarray(cameras, np.int64).reshape(-1)
    alpha = np.asarray(alpha, np.float64).reshape(-1, 2)
    Rp = np.asarray(rotations, np.float64).reshape(-1, 3, 3)
    C = alpha.shape[0]
    Rc = Rp[cam]                                                   # [R,3,3]
    q = np.einsum("rij,ri->rj", Rc, d)                             # R'^T d
    dg = (d * g_d).sum(1, keepdims=True)
    p = g_d - d * dg
    h = np.einsum("rij,ri->rj", Rc, p)
    terms = np.stack([q[:, 0] * h[:, 0], q[:, 1] * h[:, 1], q[:, 2] * h[:, 0], q[:, 2] * h[:, 1]], 1)
    aR = np.abs(Rc)
    qa = np.einsum("rij,ri->rj", aR, np.abs(d))
    pa = np.abs(g_d) + np.abs(d) * (np.abs(d) * np.abs(g_d)).sum(1, keepdims=True)
    ha = np.einsum("rij,ri->rj", aR, pa)
    tabs = np.stack([qa[:, 0] * ha[:, 0], qa[:, 1] * ha[:, 1], qa[:, 2] * ha[:, 0], qa[:, 2] * ha[:, 1]], 1)
    S, A = np.zeros((C, 4)), np.zeros((C, 4))
    np.add.at(S, cam, terms)
    np.add.at(A, cam, tabs)
    n = np.bincount(cam, minlength=C)[:C]
    scale = np.concatenate([np.ones((C, 2)), np.exp(-alpha)], 1)
    out = -scale * S
    bound = (n[:, None] + 12) * 2.0 ** -23 * scale * A + 2.0 ** -24 * np.abs(out)
    return out, n.astype(np.int32), bound


def intrinsics_matrix(alpha, beta, K):
    """B = K0 A K0^-1 for K = (fx0, fy0, cx0, cy0)."""
    ax, ay = alpha
    bx, by = beta
    fx, fy, cx, cy = K
    return np.array([[np.exp(-ax), 0.0, -cx * np.expm1(-ax) - fx * bx * np.exp(-ax)],
                     [0.0, np.exp(-ay), -cy * np.expm1(-ay) - fy * by * np.exp(-ay)],
                     [0.0, 0.0, 1.0]])


def calibration_table(inverse_kr, omega, alpha, beta, K):
    """float64 (exp([omega]x) (M0 B))^T with M0 = inverse_kr^T: the sampler table before its one rounding."""
    M0 = np.asarray(inverse_kr, np.float32).astype(np.float64).reshape(3, 3).T
    return (PO.so3_exp(omega) @ (M0 @ intrinsics_matrix(alpha, beta, K))).T


def adam(state, grad, count, fixed, lr, lr_intrinsics, betas=(0.9, 0.99), eps=1e-15):
    """torch.optim.Adam per camera on params [C,10] = (omega, tau, alpha, beta), the first six at lr and the last four
    at lr_intrinsics, one step counter per camera; only cameras with count > 0 that are not fixed move."""
    b1, b2 = betas
    lrs = np.array([lr] * 6 + [lr_intrinsics] * 4)
    for c in range(len(count)):
        if count[c] == 0 or fixed[c]:
            continue
        state["steps"][c] += 1
        k = state["steps"][c]
        g = np.asarray(grad[c], np.float64)
        state["m"][c] = b1 * state["m"][c] + (1 - b1) * g
        state["v"][c] = b2 * state["v"][c] + (1 - b2) * g * g
        denom = np.sqrt(state["v"][c]) / np.sqrt(1 - b2 ** k) + eps
        state["params"][c] -= lrs / (1 - b1 ** k) * state["m"][c] / denom
    return state


def project(points, cam):
    """Pixel coordinates [N,2] of world points in a dataset camera (rotation_axisangle, translation, focal_length,
    principal_point normalised by the image size), float64."""
    from humanrf_b200.dataset.cameras import projection_matrix_world2pixel

    P = projection_matrix_world2pixel(cam.width, cam.height, cam.rotation_axisangle, cam.translation,
                                      cam.focal_length, cam.principal_point)
    x = np.concatenate([np.asarray(points, np.float64), np.ones((len(points), 1))], 1) @ P[:3].T
    return x[:, :2] / x[:, 2:3]


def reprojection_rms(points, cam, ref_cam):
    """RMS distance in pixels between the projections of `points` in `cam` and in `ref_cam`."""
    e = project(points, cam) - project(points, ref_cam)
    return float(np.sqrt((e ** 2).sum(1).mean()))
