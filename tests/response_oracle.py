"""Float64 reference of the per-camera colour response (hrf_train_loss_response, hrf_camera_response_step,
hrf_camera_response_apply; DESIGN.md §3.17).

With w = weights_sum, bg the background, fg = color - (1 - w) bg, em = expm1(gamma) and g = 1 + em = e^gamma:
    pred = color + em fg + w b
    dpred/dcolor = g,  dpred/dw = em bg + b,  dpred/dgamma = g fg,  dpred/db = w
The Huber term is taken on pred - gt with gt = rgb m + bg (1 - m); the BCE mask term is hrf_train_loss's.  The oracle
takes em and b from the float32 table the kernel reads, so its inputs are the kernel's exactly.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np

import pose_dp_oracle as PDO
import pose_oracle as PO

U = 2.0 ** -24          # fp32 unit roundoff


def pixel_model(color, w, bg, em, b):
    """(pred, dpred/dcolor, dpred/dw, dpred/dgamma, dpred/db), all [R,3]."""
    g = 1.0 + em
    W = w[:, None]
    fg = color - (1.0 - W) * bg
    pred = color + em * fg + W * b
    return pred, g, em * bg + b, g * fg, np.broadcast_to(W, pred.shape)


def table_of(params):
    """The float32 table [C,6] of float64 params [C,6] = (gamma, b): (expm1(gamma), b), rounded once."""
    params = np.asarray(params, np.float64)
    return np.concatenate((np.expm1(params[:, :3]), params[:, 3:]), 1).astype(np.float32)


def loss_and_grads(color, w, rgba, bg, cams, table, delta=0.01, bce_w=1e-3, scale=1.0, model=pixel_model):
    """hrf_train_loss_response in float64 on the kernel's inputs (float32 arrays; table [C,6] float32).  A camera number
    outside [0, C) takes the identity and is left out of the sums.  Returns a dict: loss, d_color [R,3], d_wsum [R],
    grad [C,6], count [C], and the intermediates the GPU tests derive their bounds from."""
    color, w, rgba, bg = (np.asarray(a, np.float64) for a in (color, w.reshape(-1), rgba, bg))
    table = np.asarray(table, np.float32).astype(np.float64)
    cams = np.asarray(cams).reshape(-1).astype(np.int64)
    R, C = color.shape[0], table.shape[0]
    valid = (cams >= 0) & (cams < C)
    em = np.zeros((R, 3))
    b = np.zeros((R, 3))
    em[valid], b[valid] = table[cams[valid], :3], table[cams[valid], 3:]
    pred, d_col, d_w, d_gamma, d_b = model(color, w, bg, em, b)
    m = rgba[:, 3:]
    gt = rgba[:, :3] * m + bg * (1.0 - m)
    x = pred - gt
    quad = np.abs(x) < delta
    huber = np.where(quad, 0.5 * x * x, delta * (np.abs(x) - 0.5 * delta))
    inv3r = 1.0 / (3 * R) if R else 0.0
    invr = 1.0 / R if R else 0.0
    pc = np.clip(w, 0.0, 1.0)
    mm = m[:, 0]
    bce = -(mm * np.log(pc + 1e-10) + (1 - mm) * np.log(1 - pc + 1e-10))
    dpc = -(mm / (pc + 1e-10) - (1 - mm) / (1 - pc + 1e-10))
    dw_bce = np.where((w >= 0) & (w <= 1), dpc * invr * bce_w * scale, 0.0)
    dpred = np.where(quad, x, np.copysign(delta, x)) * inv3r * scale
    grad = np.zeros((C, 6))
    count = np.bincount(cams[valid], minlength=C).astype(np.int32)
    np.add.at(grad, cams[valid], np.concatenate((dpred * d_gamma, dpred * d_b), 1)[valid])
    return {"loss": float(huber.sum() * inv3r + bce.sum() * invr * bce_w), "d_color": dpred * d_col,
            "d_wsum": dw_bce + (dpred * d_w).sum(1), "grad": grad, "count": count, "pred": pred, "x": x, "gt": gt,
            "dpred": dpred, "dw_bce": dw_bce, "em": em, "b": b, "fg": color - (1.0 - w[:, None]) * bg,
            "huber": huber, "bce": bce, "w": w, "g": 1.0 + table[:, :3]}


def apply(color, alpha, bg, row):
    """hrf_camera_response_apply in float64: color [P,3], alpha [P], bg [3], row = the camera's table row [6]."""
    row = np.asarray(row, np.float32).astype(np.float64)
    color, alpha = np.asarray(color, np.float64), np.asarray(alpha, np.float64).reshape(-1)
    pred, *_ = pixel_model(color, alpha, np.asarray(bg, np.float64)[None, :], row[None, :3], row[None, 3:])
    return pred


def adam(state, grad, count, fixed, lr, betas=(0.9, 0.99), eps=1e-15):
    """torch.optim.Adam per camera on params [C,6] = (gamma, b) (tests/pose_oracle.py's per-camera Adam)."""
    return PO.adam(state, grad, count, fixed, lr, betas, eps)


def ranked_step(state, grads, counts, errors, fixed, lr, betas=(0.9, 0.99), eps=1e-15):
    """One data-parallel response step of every replica, in place on `state`: the records reduced in rank order, the
    union of the touched cameras and the error words of tests/pose_dp_oracle.py.  Returns (g, touched, errors after)."""
    stop, after = PDO.error_words(errors)
    g, touched = PDO.reduce_records(grads, counts)
    if not stop:
        adam(state, g, touched.astype(np.int64), fixed, lr, betas, eps)
    return g, touched, after
