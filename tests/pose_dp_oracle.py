"""Float64 reference of the data-parallel pose step (hrf_camera_pose_step_ranks, hrf_camera_calib_step_ranks, DESIGN.md
§3.16): every rank's gradient record reduced in rank order, the union of the touched cameras, the error words, then the
single-rank step of tests/pose_oracle.py (pose only) or tests/intrinsics_oracle.py (with intrinsics).

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import numpy as np

import intrinsics_oracle as IO
import pose_oracle as PO


def reduce_records(grads, counts):
    """(g [C,K] float64, touched bool [C]) of W ranks' gradients grads[r] [C,K] and ray counts counts[r] [C]:
    g = (sum over r = 0..W-1, in rank order, of float64(grads[r])) / W -- the kernel's additions, one at a time, so the
    result is its bits -- and touched = some rank's count > 0."""
    W = len(grads)
    s = np.asarray(grads[0]).astype(np.float64)
    for r in range(1, W):
        s = s + np.asarray(grads[r]).astype(np.float64)
    touched = np.zeros(s.shape[0], bool)
    for c in counts:
        touched |= np.asarray(c) != 0
    return s / W, touched


def error_words(errors):
    """(stop, errors after the step): no rank writes when any word is set; a rank that sees bit 0 in another rank's word
    sets bit 1 of its own."""
    errors = [int(e) for e in errors]
    stop = any(errors)
    after = [e | (2 if any(o & 1 for q, o in enumerate(errors) if q != r) else 0) for r, e in enumerate(errors)]
    return stop, after


def ranked_step(state, grads, counts, errors, fixed, lr, lr_intrinsics=None, betas=(0.9, 0.99), eps=1e-15):
    """One data-parallel step of every replica, in place on `state` (dict(params [C,6 or 10], m, v, steps), the
    parameters in (omega, tau[, alpha, beta]) order).  grads[r] holds rank r's pose gradient [C,6], or pose and
    intrinsics side by side [C,10] when lr_intrinsics is given.  Returns (reduced gradient, touched, errors after)."""
    stop, after = error_words(errors)
    g, touched = reduce_records(grads, counts)
    if stop:
        return g, touched, after
    if lr_intrinsics is None:
        PO.adam(state, g, touched.astype(np.int64), fixed, lr, betas, eps)
    else:
        IO.adam(state, g, touched.astype(np.int64), fixed, lr, lr_intrinsics, betas, eps)
    return g, touched, after
