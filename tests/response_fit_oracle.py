"""Float64 reference of the held-out response fit (hrf_response_fit_accumulate, hrf_response_fit_solve; DESIGN.md §3.18).

Per camera and channel, the gain g and offset b minimising
    sum over the fit pixels of (g f + a b - y / 255)^2  +  lambda n ((g - 1)^2 + b^2)
with f the rendered colour, a its alpha and y the dataset's 8-bit colour.  The moments row is
    [n, S_aa, then per channel: S_ff, S_fa, S_fy, S_ay, S_yy]      (y the integer 0..255)
Every addend is exact in float64, and ``moments`` sums them with ``math.fsum`` (correctly rounded), so the kernel's
only error is its summation order.  ``solve`` takes the operations in the kernel's order, each rounded once.

TEST INFRASTRUCTURE ONLY.
"""
from __future__ import annotations

import math

import numpy as np

ROW = 17
OK, TOO_FEW, NOT_FINITE, GAIN_NOT_POSITIVE, BAD_CAMERA = 0, 1, 2, 3, 4


def addends(color, alpha, gt, mask):
    """The exact float64 addends of every row entry over the masked pixels, one array per entry (a generator: a
    12 MP view's 17 arrays would not fit in memory at once)."""
    m = np.asarray(mask).reshape(-1) != 0
    f = np.asarray(color, np.float32).reshape(-1, 3)[m]
    a = np.asarray(alpha, np.float32).reshape(-1)[m].astype(np.float64)
    y = np.asarray(gt, np.uint8).reshape(-1, 3)[m]
    yield np.ones(a.shape[0])
    yield a * a
    for k in range(3):
        fk, yk = f[:, k].astype(np.float64), y[:, k].astype(np.float64)
        yield from (fk * fk, fk * a, fk * yk, a * yk, yk * yk)


def moments(color, alpha, gt, mask):
    """(row float64 [17] correctly rounded, sum |addends| [17], addend count m)."""
    row, mag, m = np.zeros(ROW), np.zeros(ROW), 0
    for e, t in enumerate(addends(color, alpha, gt, mask)):
        row[e] = math.fsum(t.tolist())
        mag[e] = math.fsum(np.abs(t).tolist())
        m = t.shape[0]
    return row, mag, m


def solve_channel(n, saa, m, lam):
    """(g, b, SSE at the identity, SSE at (g, b)) of one channel from its moments m = (S_ff, S_fa, S_fy, S_ay, S_yy),
    in the kernel's operation order (Python floats: every operation rounded once)."""
    n, saa, lam = float(n), float(saa), float(lam)
    inv255 = 1.0 / 255.0
    sff, sfa, sfy, say = float(m[0]), float(m[1]), float(m[2]) * inv255, float(m[3]) * inv255
    syy = float(m[4]) * inv255 * inv255
    ln = lam * n
    a11, a22, r1 = sff + ln, saa + ln, sfy + ln
    det = a11 * a22 - sfa * sfa
    with np.errstate(divide="ignore", invalid="ignore"):
        g = float(np.float64(r1 * a22 - sfa * say) / np.float64(det))
        b = float(np.float64(a11 * say - sfa * r1) / np.float64(det))
    sse_id = (sff - 2.0 * sfy) + syy
    q = g * g * sff
    q = q + b * b * saa
    q = q + 2.0 * (g * b) * sfa
    q = q - 2.0 * g * sfy
    q = q - 2.0 * b * say
    return g, b, sse_id, q + syy


def solve(rows, cameras, lam, min_pixels, num_cameras=None):
    """hrf_response_fit_solve on moments rows [C,17]: (gains [K,3], offsets [K,3], report [K,8], status [K])."""
    rows = np.asarray(rows, np.float64)
    C = rows.shape[0] if num_cameras is None else num_cameras
    K = len(cameras)
    gains, offs, report, status = np.zeros((K, 3)), np.zeros((K, 3)), np.zeros((K, 8)), np.zeros(K, np.int32)
    for k, c in enumerate(cameras):
        if not 0 <= c < C:
            status[k] = BAD_CAMERA
            report[k, 7] = BAD_CAMERA
            continue
        row = rows[c]
        st = TOO_FEW if row[0] < min_pixels else OK
        report[k, 0] = row[0]
        for ch in range(3):
            g, b, e0, e1 = solve_channel(row[0], row[1], row[2 + 5 * ch:7 + 5 * ch], lam)
            gains[k, ch], offs[k, ch] = g, b
            report[k, 1 + ch], report[k, 4 + ch] = e0, e1
            if st == OK and not (math.isfinite(g) and math.isfinite(b)):
                st = NOT_FINITE
            if st == OK and not g > 0:
                st = GAIN_NOT_POSITIVE
        status[k] = st
        report[k, 7] = st
    return gains, offs, report, status


def direct_sse(color, alpha, gt, mask, g, b):
    """sum over the masked pixels of (g f + a b - y / 255)^2 per channel, by fsum of the rounded squares."""
    m = np.asarray(mask).reshape(-1) != 0
    f = np.asarray(color, np.float32).reshape(-1, 3)[m].astype(np.float64)
    a = np.asarray(alpha, np.float32).reshape(-1)[m].astype(np.float64)
    y = np.asarray(gt, np.uint8).reshape(-1, 3)[m].astype(np.float64) / 255.0
    return np.array([math.fsum(((g[k] * f[:, k] + a * b[k] - y[:, k]) ** 2).tolist()) for k in range(3)])
