"""Rounding-faithful float64 reference of the field kernels' two MLPs, forward and backward.

TEST INFRASTRUCTURE ONLY.  It restates csrc/field_fwd.cu:126-158 (+ field_mlp.cuh, field_common.cuh:write_color_input)
and csrc/field_bwd.cu:546-690 in float64 numpy, rounding to bf16 (round-to-nearest-even) exactly where the kernels
round and nowhere else:

  forward   hs = bf16(relu(W1s feat));  o = W2s hs (fp32);  sigma = exp(o0) * scale;  geo = bf16(o[0..15])
            cin = [bf16(SH4(d)) | bf16(o[1..15]) | bf16(emb[cam]) or 0 | 1.0 ...]  (K = 32 | 48)
            h1 = bf16(relu(W1c cin));  h2 = bf16(relu(W2c h1));  rgb = sigmoid((W3c h2)[:3])
  backward  g3 = bf16(d_rgb r (1 - r)) in cols 0..2, 0 elsewhere
            dH2 = bf16((g3 W3c) [h2 > 0]);  dH1 = bf16((dH2 W2c) [h1 > 0]);  dcin = dH1 W1c (fp32)
            d_emb[cam] += dcin[31..30+E] (valid cameras only)
            gs = bf16([d_sigma scale exp(clamp(h0, +-15)) | dcin[16..30] + d_geo]);  dHs = bf16((gs W2s) [hs > 0])
            dfeat = dHs W1s (fp32);  dW* = sum over samples of the outer products, in the d_mlp layout

Error model (every tolerance the tests use derives from these two constants):

* ``acc_delta(n)``: an fp32 sum of n exact terms (a bf16 x bf16 product is exact in fp32) computed in ANY order and
  grouping, with each addition rounded to nearest or truncated (the tensor cores' fused multi-term adders truncate), is
  within n * 2^-23 * sum|terms| of the exact sum: at most n roundings, each off by less than one fp32 ulp (2^-23
  relative) of a partial sum whose magnitude is at most sum|terms|.
* ``exp_eps(x)``: __expf(x) is ex2.approx(x * log2 e).  The product's rounding perturbs the exponent by at most
  |x log2 e| 2^-24, i.e. the result by |x| 2^-24 relative; ex2.approx.f32 has a documented maximum relative error of
  2^-22.  The bound used is 2^-21 + |x| 2^-23 (twice both).

An fp32 accumulation is **exact** when all its terms are multiples of 2^-q and sum|terms| < 2^(24-q): every partial sum
is then a multiple of 2^-q below 2^(24-q), representable in fp32, so no order and no adder can round.  For such a sum
the kernel's fp32 value equals the float64 value, and its bf16 rounding (RN-even, ties included) is determined.
Otherwise the kernel's value lies within ``e`` (the bound above) of the float64 value, and a bf16 rounding is
**ambiguous** when a rounding tie lies within e of the value, a relu mask when |value| <= e.  Ambiguity is tracked per
sample; a sample whose path has no ambiguous decision has exactly the reference's bf16 tiles, so its fp32 outputs
differ from the reference only by the accumulation bound of their last sum (**tight**), or not at all when every sum
on its path is exact (**exact**).

With ``rounding=False`` every bf16 rounding, __expf error and clamp-free detail is switched off: the same code is then
the plain float64 MLP and its hand-written backward, which the CPU suite checks against torch autograd.
"""
from __future__ import annotations

import numpy as np

U23 = 2.0 ** -23
TILE = 128
BIG = 1 << 20   # valuation of zero (no term)


def acc_delta(n):
    return n * U23


def exp_eps(x):
    return 2.0 ** -21 + np.abs(x) * U23


def bf16(x):
    """float64 -> nearest bf16 (8 significant bits, ties to even), as float64."""
    x = np.asarray(x, np.float64)
    _, e = np.frexp(x)
    s = np.ldexp(1.0, 8 - e)
    return np.round(x * s) / s    # np.round rounds half to even; the scaling is exact


def tie_distance(x):
    """Distance of x from the nearest bf16 rounding tie (midpoint of two neighbouring bf16 values)."""
    x = np.asarray(x, np.float64)
    _, e = np.frexp(x)
    t = np.abs(x) * np.ldexp(1.0, 8 - e)
    return np.abs(t - np.floor(t) - 0.5) * np.ldexp(1.0, e - 8)


def valuation(x):
    """Exponent of the lowest set bit of each float64 (BIG for zero): x is a multiple of 2^valuation(x)."""
    x = np.abs(np.asarray(x, np.float64))
    m, e = np.frexp(x)
    M = np.ldexp(m, 53).astype(np.int64)
    low = (M & -M).astype(np.float64)
    tz = np.frexp(low)[1] - 1
    return np.where(x == 0, BIG, e - 53 + tz).astype(np.int64)


def _minval_rows(X):
    return valuation(X).min(axis=1) if X.shape[1] else np.full(X.shape[0], BIG, np.int64)


def premise(S, vmin):
    """Exactness premise per output: terms multiples of 2^vmin (vmin = lowest term valuation) and S < 2^(24 + vmin)."""
    vmin = np.asarray(vmin, np.int64)
    none = vmin >= BIG // 2
    with np.errstate(over="ignore"):
        ok = S < np.ldexp(1.0, np.clip(24 + vmin, -1000, 1000))
    return none | ok


class Dense:
    """Y = X W^T with the bookkeeping the classifier needs: S = sum|terms|, exact premise, error bound e."""

    def __init__(self, X, W, n=None):
        self.v = X @ W.T
        self.S = np.abs(X) @ np.abs(W).T
        vmin = _minval_rows(X)[:, None] + _minval_rows(W)[None, :]
        vmin = np.where((vmin >= BIG // 2), BIG, vmin)
        self.exact = premise(self.S, vmin)
        self.e = np.where(self.exact, 0.0, acc_delta(n if n is not None else X.shape[1]) * self.S)


def round_amb(v, e):
    """(bf16(v), ambiguous): a rounding is ambiguous when a tie lies within the error bound e (> 0) of v."""
    return bf16(v), (e > 0) & (tie_distance(v) <= e)


def mask_amb(v, e):
    return (e > 0) & (np.abs(v) <= e)


# ---- deviation bounds of ambiguous samples --------------------------------------------------------------------------------
# An ambiguous sample's kernel tiles may differ from the reference's.  Each tile gets a bound D >= |kernel - reference|,
# propagated layer by layer: a sum's value moves by at most D_in @ |W| (inputs) + e (its own accumulation); relu is
# 1-Lipschitz; a bf16 rounding keeps two values that have no tie between them on the same bf16 number (D = 0) and
# otherwise moves them apart by at most their distance plus one bf16 ulp (2^-7 of the magnitude); a backward relu mask
# taken on a stored activation that might be 0 on one side and positive on the other passes or blocks the whole value.
# Non-ambiguous samples get D = 0 throughout, so the same arithmetic also gives them their usual bars.
def dev_relu_round(pre, tot, rounding=True):
    """Bound on |bf16(relu(x')) - bf16(relu(pre))| for |x' - pre| <= tot."""
    a = np.maximum(pre, 0.0)
    if not rounding:
        return np.zeros_like(pre)
    near0 = (np.abs(pre) < tot)
    flip = (pre >= tot) & (tot > 0) & (tie_distance(pre) <= tot)
    return np.where(near0, (a + tot) * (1 + 2.0 ** -7), np.where(flip, tot + 2.0 ** -7 * (a + tot), 0.0))


def dev_round(v, tot):
    """Bound on |bf16(x') - bf16(v)| for |x' - v| <= tot (no relu)."""
    near0 = np.abs(v) < tot
    flip = tie_distance(v) <= tot
    return np.where(near0, (np.abs(v) + tot) * (1 + 2.0 ** -7), np.where(flip & (tot > 0), tot + 2.0 ** -7 * (np.abs(v) + tot), 0.0))


def dev_mask(hq, dh):
    """Backward relu mask on a stored activation hq whose kernel value is within dh: can the mask differ?"""
    return ((hq > 0) & (hq <= dh)) | ((hq == 0) & (dh > 0))


# ---- SH4 (field_common.cuh:sh4), in float64 from the kernel's fp32 x, y, z, with sum|terms| per output ----------------
def sh4(d):
    d = np.asarray(d, np.float32)
    v = ((d + np.float32(1)) * np.float32(0.5)) * np.float32(2) - np.float32(1)   # fp32, as the kernel
    x, y, z = [v[:, i].astype(np.float64) for i in range(3)]
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    c = np.ones_like(x)
    vals = [0.28209479177387814 * c, -0.48860251190291987 * y, 0.48860251190291987 * z, -0.48860251190291987 * x,
            1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.94617469575755997 * z2 - 0.31539156525251999,
            -1.0925484305920792 * xz, 0.54627421529603959 * x2 - 0.54627421529603959 * y2,
            0.59004358992664352 * y * (-3.0 * x2 + y2), 2.8906114426405538 * xy * z,
            0.45704579946446572 * y * (1.0 - 5.0 * z2), 0.3731763325901154 * z * (5.0 * z2 - 3.0),
            0.45704579946446572 * x * (1.0 - 5.0 * z2), 1.4453057213202769 * z * (x2 - y2),
            0.59004358992664352 * x * (-x2 + 3.0 * y2)]
    ax, ay, az = np.abs(x), np.abs(y), np.abs(z)
    mags = [0.28209479177387814 * c, 0.49 * ay, 0.49 * az, 0.49 * ax, 1.1 * ax * ay, 1.1 * ay * az, 0.95 * z2 + 0.32,
            1.1 * ax * az, 0.55 * (x2 + y2), 0.6 * ay * (3 * x2 + y2), 2.9 * ax * ay * az, 0.46 * ay * (1 + 5 * z2),
            0.38 * az * (5 * z2 + 3), 0.46 * ax * (1 + 5 * z2), 1.45 * az * (x2 + y2), 0.6 * ax * (x2 + 3 * y2)]
    return np.stack(vals, 1), np.stack(mags, 1)


# sh4 is at most 8 fp32 operations per output (constants rounded to fp32 included, FMA contraction or not), each off by
# at most 2^-24 of a quantity bounded by that output's sum of |monomials|: 16 x 2^-24 is a safe bound.
SH_DELTA = 2.0 ** -20


def split_params(sigma_params, color_params, K):
    """Flat fp32 parameter vectors (sigma_net.params, color_net.params) -> bf16-rounded float64 matrices, as repack_mlp
    writes the blob: W1s [64,32], W2s [16,64], W1c [64,K], W2c [64,64], W3c [16,64]."""
    sp = np.asarray(sigma_params, np.float32).astype(np.float64)
    cp = np.asarray(color_params, np.float32).astype(np.float64)
    P = dict(W1s=sp[:2048].reshape(64, 32), W2s=sp[2048:3072].reshape(16, 64),
             W1c=cp[:64 * K].reshape(64, K), W2c=cp[64 * K:64 * K + 4096].reshape(64, 64),
             W3c=cp[64 * K + 4096:64 * K + 5120].reshape(16, 64))
    return {k: bf16(v) for k, v in P.items()}


def d_mlp_layout(dW1s, dW2s, dW1c, dW2c, dW3c):
    """Gradients in the kernel's d_mlp order (kGSig1, kGSig2, kGCol1, then colour W2 / W3; field_bwd.cu:684)."""
    return np.concatenate([m.reshape(-1) for m in (dW1s, dW2s, dW1c, dW2c, dW3c)])


class Forward:
    """Forward of both MLPs for a batch.  feat [N,32] (bf16 values), dirs [N,3] fp32, cams [N] (-1: no embedding),
    emb [C,E] fp32 table or None, P from split_params."""

    def __init__(self, feat, dirs, cams, emb, P, density_scale, K, rounding=True):
        rnd = bf16 if rounding else (lambda v: v)
        self.rounding = rounding
        N = feat.shape[0]
        self.N, self.K, self.P = N, K, P
        self.feat = np.asarray(feat, np.float64)
        self.cams = np.asarray(cams, np.int64) if cams is not None else np.full(N, -1, np.int64)
        E = 0 if emb is None else emb.shape[1]
        self.E = E
        amb = np.zeros(N, bool)
        # sigma net
        L1 = Dense(self.feat, P["W1s"])
        self.hs_pre, self.hs_e = L1.v, L1.e
        am = mask_amb(L1.v, L1.e)
        self.hs = rnd(np.maximum(L1.v, 0.0))
        ar = (L1.e > 0) & (L1.v > 0) & (tie_distance(L1.v) <= L1.e)
        amb |= (am | ar).any(1)
        exact = L1.exact.all(1)
        L2 = Dense(self.hs, P["W2s"])
        self.o, self.o_e, self.o_S = L2.v, L2.e, L2.S
        geo, ag = round_amb(L2.v, L2.e)
        self.geo = geo if rounding else L2.v                      # bf16(o[0..15]) as the forward writes it
        amb |= ag.any(1)
        exact &= L2.exact.all(1)
        self.amb_geo, self.exact_geo = amb.copy(), exact & ~amb
        h0 = L2.v[:, 0]
        self.sigma = np.exp(h0) * density_scale
        # |d sigma| <= sigma (exp error + error of h0) + one fp32 product
        self.sigma_tol = self.sigma * (exp_eps(h0) + 1.01 * L2.e[:, 0] + U23) if rounding else np.zeros(N)
        # colour input
        sh, shm = sh4(dirs)
        she = SH_DELTA * shm if rounding else np.zeros_like(shm)
        cin = np.ones((N, K))
        cin[:, :16] = rnd(sh)
        ash = (she > 0) & (tie_distance(sh) <= she) if rounding else np.zeros_like(sh, bool)
        amb |= ash.any(1)
        cin[:, 16:31] = self.geo[:, 1:16]
        if E:
            ok = self.cams >= 0
            rows = np.zeros((N, E))
            rows[ok] = np.asarray(emb, np.float32).astype(np.float64)[self.cams[ok]]
            cin[:, 31:31 + E] = rnd(rows)
        self.cin = cin
        L3 = Dense(cin, P["W1c"])
        self.h1_pre, self.h1_e = L3.v, L3.e
        self.h1 = rnd(np.maximum(L3.v, 0.0))
        a3 = mask_amb(L3.v, L3.e) | ((L3.e > 0) & (L3.v > 0) & (tie_distance(L3.v) <= L3.e))
        L4 = Dense(self.h1, P["W2c"])
        self.h2_pre, self.h2_e = L4.v, L4.e
        self.h2 = rnd(np.maximum(L4.v, 0.0))
        a4 = mask_amb(L4.v, L4.e) | ((L4.e > 0) & (L4.v > 0) & (tie_distance(L4.v) <= L4.e))
        L5 = Dense(self.h2, P["W3c"][:3])
        self.oc, self.oc_e = L5.v, L5.e
        self.rgb = 1.0 / (1.0 + np.exp(-L5.v))
        r = self.rgb
        # |d r| <= r (1 - r) (exp error + error of the pre-activation) + the add and the IEEE division
        self.rgb_tol = (r * (1 - r) * (exp_eps(L5.v) + 1.01 * L5.e) + 2 * U23 * r) if rounding else np.zeros_like(r)
        amb |= a3.any(1) | a4.any(1)
        self.amb = amb if rounding else np.zeros(N, bool)
        self.exact = (exact & L3.exact.all(1) & L4.exact.all(1) & L5.exact.all(1) & ~amb) if rounding else np.zeros(N, bool)
        if not rounding:
            self.amb_geo = np.zeros(N, bool)
            self.exact_geo = np.zeros(N, bool)
        # deviation bounds (see dev_relu_round); SH rounding: within she of its value
        if rounding:
            Dh = dev_relu_round(L1.v, L1.e)
            Do_pre = Dh @ np.abs(P["W2s"]).T
            self.D_o = Do_pre + L2.e                                   # fp32 o vs the reference's o
            Dcin = np.zeros((N, K))
            Dcin[:, :16] = dev_round(sh, she)
            Dcin[:, 16:31] = dev_round(L2.v[:, 1:16], self.D_o[:, 1:16])
            self.D_geo = dev_round(L2.v, self.D_o)                     # geo bits as stored
            D1 = dev_relu_round(L3.v, Dcin @ np.abs(P["W1c"]).T + L3.e)
            D2 = dev_relu_round(L4.v, D1 @ np.abs(P["W2c"]).T + L4.e)
            self.D_oc = D2 @ np.abs(P["W3c"][:3]).T + L5.e
            self.D = dict(hs=Dh, cin=Dcin, h1=D1, h2=D2, feat=np.zeros((N, 32)))
            # sigma and rgb of any sample: exp / sigmoid of a pre-activation within D of the reference's
            self.sigma_dev = self.sigma * (np.expm1(np.minimum(self.D_o[:, 0], 50.0)) + exp_eps(h0) + U23)
            self.rgb_dev = 0.25 * self.D_oc + r * (1 - r) * exp_eps(L5.v) + 2 * U23 * r

    def classes(self):
        """(exact, tight, ambiguous) sample counts of the whole forward."""
        return int(self.exact.sum()), int((~self.exact & ~self.amb).sum()), int(self.amb.sum())


class Backward:
    """Backward of both MLPs from a Forward.  d_sigma [N] | None, d_rgb [N,3] | None, d_geo [N,15] | None.
    num_cameras: rows of the embedding table (d_emb is [num_cameras, E])."""

    def __init__(self, F: Forward, d_sigma, d_rgb, d_geo, density_scale, num_cameras=0, wgrad_chain=None,
                 invert_mask=None):
        rounding = F.rounding
        rnd = bf16 if rounding else (lambda v: v)
        P, N, K, E = F.P, F.N, F.K, F.E
        amb = F.amb.copy()
        exact = F.exact.copy()
        # d(colour pre-activation), only the three used outputs
        g3 = np.zeros((N, 16))
        g3e = np.zeros((N, 3))
        if d_rgb is not None:
            r = F.rgb
            v3 = np.asarray(d_rgb, np.float64) * r * (1 - r)
            # r (1 - r) has relative error <= 2 (exp error + error of the pre-activation) + the add, the division, 1 - r
            # and the two products (5 roundings of 2^-24 each, rounded up to 2^-21)
            g3e = np.abs(v3) * (2 * (exp_eps(F.oc) + F.oc_e) + 2.0 ** -21) if rounding else np.zeros_like(v3)
            g3[:, :3] = rnd(v3)
            if rounding:
                amb |= ((g3e > 0) & (tie_distance(v3) <= g3e)).any(1)
            exact &= (v3 == 0).all(1) | (not rounding)     # __expf-derived: never provably exact unless zero
        self.g3 = g3
        h2m = F.h2 > 0
        h1m = F.h1 > 0
        hsm = F.hs > 0
        if invert_mask is not None:              # deliberately wrong reference: one unit's relu mask inverted
            which, j = invert_mask
            {"h2": h2m, "h1": h1m, "hs": hsm}[which][:, j] ^= True
        D2 = Dense(g3[:, :3], P["W3c"][:3].T)
        v = D2.v * h2m
        a = ((D2.e > 0) & h2m & (tie_distance(D2.v) <= D2.e))
        self.dH2 = rnd(v)
        amb |= a.any(1)
        exact &= (D2.exact | ~h2m).all(1)
        D1 = Dense(self.dH2, P["W2c"].T)
        v = D1.v * h1m
        a = ((D1.e > 0) & h1m & (tie_distance(D1.v) <= D1.e))
        self.dH1 = rnd(v)
        amb |= a.any(1)
        exact &= (D1.exact | ~h1m).all(1)
        DC = Dense(self.dH1, P["W1c"].T)
        self.dcin, self.dcin_e, self.dcin_S = DC.v, DC.e, DC.S
        exact_dcin = DC.exact
        # d(sigma-net output)
        gs = np.zeros((N, 16))
        gse = np.zeros((N, 16))
        if d_sigma is not None:
            h0 = F.o[:, 0]
            hc = np.clip(h0, -15, 15) if rounding else h0
            v0 = np.asarray(d_sigma, np.float64) * density_scale * np.exp(hc)
            gse[:, 0] = np.abs(v0) * (exp_eps(hc) + 1.01 * F.o_e[:, 0] * (np.abs(h0) < 15) + 2 * U23) if rounding else 0.0
            gs[:, 0] = v0
            exact &= (v0 == 0) | (not rounding)
        dg = np.zeros((N, 15)) if d_geo is None else np.asarray(d_geo, np.float32).astype(np.float64)
        gs[:, 1:] = DC.v[:, 16:31] + dg
        # one more fp32 addition on top of the colour net's sum: its bound over n + 1 terms, and the premise with d_geo
        S1 = DC.S[:, 16:31] + np.abs(dg)
        vmin = np.minimum(_minval_rows(self.dH1)[:, None] + _minval_rows(P["W1c"].T[16:31])[None, :], valuation(dg))
        ex1 = premise(S1, vmin)
        gse[:, 1:] = np.where(ex1, 0.0, acc_delta(65) * S1) if rounding else 0.0
        exact &= ex1.all(1)
        self.gs_exact = gs.copy()              # the unrounded value (the autograd check reads it as d(geo), d(o0))
        a = (gse > 0) & (tie_distance(gs) <= gse)
        self.gs = rnd(gs)
        if rounding:
            amb |= a.any(1)
        DS = Dense(self.gs, P["W2s"].T)
        v = DS.v * hsm
        a = ((DS.e > 0) & hsm & (tie_distance(DS.v) <= DS.e))
        self.dHs = rnd(v)
        amb |= a.any(1)
        exact &= (DS.exact | ~hsm).all(1)
        DF = Dense(self.dHs, P["W1s"].T)
        self.dfeat, self.dfeat_e = DF.v, DF.e
        if rounding:
            D = F.D
            Dg3 = np.zeros((N, 16))
            if d_rgb is not None:
                # |d r(1-r) / do| <= 1/10 (max of r (1-r) |1 - 2r|), plus the __expf-derived bound g3e
                dv3 = np.abs(np.asarray(d_rgb, np.float64)) * 0.1 * F.D_oc + g3e
                Dg3[:, :3] = dev_round(v3, dv3)
            Dp = Dg3[:, :3] @ np.abs(P["W3c"][:3]) + D2.e
            f2 = dev_mask(F.h2, D["h2"])
            DdH2 = dev_round(D2.v * h2m, np.where(f2, np.abs(D2.v) + Dp, Dp * h2m))
            Dp = DdH2 @ np.abs(P["W2c"]) + D1.e
            f1 = dev_mask(F.h1, D["h1"])
            DdH1 = dev_round(D1.v * h1m, np.where(f1, np.abs(D1.v) + Dp, Dp * h1m))
            self.dcin_dev = DdH1 @ np.abs(P["W1c"]) + DC.e
            Dgs = np.zeros((N, 16))
            if d_sigma is not None:
                Dgs[:, 0] = dev_round(gs[:, 0], np.abs(gs[:, 0]) * np.expm1(np.minimum(F.D_o[:, 0], 50.0)) + gse[:, 0])
            Dgs[:, 1:] = dev_round(gs[:, 1:], self.dcin_dev[:, 16:31] + gse[:, 1:])
            Dp = Dgs @ np.abs(P["W2s"]) + DS.e
            fs = dev_mask(F.hs, D["hs"])
            DdHs = dev_round(DS.v * hsm, np.where(fs, np.abs(DS.v) + Dp, Dp * hsm))
            self.dfeat_dev = DdHs @ np.abs(P["W1s"]) + DF.e
            self.D = dict(D, g3=Dg3, dH2=DdH2, dH1=DdH1, gs=Dgs, dHs=DdHs)
        self.amb = amb if rounding else np.zeros(N, bool)
        self.exact_dfeat = (exact & DF.exact.all(1) & ~amb) if rounding else np.zeros(N, bool)
        self.exact = self.exact_dfeat
        # camera-embedding gradient
        self.d_emb = np.zeros((num_cameras, E))
        if E:
            ok = (F.cams >= 0) & (F.cams < num_cameras)
            np.add.at(self.d_emb, F.cams[ok], DC.v[ok, 31:31 + E])
        # weight gradients: sums over the batch, fp32 chains of at most `wgrad_chain` additions
        outs = [(self.dHs, F.feat), (self.gs, F.hs), (self.dH1, F.cin), (self.dH2, F.h1), (g3, F.h2)]
        self.d_mlp = d_mlp_layout(*[a_.T @ b_ for a_, b_ in outs])
        self.d_mlp_S = d_mlp_layout(*[np.abs(a_).T @ np.abs(b_) for a_, b_ in outs])
        amb_s = self.amb
        # an ambiguous sample's kernel contribution a' b' differs from a b by at most |a| Db + Da |b| + Da Db
        names = (("dHs", "feat"), ("gs", "hs"), ("dH1", "cin"), ("dH2", "h1"), ("g3", "h2"))
        if rounding:
            Dd = self.D
            self.d_mlp_A = d_mlp_layout(*[np.abs(a_[amb_s]).T @ Dd[nb][amb_s] + Dd[na][amb_s].T @ np.abs(b_[amb_s])
                                          + Dd[na][amb_s].T @ Dd[nb][amb_s] for (a_, b_), (na, nb) in zip(outs, names)])
        else:
            self.d_mlp_A = np.zeros_like(self.d_mlp)
        vm = []
        for a_, b_ in outs:
            va = np.where(np.abs(a_) > 0, valuation(a_), BIG).min(0)
            vb = np.where(np.abs(b_) > 0, valuation(b_), BIG).min(0)
            vm.append(np.where((va[:, None] >= BIG // 2) | (vb[None, :] >= BIG // 2), BIG, va[:, None] + vb[None, :]))
        self.d_mlp_exact = premise(self.d_mlp_S, d_mlp_layout(*vm)) & (self.d_mlp_A == 0) if rounding else None
        n_chain = wgrad_chain if wgrad_chain is not None else N
        self.d_mlp_tol = acc_delta(n_chain) * self.d_mlp_S + self.d_mlp_A

    def classes(self):
        return int(self.exact.sum()), int((~self.exact & ~self.amb).sum()), int(self.amb.sum())


def wgrad_chain(num_samples, num_ctas):
    """Longest fp32 addition chain of one weight-gradient entry: the 128 products of each tile a CTA owns, accumulated in
    its registers across its tiles, then one atomic add per CTA."""
    tiles = (num_samples + TILE - 1) // TILE
    per_cta = (tiles + num_ctas - 1) // num_ctas
    return TILE * per_cta + num_ctas


# ---- comparators ------------------------------------------------------------------------------------------------------
def compare_rows(got, ref, tol, exact, amb, dev):
    """Per-sample comparison: bit-identical on exact rows, |d| <= tol on tight rows, |d| <= dev (the propagated deviation
    bound, which includes the accumulation bound) on ambiguous rows; all entrywise.  Returns (ok, report)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    n = ref.shape[0]
    d = np.abs(got - ref).reshape(n, -1)
    tol = np.broadcast_to(np.asarray(tol, np.float64), ref.shape).reshape(n, -1)
    dev = np.broadcast_to(np.asarray(dev, np.float64), ref.shape).reshape(n, -1)
    tight = ~exact & ~amb
    bad_exact = exact & (d != 0).any(1)
    bad_tight = tight & ~(d <= tol).all(1)
    bad_amb = amb & ~(d <= dev).all(1)
    worst = float(np.max(np.where((exact | tight)[:, None], d, 0.0), initial=0.0))
    ratio = lambda m, b: float(np.max(np.where(m[:, None], d / np.maximum(b, 1e-300), 0.0), initial=0.0))  # noqa: E731
    rep = dict(n=n, exact=int(exact.sum()), tight=int(tight.sum()), ambiguous=int(amb.sum()),
               amb_share=float(amb.mean()) if n else 0.0, bad_exact=int(bad_exact.sum()), bad_tight=int(bad_tight.sum()),
               bad_amb=int(bad_amb.sum()), worst_nonamb=worst, worst_tight_over_bar=ratio(tight, tol),
               worst_amb_over_bar=ratio(amb, dev))
    ok = rep["bad_exact"] == 0 and rep["bad_tight"] == 0 and rep["bad_amb"] == 0 and np.isfinite(got).all()
    return bool(ok), rep


def compare_dmlp(got, B: Backward):
    """d_mlp: bit-identical on entries whose whole-batch sum is provably exact and touched by no ambiguous deviation;
    |d| <= acc_delta(chain) S + A elsewhere (A: the ambiguous samples' deviation bound, see Backward)."""
    got = np.asarray(got, np.float64)
    d = np.abs(got - B.d_mlp)
    ex = B.d_mlp_exact if B.d_mlp_exact is not None else np.zeros_like(d, bool)
    bad_exact = int((ex & (d != 0)).sum())
    bad = int((~ex & ~(d <= B.d_mlp_tol)).sum())
    rel = float(np.linalg.norm(got - B.d_mlp) / max(np.linalg.norm(B.d_mlp), 1e-300))
    rep = dict(entries=len(d), exact_entries=int(ex.sum()), bad_exact=bad_exact, bad=bad, relnorm=rel,
               worst_over_bar=float(np.max(np.where(~ex, d / np.maximum(B.d_mlp_tol, 1e-300), 0.0), initial=0.0)))
    return bool(bad_exact == 0 and bad == 0), rep


# ---- dyadic inputs: sparse powers of two, so that most sums are provably exact ------------------------------------------
def _dyadic(rng, shape, p_zero, exps):
    v = rng.choice([-1.0, 1.0], size=shape) * np.ldexp(1.0, -rng.choice(exps, size=shape))
    return np.where(rng.random(shape) < p_zero, 0.0, v)


def dyadic_params(rng, K):
    """fp32 (sigma_params, color_params) whose entries are 0 or +-2^-j: bf16-exact, and short sums stay exact."""
    W = [_dyadic(rng, (64, 32), 0.7, [1, 2, 3]), _dyadic(rng, (16, 64), 0.7, [2, 3, 4]), _dyadic(rng, (64, K), 0.7, [1, 2, 3]),
         _dyadic(rng, (64, 64), 0.7, [2, 3, 4]), _dyadic(rng, (16, 64), 0.7, [2, 3])]
    return (np.concatenate([w.reshape(-1) for w in W[:2]]).astype(np.float32),
            np.concatenate([w.reshape(-1) for w in W[2:]]).astype(np.float32))


def dyadic_features(rng, n):
    return rng.integers(-8, 9, size=(n, 32)) / 8.0


def axis_directions(rng, n):
    """Axis-aligned unit directions: SH4 of them is a handful of constants."""
    d = np.zeros((n, 3), np.float32)
    d[np.arange(n), rng.integers(0, 3, n)] = rng.choice([-1.0, 1.0], n)
    return d


def dyadic_upstream(rng, n):
    """(d_sigma, d_rgb, d_geo), multiples of 2^-10 / 2^-6 / 2^-6."""
    return (rng.integers(-8, 9, size=n) / 1024.0).astype(np.float32), \
        (rng.integers(-8, 9, size=(n, 3)) / 64.0).astype(np.float32), (rng.integers(-8, 9, size=(n, 15)) / 64.0).astype(np.float32)
