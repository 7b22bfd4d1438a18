"""Float64 reference of the volume-rendering stage, with a per-element error bound for every output.

TEST INFRASTRUCTURE ONLY.  It restates csrc/composite.cu (hrf_ray_offsets; hrf_prune = visibility, count scan and
compaction; hrf_composite_forward; hrf_composite_backward) and the compositing epilogue of csrc/field_fwd.cu with its
fix-up kernel (hrf_render_fused, hrf_render_fused_depth), i.e. nerfacc 0.3.1's render_visibility,
render_weight_from_density and accumulate_along_rays as humanrf/volume_rendering.py calls them.

Inputs are the kernels' own float32 arrays.  What the kernels compute exactly is mirrored exactly: dt = fl32(fl32(t +
step) - t), t_mid = fl32(0.5 * fl32(t + fl32(t + step))).  Everything else is float64, and exclusive sums are running
sums taken before each sample is added, so a density of +inf renders as nerfacc renders it: that sample is opaque
(weight T, transmittance 0 behind it), and nothing is NaN.

Error model.  u = 2^-24 is the fp32 unit roundoff.  A sum of non-negative terms formed by fp32 additions in any order
and grouping, k additions deep, is within k u of the exact sum times the sum itself.  __expf(x) is within
(2 + floor(1.173 |x|)) ulp of exp(x) (CUDA Programming Guide, intrinsic functions), i.e. that many 2^-23 relative; its
result flushes to zero below 2^-126.  The kernels' operation order gives the depth k of each sum:

* unfused (composite.cu, warp per ray, 32-sample chunks): the exclusive optical depth of a sample in chunk c is a
  shuffle scan of at most 31 terms plus the running carry, at most 32 + c additions, plus the rounding of sigma * dt;
  colour and weight sums are per-lane running sums over the chunks then a 5-level butterfly.
* fused (field_fwd.cu, 128-sample tiles): a segmented scan within the tile (31 lane additions + 3 warp carries + the
  shift) gives the depth relative to the segment; the fix-up chains the tiles' partials in order, one addition and one
  __expf per tile, and scales each partial by its T.  A sample's weight is thus T_tile * __expf(-depth in tile) * alpha:
  two __expf and one more product than the unfused kernel.
* backward: d(sigma_k dt_k) = g_k T_k exp(-sdt_k) - sum_{i>k} g_i w_i.  The kernel forms the suffix as
  total - (prefix + inclusive), which cancels: its error is bounded by (2 chunks + 14) u sum_i |g_i w_i| over the ray,
  plus the error of the terms behind k.  A sample behind an opaque prefix (T = 0) therefore may carry noise of exactly
  that size and no larger.

Visibility (render_visibility) is an fp32 product T_k = prod_{j<k} (1 - alpha_j) with alpha_j = 1 - expf(-sigma_j step)
(the accurate expf, 2 ulp).  The reference carries T as an interval [T_lo, T_hi]; a sample's keep decision is
ambiguous only where that interval (or alpha's) straddles its threshold, and only there may the kernel differ.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24        # fp32 unit roundoff
ULP = 2.0 ** -23      # one ulp of a normal fp32 value, relative
TINY = 2.0 ** -125    # absolute slack for results that flush to zero / subnormals
LANES = 32
TILE = 128
SCAN_BLOCK = 1024     # scan_i32_kernel's block


def f32(x):
    return np.asarray(x, np.float32)


def dt32(t, step):
    t, s = f32(t), np.float32(step)
    return (t + s) - t


def tmid32(t, step):
    t, s = f32(t), np.float32(step)
    return np.float32(0.5) * (t + (t + s))


def expf_rel(x):
    """Relative error bound of __expf(-x) for x >= 0 (+inf gives an exact 0, bound 0)."""
    x = np.abs(np.asarray(x, np.float64))
    return np.where(np.isinf(x), 0.0, (2.0 + np.floor(1.173 * np.where(np.isinf(x), 0.0, x))) * ULP)


def _mul0(a, b):
    """a * b with 0 * inf = 0 (an exact zero times an unbounded bound is still an exact zero)."""
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    out = np.zeros(a.shape)
    nz = (a != 0) & (b != 0)
    out[nz] = a[nz] * b[nz]
    return out


def ray_offsets(ray_indices, num_rays):
    """hrf_ray_offsets: lower bound of every ray index 0..num_rays in the sorted ray indices."""
    return np.searchsorted(np.asarray(ray_indices, np.int64), np.arange(num_rays + 1), side="left").astype(np.int64)


def ray_of(off):
    off = np.asarray(off, np.int64)
    return np.repeat(np.arange(off.shape[0] - 1), np.diff(off))


def seg_excl_sum(x, off):
    """Exclusive running sum per ray, in float64: the sum of the samples before each one (+inf stays +inf after it)."""
    out = np.zeros(x.shape[0])
    for b, e in zip(off[:-1], off[1:]):
        if e - b > 1:
            out[b + 1:e] = np.cumsum(x[b:e - 1])
    return out


def seg_excl_prod(x, off):
    out = np.ones(x.shape[0])
    for b, e in zip(off[:-1], off[1:]):
        if e - b > 1:
            out[b + 1:e] = np.cumprod(x[b:e - 1])
    return out


def seg_suffix_sum(x, off):
    """sum_{i>k} x_i per ray, as a running sum from the back."""
    out = np.zeros(x.shape[0])
    for b, e in zip(off[:-1], off[1:]):
        if e - b > 1:
            out[b:e - 1] = np.cumsum(x[b + 1:e][::-1])[::-1]
    return out


def per_ray(x, off):
    return np.bincount(ray_of(off), weights=x, minlength=off.shape[0] - 1) if x.shape[0] else np.zeros(off.shape[0] - 1)


# ---------------------------------------------------------------------------------------------------------------------
# hrf_prune
# ---------------------------------------------------------------------------------------------------------------------
def visibility(sigma, off, step, eps=1e-4, thre=1e-4):
    """keep (float64 decision), ambiguous (where the kernel may decide either way), per-ray kept counts of `keep`."""
    s = f32(sigma).astype(np.float64)
    x = s * float(np.float32(step))                            # exact in float64; the kernel rounds it once
    inf = np.isinf(x)
    xf = np.where(inf, 0.0, x)
    om = np.exp(-x)                                            # 1 - alpha, 0 for +inf
    alpha = -np.expm1(-x)
    de = np.where(inf, 0.0, om * (2 * ULP + 1.01 * xf * U)) + TINY     # expf: 2 ulp, plus the argument's rounding
    dalpha = de * (1 + U) + U * alpha                          # fl(1 - e)
    dom = dalpha + U * (om + dalpha)                           # fl(1 - alpha)
    zero = x == 0                                              # expf(-0) = 1: alpha = 0 and 1 - alpha = 1 exactly
    dalpha, dom = np.where(zero, 0.0, dalpha), np.where(zero, 0.0, dom)
    T = seg_excl_prod(om, off)
    pos = np.arange(s.shape[0]) - np.repeat(np.asarray(off[:-1]), np.diff(off))
    mults = pos + pos // LANES + 1                             # fp32 products in the scan and the carry
    T_lo = seg_excl_prod(np.maximum(om - dom, 0.0), off) * np.exp(-mults * 1.01 * U)
    T_hi = seg_excl_prod(om + dom, off) * np.exp(mults * 1.01 * U) + TINY
    exact = seg_excl_prod(zero.astype(np.float64), off) == 1   # only factors of exactly 1 before: T = 1 exactly
    T_lo, T_hi = np.where(exact, 1.0, T_lo), np.where(exact, 1.0, T_hi)
    e32, t32 = float(np.float32(eps)), float(np.float32(thre))
    keep = (T >= e32) & (alpha >= t32)
    a_lo, a_hi = alpha - dalpha, alpha + dalpha
    amb = ((T_lo < e32) & (T_hi >= e32) & (a_hi >= t32)) | ((a_lo < t32) & (a_hi >= t32) & (T_hi >= e32))
    return keep, amb, T


def kept_offsets(keep, off):
    """Exclusive scan of the kept counts (hrf_prune's in-place count scan), length num_rays + 1."""
    c = per_ray(np.asarray(keep, np.float64), off).astype(np.int64)
    return np.concatenate(([0], np.cumsum(c)))


def compact(keep, t, off):
    """Compaction of the kept samples: (distances, ray indices, source index), in sample order."""
    keep = np.asarray(keep, bool)
    src = np.nonzero(keep)[0]
    return f32(t)[src], ray_of(off)[src], src


# ---------------------------------------------------------------------------------------------------------------------
# compositing
# ---------------------------------------------------------------------------------------------------------------------
class Forward:
    """Weights, colour, weights sum, depth sum w t_mid, with bounds, for kernel = "unfused" or "fused"."""

    def __init__(self, sigma, rgb, t, off, step, bg=None, kernel="unfused"):
        off = np.asarray(off, np.int64)
        self.off, self.kernel = off, kernel
        n, R = int(off[-1]), off.shape[0] - 1
        s = f32(sigma)[:n].astype(np.float64)
        c = f32(rgb)[:n].astype(np.float64).reshape(n, 3)
        self.dt = dt32(f32(t)[:n], step).astype(np.float64)
        self.tmid = tmid32(f32(t)[:n], step).astype(np.float64)
        b = np.repeat(off[:-1], np.diff(off))
        pos = np.arange(n) - b
        sdt = s * self.dt
        self.sdt = sdt
        inf = np.isinf(sdt)
        sdtf = np.where(inf, 0.0, sdt)
        excl = seg_excl_sum(sdt, off)
        self.excl = excl
        T = np.exp(-excl)
        if kernel == "unfused":
            n_add = 33 + pos // LANES                                     # shuffle scan + carry + sigma*dt
            t_rel = expf_rel(excl)
            n_sum = (np.diff(off) + LANES - 1) // LANES + 6               # lane running sums + product + butterfly
        else:
            tiles_before = np.arange(n) // TILE - b // TILE               # tile borders between the ray start and k
            n_add = 37 + tiles_before
            # T_tile = __expf(-depth of the earlier tiles), then __expf(-depth within this tile): both arguments <= excl
            t_rel = 2 * expf_rel(excl) + 2 * U
            ntiles = np.where(np.diff(off) > 0, (off[1:] - 1) // TILE - off[:-1] // TILE + 1, 0)
            n_sum = 36 + ntiles                                           # segmented scan + carries + chain
        dex = _mul0(n_add * 1.01 * U, excl)
        self.dT = _mul0(T, (1 + t_rel) * np.exp(dex) - 1) + TINY
        ea = np.exp(-sdt)
        alpha = -np.expm1(-sdt)
        self.de = np.where(inf, 0.0, ea * (expf_rel(sdt) + 1.01 * U * sdtf)) + TINY    # __expf(-fl(sigma dt))
        dalpha = self.de + U * (alpha + self.de)
        w = T * alpha
        dw = (T + self.dT) * (alpha + dalpha) * (1 + U) - w + TINY
        self.T, self.ea, self.alpha, self.w, self.dw = T, ea, alpha, w, dw
        self.n_sum_ray = n_sum
        ns = n_sum[ray_of(off)] if np.ndim(n_sum) else n_sum
        self.color = np.stack([per_ray(w * c[:, k], off) for k in range(3)], 1)
        self.color_err = np.stack([per_ray(dw * c[:, k] + ns * U * w * c[:, k], off) for k in range(3)], 1)
        self.wsum = per_ray(w, off)
        self.wsum_err = per_ray(dw + ns * U * w, off)
        self.depth = per_ray(w * self.tmid, off)
        self.depth_err = per_ray((dw + ns * U * w) * self.tmid, off)
        self.weights_err = dw
        if bg is not None:
            bgv = f32(bg).astype(np.float64).reshape(R, 3)
            k = 1.0 - self.wsum
            self.color = self.color + bgv * k[:, None]
            self.color_err = (self.color_err + bgv * (self.wsum_err + U * np.abs(k))[:, None] * (1 + U)
                              + U * np.abs(bgv * k[:, None]) + U * np.abs(self.color))
        self.weights = w


class Backward:
    """Analytic backward of colour (with the background blend) and weights sum, for the unfused kernel."""

    def __init__(self, F: Forward, rgb, bg, dcolor, dwsum):
        off = F.off
        n, R = int(off[-1]), off.shape[0] - 1
        ray = ray_of(off)
        c = f32(rgb)[:n].astype(np.float64).reshape(n, 3)
        d = f32(dcolor).astype(np.float64).reshape(R, 3)
        gw = np.zeros(R) if dwsum is None else f32(dwsum).astype(np.float64).reshape(R).copy()
        gabs = np.abs(gw)
        if bg is not None:
            bgv = f32(bg).astype(np.float64).reshape(R, 3)
            gw -= (d * bgv).sum(1)
            gabs = gabs + np.abs(d * bgv).sum(1)
        g = (d[ray] * c).sum(1) + gw[ray]
        dg = 6 * U * (np.abs(d[ray] * c).sum(1) + gabs[ray])
        gwv = g * F.w
        dgw = np.abs(g) * F.dw + dg * F.w + 2 * U * np.abs(gwv)
        suffix = seg_suffix_sum(gwv, off)
        nch = (np.diff(off) + LANES - 1) // LANES
        sgw = per_ray(np.abs(gwv), off)
        dsuffix = seg_suffix_sum(dgw, off) + ((2 * nch + 14) * U * sgw)[ray]
        A = g * F.T * F.ea
        dA = (np.abs(g) * (_mul0(F.dT, F.ea) + _mul0(F.T, F.de) + _mul0(F.dT, F.de)) + dg * F.T * F.ea
              + 2 * U * np.abs(A))
        self.g = g
        self.d_sigma = (A - suffix) * F.dt
        self.d_sigma_err = F.dt * (dA + dsuffix) * (1 + 2 * U) + 2 * U * np.abs(self.d_sigma)
        self.d_rgb = F.w[:, None] * d[ray]
        self.d_rgb_err = F.dw[:, None] * np.abs(d[ray]) + U * np.abs(self.d_rgb) + TINY


def ratio(got, ref, bound):
    """Largest |got - ref| / bound (0 / 0 counts as 0; a difference where the bound is 0 is inf; NaN is inf)."""
    got, ref, bound = (np.asarray(x, np.float64) for x in (got, ref, bound))
    err = np.abs(got - ref)
    err = np.where(got == ref, 0.0, err)          # equal infinities
    err = np.where(np.isnan(err), np.inf, err)
    r = np.full(err.shape, np.inf)
    np.divide(err, bound, out=r, where=bound > 0)
    r[err == 0] = 0.0
    return float(r.max()) if r.size else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# fp32 restatements of the kernels, each with one optional deliberate mistake
# ---------------------------------------------------------------------------------------------------------------------
MUTANTS = ("no_lane_carry", "inclusive_T", "step_for_dt", "background_sign", "d_sigma_without_dt",
           "fixup_without_T", "scan_without_block_carry")


def _chunks(x, b, e):
    """Samples b..e of a ray padded to whole 32-lane chunks: [chunks, 32] fp32."""
    m = e - b
    nc = (m + LANES - 1) // LANES
    out = np.zeros(nc * LANES, np.float32)
    out[:m] = x[b:e]
    return out.reshape(nc, LANES)


def _excl_chunked(sdt, mutant):
    """The unfused kernel's exclusive optical depth of one ray's chunks (fp32)."""
    incl = np.cumsum(sdt, axis=1, dtype=np.float32)
    tot = incl[:, -1]
    carry = np.concatenate(([0], np.cumsum(tot, dtype=np.float32)[:-1])).astype(np.float32)
    shifted = np.concatenate([np.zeros((sdt.shape[0], 1), np.float32), incl[:, :-1]], 1)
    if mutant == "no_lane_carry":
        return shifted
    if mutant == "inclusive_T":
        return carry[:, None] + incl
    return carry[:, None] + shifted


def kernel_forward32(sigma, rgb, t, off, step, bg=None, mutant=None):
    """composite_fwd_kernel in fp32 numpy: (weights, color, wsum)."""
    off = np.asarray(off, np.int64)
    n, R = int(off[-1]), off.shape[0] - 1
    dt = np.full(n, np.float32(step)) if mutant == "step_for_dt" else dt32(f32(t)[:n], step)
    sdt = f32(sigma)[:n] * dt
    rgb = f32(rgb).reshape(-1, 3)
    w_out = np.zeros(n, np.float32)
    color = np.zeros((R, 3), np.float32)
    ws = np.zeros(R, np.float32)
    for r in range(R):
        b, e = off[r], off[r + 1]
        if e == b:
            continue
        s = _chunks(sdt, b, e)
        excl = _excl_chunked(s, mutant)
        w = (np.exp(-excl) * (np.float32(1) - np.exp(-s))).reshape(-1)[:e - b].astype(np.float32)
        w_out[b:e] = w
        color[r] = (w[:, None] * rgb[b:e]).sum(0, dtype=np.float32)
        ws[r] = w.sum(dtype=np.float32)
    if bg is not None:
        sign = np.float32(-1 if mutant == "background_sign" else 1)
        color = color + sign * f32(bg).reshape(R, 3) * (np.float32(1) - ws)[:, None]
    return w_out, color, ws


def kernel_backward32(sigma, rgb, t, off, step, bg, dcolor, dwsum, mutant=None):
    """composite_bwd_kernel in fp32 numpy: (d_sigma, d_rgb)."""
    off = np.asarray(off, np.int64)
    n, R = int(off[-1]), off.shape[0] - 1
    dt = dt32(f32(t)[:n], step)
    sdt = f32(sigma)[:n] * dt
    rgb = f32(rgb).reshape(-1, 3)
    d = f32(dcolor).reshape(R, 3)
    gw = np.zeros(R, np.float32) if dwsum is None else f32(dwsum).reshape(R).copy()
    if bg is not None:
        gw = gw - (d * f32(bg).reshape(R, 3)).sum(1, dtype=np.float32)
    ds = np.zeros(n, np.float32)
    drgb = np.zeros((n, 3), np.float32)
    for r in range(R):
        b, e = off[r], off[r + 1]
        if e == b:
            continue
        s = _chunks(sdt, b, e)
        T = np.exp(-_excl_chunked(s, None)).reshape(-1)[:e - b]
        ea = np.exp(-s).reshape(-1)[:e - b]
        w = T * (np.float32(1) - ea)
        g = (rgb[b:e] * d[r]).sum(1, dtype=np.float32) + gw[r]
        gwv = g * w
        suffix = np.cumsum(gwv[::-1], dtype=np.float32)[::-1] - gwv
        v = g * T * ea - suffix
        ds[b:e] = v if mutant == "d_sigma_without_dt" else v * dt[b:e]
        drgb[b:e] = w[:, None] * d[r]
    return ds, drgb


def fused_forward32(sigma, rgb, t, off, step, bg=None, mutant=None):
    """The fused epilogue + fix-up in fp32 numpy: each ray is cut at 128-sample tile borders; a segment's weights are
    relative to its start, and the segments are chained with T = exp(-depth of the earlier segments).
    Returns (color, wsum, depth sum w t_mid)."""
    off = np.asarray(off, np.int64)
    n, R = int(off[-1]), off.shape[0] - 1
    dt = dt32(f32(t)[:n], step)
    tm = tmid32(f32(t)[:n], step)
    sdt = f32(sigma)[:n] * dt
    rgb = f32(rgb).reshape(-1, 3)
    color = np.zeros((R, 3), np.float32)
    ws = np.zeros(R, np.float32)
    dep = np.zeros(R, np.float32)
    for r in range(R):
        b, e = off[r], off[r + 1]
        depth = np.float32(0)
        k = b
        while k < e:
            kend = min(e, (k // TILE + 1) * TILE)
            s = sdt[k:kend]
            incl = np.cumsum(s, dtype=np.float32)
            excl = np.concatenate(([0], incl[:-1])).astype(np.float32)
            w = (np.exp(-excl) * (np.float32(1) - np.exp(-s))).astype(np.float32)
            T = np.float32(1) if mutant == "fixup_without_T" else np.exp(-depth).astype(np.float32)
            color[r] += T * (w[:, None] * rgb[k:kend]).sum(0, dtype=np.float32)
            ws[r] += T * w.sum(dtype=np.float32)
            dep[r] += T * (w * tm[k:kend]).sum(dtype=np.float32)
            depth = np.float32(depth + incl[-1])
            k = kend
    if bg is not None:
        color = color + f32(bg).reshape(R, 3) * (np.float32(1) - ws)[:, None]
    return color, ws, dep


def scan32(counts, mutant=None):
    """scan_i32_kernel: exclusive scan in blocks of 1024 with a carry between blocks; length n + 1."""
    c = np.asarray(counts, np.int64)
    out = np.zeros(c.shape[0] + 1, np.int64)
    carry = 0
    for base in range(0, c.shape[0], SCAN_BLOCK):
        blk = c[base:base + SCAN_BLOCK]
        if mutant == "scan_without_block_carry":
            carry = 0
        incl = np.cumsum(blk)
        out[base:base + blk.shape[0]] = carry + incl - blk
        carry = carry + int(incl[-1])
    out[-1] = carry
    return out


# ---------------------------------------------------------------------------------------------------------------------
# inputs shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------
STEP = 4e-4
SPECIAL_LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 4100)
REGIMES = ("zero", "tiny", "typical", "opaque", "inf", "mixed")


def _sigma_of(regime, m, rng):
    if regime == "zero":
        return np.zeros(m)
    if regime == "tiny":
        return np.full(m, 1e-6)
    if regime == "opaque":
        return np.full(m, 1e4)
    s = rng.random(m) ** 4 * 400.0
    s[rng.random(m) < 0.3] *= 1e-3
    if regime == "inf" and m:
        s[rng.integers(0, m)] = np.inf
    if regime == "mixed" and m:
        s[rng.random(m) < 0.05] = 0.0
        s[rng.random(m) < 0.02] = 1e4
    return s


def ray_batch(num_rays=2600, max_random=200, seed=0):
    """Rays of every special length under every density regime (0, 1e-6, typical, 1e4, one +inf, mixed), then random
    lengths 0..max_random with random regimes: num_rays rays in all (more than 2048, not a multiple of 1024).
    t_k = t_0 + k step in fp32 with t_0 in [0.5, 6.2], so t reaches about 8 and dt = (t + step) - t differs from step."""
    rng = np.random.default_rng(seed)
    lens, regs = [], []
    for reg in REGIMES:
        for m in SPECIAL_LENGTHS:
            lens.append(m), regs.append(reg)
    while len(lens) < num_rays:
        lens.append(int(rng.integers(0, max_random + 1))), regs.append(REGIMES[int(rng.integers(0, len(REGIMES)))])
    order = rng.permutation(num_rays)
    lens, regs = [lens[i] for i in order], [regs[i] for i in order]
    sigma = np.concatenate([_sigma_of(r, m, rng) for r, m in zip(regs, lens)]).astype(np.float32)
    counts = np.asarray(lens, np.int64)
    ri = np.repeat(np.arange(num_rays), counts)
    off = np.concatenate(([0], np.cumsum(counts)))
    k = np.arange(ri.shape[0]) - off[:-1][ri]
    t0 = rng.uniform(0.5, 6.2, num_rays).astype(np.float32)
    t = (t0[ri] + k.astype(np.float32) * np.float32(STEP)).astype(np.float32)
    n = t.shape[0]
    return dict(sigma=sigma, rgb=rng.random((n, 3)).astype(np.float32), t=t, ri=ri, off=off, num_rays=num_rays,
                bg=rng.random((num_rays, 3)).astype(np.float32),
                dcolor=rng.standard_normal((num_rays, 3)).astype(np.float32),
                dwsum=rng.standard_normal(num_rays).astype(np.float32))
