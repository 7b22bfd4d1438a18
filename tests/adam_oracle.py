"""Float64 reference for one step of the fused Adam kernels (hrf_adam_multi, hrf_dp_reduce_adam, hrf_adam_step), with an
entrywise error bound on each output, plus the input sets the CPU and GPU tests share.

TEST INFRASTRUCTURE ONLY.

The kernels (csrc/common.cuh adam_update), per element, all in fp32:
    s   = g_0 + g_1 + ... + g_{W-1}            (rank order; W = 1 outside the data-parallel exchange)
    g'  = s * gscale
    m'  = fma(b1, m, (1-b1) g')
    v'  = fma(b2, v, ((1-b2) g') g')
    p'  = fma(-lr1, m' / (sqrt(v') / bc2s + eps), p)
    bc1 = 1 - powf(b1, k), bc2s = sqrtf(1 - powf(b2, k)), lr1 = lr / bc1           (k = the tensor's step counter)

Rules of the reference:
* Gradient sum.  s is formed in fp32 in rank order exactly as the kernels do (pure adds: numpy reproduces it bit for
  bit, `grad_sum`).  Everything after it is float64 of the kernel's fp32 inputs and scalars, widened.
* Each output is referenced from the kernel's own values of what it reads: m' and v' from the state (p, m, v) before
  the step, p' from the kernel's own m' and v' (so errors do not compound), and each step starts from the kernel's state
  after the previous one.
* Rounding budget.  One rounding of a result x errs by at most u|x| (u = 2^-24) or, where x is subnormal, by half a
  subnormal ulp (2^-150) absolute.  The bound takes, over the absolute value of each term, one u per rounding that
  term passes through (as gamma_n = n u / (1 - n u)), plus 2^-150 per rounding:
    m': b1 m passes <= 2 roundings (the fma, or its own product if the compiler does not contract),
        (1-b1) g' passes 3 (the grad_scale product, the (1-b1) product, the fma).
    v': b2 v <= 2;  (1-b2) g'^2 passes 5 (g' enters twice, two products, the fma).
    p': the final fma (u |p'|) plus, on the step lr/B1 * m'/D, the relative errors of lr1, sqrtf, the divide by bc2s,
        the eps add (weighted by the sqrt term's share of D), the divide and the bias corrections.  Second-order terms
        are covered by a factor 1 + 1e-3.
  These hold for either contraction order (`emulate_fp32` runs both).
* powf.  The CUDA Math API documentation gives powf a maximum error of 4 ulp over the full range (POWF_ULP); one ulp
  of y is at most 2^-23 |y| for a normal y and 2^-149 for a subnormal one.  1 - b (b in [0.5, 1]) and 1 - b^k for
  b^k >= 0.5 are exact by Sterbenz's lemma; only 1 - b^k for b^k < 0.5 takes a rounding.  The relative error of
  powf's result is amplified by b^k / (1 - b^k) in the bias correction; at b2 = 0.99, k = 1 that is 99.
* Underflow and overflow (`regime`):
    NORMAL     bounded as above;
    SUBNORMAL  (1-b2) g'^2 lies in the fp32 subnormal range: still bounded, the absolute 2^-150 terms carry it;
    UNDERFLOW  (1-b2) g'^2 rounds to 0: v' is not referenced in float64; the rule (fp32 torch.optim.Adam) is
               v' == fl(b2 v) bit for bit.  p' stays bounded from the kernel's v' -- where v' = 0 the step is m'/eps
               sized: lr/B1 * m'/eps;
    OVERFLOW   v' rounds to +inf: the rule is v' = inf and p' == p (m'/inf = 0).  m' stays bounded;
    AMBIGUOUS  within the rounding band of either threshold: the input sets must have none.
  m' is bounded in every regime.
* Copies.  The bf16 shadows equal torch's .to(torch.bfloat16) of the kernel's fp32 p' (round to nearest even), and
  vectors_t equals `transpose_vectors`, a restatement of the [4, VR, 32] -> [4, 16, VR, 2] layout of field_common.cuh.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                       # unit roundoff of fp32
ETA = 2.0 ** -150                    # half a subnormal ulp: the absolute error of one rounding into the subnormals
SUB_ULP = 2.0 ** -149
POWF_ULP = 4                         # CUDA Math API: powf(x, y), maximum ulp error over the full range
FLT_MIN_NORMAL = 2.0 ** -126
OVERFLOW_AT = (2.0 - 2.0 ** -24) * 2.0 ** 127    # exact values at or above this round to +inf
SECOND_ORDER = 1.0 + 1e-3

NORMAL, SUBNORMAL, UNDERFLOW, OVERFLOW, AMBIGUOUS = range(5)
REGIME_NAMES = ("normal", "subnormal", "underflow", "overflow", "ambiguous")


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


@dataclass
class Scalars:
    """The kernel's fp32 arguments (lr, beta1, beta2, eps, grad_scale), stored as fp32 and widened where used."""
    lr: float = 1e-2
    b1: float = 0.9
    b2: float = 0.99
    eps: float = 1e-15
    gscale: float = 1.0

    def __post_init__(self):
        for k in ("lr", "b1", "b2", "eps", "gscale"):
            setattr(self, k, float(F32(getattr(self, k))))


def grad_sum(grads) -> np.ndarray:
    """fp32 sum over the ranks in rank order (the kernels' order, bit for bit)."""
    grads = [np.asarray(g, F32) for g in grads]
    s = grads[0].copy()
    for g in grads[1:]:
        s = (s + g).astype(F32)
    return s


def _powf_abs_err(b: float, k: int) -> float:
    y = b ** k
    return POWF_ULP * (2.0 ** -23 * y if y >= FLT_MIN_NORMAL else SUB_ULP)


def bias_correction(b: float, k: int):
    """(1 - b^k in float64, bound on |fl(1 - powf(b, k)) - (1 - b^k)|)."""
    y = b ** k
    e = _powf_abs_err(b, k)
    if y < 0.5 * (1.0 + 1e-6):       # Sterbenz: 1 - y is exact for y in [0.5, 2]
        e += U * (1.0 - y + e)
    return 1.0 - y, e


@dataclass
class Step:
    m: np.ndarray          # float64 references
    v: np.ndarray
    p: np.ndarray
    bm: np.ndarray         # entrywise bounds
    bv: np.ndarray
    bp: np.ndarray
    regime: np.ndarray     # int8, NORMAL ... AMBIGUOUS
    v_rule: np.ndarray     # fp32: what v' must equal bit for bit in the UNDERFLOW / OVERFLOW regimes

    @property
    def v_bounded(self):
        return (self.regime == NORMAL) | (self.regime == SUBNORMAL)

    @property
    def p_bounded(self):
        return self.regime != OVERFLOW


def moments(m, v, grads, sc: Scalars):
    """(M, V, bound_m, bound_v, regime, v_rule) from the kernel's fp32 state before the step and the per-rank gradients."""
    m32, v32 = np.asarray(m, F32), np.asarray(v, F32)
    G = grad_sum(grads).astype(F64) * sc.gscale
    m64, v64 = m32.astype(F64), v32.astype(F64)
    b1, b2 = sc.b1, sc.b2
    t1 = (1.0 - b1) * G
    t2 = (1.0 - b2) * G * G
    M = b1 * m64 + t1
    V = b2 * v64 + t2
    bm = gamma(2) * np.abs(b1 * m64) + gamma(3) * np.abs(t1) + 3 * ETA
    bv = gamma(2) * b2 * np.abs(v64) + gamma(5) * t2 + 4 * ETA
    regime = np.full(G.shape, NORMAL, np.int8)
    g5 = gamma(5)
    with np.errstate(over="ignore", invalid="ignore"):
        sub = t2 < FLT_MIN_NORMAL
        regime[sub & (t2 * (1 - g5) >= ETA)] = SUBNORMAL
        regime[t2 == 0] = NORMAL                                     # a zero gradient: nothing rounds
        regime[(t2 > 0) & (t2 * (1 + g5) < ETA)] = UNDERFLOW
        regime[(t2 > 0) & (t2 * (1 + g5) >= ETA) & (t2 * (1 - g5) < ETA)] = AMBIGUOUS
        vv = np.where(np.isinf(V), np.inf, V)
        regime[vv * (1 - g5) >= OVERFLOW_AT] = OVERFLOW
        regime[(vv * (1 - g5) < OVERFLOW_AT) & (vv * (1 + g5) >= OVERFLOW_AT)] = AMBIGUOUS
    v_rule = np.where(regime == OVERFLOW, F32(np.inf), (F32(b2) * v32).astype(F32)).astype(F32)
    return M, V, bm, bv, regime, v_rule


def param(p, m_new, v_new, k: int, sc: Scalars):
    """(P, bound_p) from the kernel's fp32 p before the step and its own m', v' after it, at step counter k >= 1."""
    p64 = np.asarray(p, F32).astype(F64)
    mk, vk = np.asarray(m_new, F32).astype(F64), np.asarray(v_new, F32).astype(F64)
    B1, e1 = bias_correction(sc.b1, k)
    B2, e2 = bias_correction(sc.b2, k)
    r1, r2 = e1 / B1, e2 / B2
    r2s = 0.5 * r2 + U                               # sqrtf of bc2
    r_lr = r1 + U                                    # lr / bc1
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        Q = np.sqrt(vk) / np.sqrt(B2)
        D = Q + sc.eps
        share = np.where(np.isinf(Q), 1.0, Q / D)
        r_d = U + (2 * U + r2s) * share              # sqrtf, / bc2s, + eps
        r_r = U + r_d                                # m' / d
        step = (sc.lr / B1) * np.where(np.isinf(D), 0.0, mk / D)
        P = p64 - step
        bp = SECOND_ORDER * (U * np.abs(P) + np.abs(step) * (r_lr + r_r)) + 2 * ETA
    return P, bp


def reference(p, m, v, grads, k: int, sc: Scalars, m_new, v_new) -> Step:
    M, V, bm, bv, regime, v_rule = moments(m, v, grads, sc)
    P, bp = param(p, m_new, v_new, k, sc)
    return Step(M, V, P, bm, bv, bp, regime, v_rule)


def check(got_p, got_m, got_v, p, ref: Step):
    """Worst err/bound per output and regime over the bounded entries, and the rule entries' pass flags.  Returns a dict
    name -> (worst err/bound or None, entries); raises AssertionError on a broken rule."""
    gp, gm, gv = (np.asarray(a, F32) for a in (got_p, got_m, got_v))
    out = {}
    assert not (ref.regime == AMBIGUOUS).any(), "an input sits on a regime threshold"
    with np.errstate(invalid="ignore", over="ignore"):
        em = np.abs(gm.astype(F64) - ref.m) / ref.bm
        ev = np.abs(gv.astype(F64) - ref.v) / ref.bv
        ep = np.abs(gp.astype(F64) - ref.p) / ref.bp
    for r in (NORMAL, SUBNORMAL, UNDERFLOW, OVERFLOW):
        sel = ref.regime == r
        n = int(sel.sum())
        if n == 0:
            continue
        name = REGIME_NAMES[r]
        out[f"m/{name}"] = (float(np.max(em[sel])), n)
        if r in (NORMAL, SUBNORMAL):
            out[f"v/{name}"] = (float(np.max(ev[sel])), n)
        else:
            bad = np.nonzero(gv[sel].view(np.uint32) != ref.v_rule[sel].view(np.uint32))[0]
            assert bad.size == 0, f"v' rule broken in the {name} regime at {np.nonzero(sel)[0][bad[:5]]}"
            out[f"v/{name} (rule)"] = (None, n)
        if r != OVERFLOW:
            out[f"p/{name}"] = (float(np.max(ep[sel])), n)
        else:
            p32 = np.asarray(p, F32)
            bad = np.nonzero(gp[sel] != p32[sel])[0]          # (a zero may change sign: -0 + +0 = +0)
            assert bad.size == 0, f"p moved where v' = inf at {np.nonzero(sel)[0][bad[:5]]}"
            out[f"p/{name} (rule)"] = (None, n)
    return out


def worst(stats) -> float:
    vals = [w for w, _ in stats.values() if w is not None]
    return max(vals) if vals else 0.0


def transpose_vectors(vec) -> np.ndarray:
    """vectors [4, VR, 32] (flat) -> vectors_t [4 axes][16 levels][VR rows][2 features] (flat), field_common.cuh."""
    a = np.asarray(vec)
    vr = a.size // (4 * 32)
    return a.reshape(4, vr, 16, 2).transpose(0, 2, 1, 3).reshape(-1).copy()


# ------------------------------------------------------------------------------------------- fp32 emulation (CPU tests)
def _fma32(a, b, c):
    """fp32 fma through float64: a*b is exact in float64; the add rounds twice (to float64, then fp32), which stays
    within one fp32 rounding plus 2^-53 relative -- inside the bound's gamma slack."""
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64) + np.asarray(c, F32).astype(F64)).astype(F32)


def emulate_fp32(p, m, v, grads, k: int, sc: Scalars, contract: str = "kernel"):
    """The kernels' fp32 arithmetic on the CPU.  contract="kernel": adam_update's order (fma over b1 m and b2 v);
    "other": fma over the gradient term with b1 m and b2 v rounded first; "none": every product and add rounded.
    bc1/bc2 use float64 powers rounded to fp32 (powf is within 1 ulp of that here)."""
    f = F32
    s = grad_sum(grads)
    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        g = (s * f(sc.gscale)).astype(f)
        omb1, omb2 = f(1) - f(sc.b1), f(1) - f(sc.b2)
        c1 = (omb1 * g).astype(f)
        c2 = ((omb2 * g).astype(f) * g).astype(f)
        m32, v32 = np.asarray(m, f), np.asarray(v, f)
        if contract == "kernel":
            mn, vn = _fma32(f(sc.b1), m32, c1), _fma32(f(sc.b2), v32, c2)
        elif contract == "other":
            mn = _fma32(g, omb1, (f(sc.b1) * m32).astype(f))
            vn = _fma32(g, (omb2 * g).astype(f), (f(sc.b2) * v32).astype(f))
        else:
            mn = ((f(sc.b1) * m32).astype(f) + c1).astype(f)
            vn = ((f(sc.b2) * v32).astype(f) + c2).astype(f)
        bc1 = f(1) - f(F64(sc.b1) ** k)
        bc2 = f(1) - f(F64(sc.b2) ** k)
        bc2s = np.sqrt(bc2).astype(f)
        lr1 = f(f(sc.lr) / bc1)
        d = ((np.sqrt(vn).astype(f) / bc2s).astype(f) + f(sc.eps)).astype(f)
        q = (mn / d).astype(f)
        if contract == "none":
            pn = (np.asarray(p, f) - (lr1 * q).astype(f)).astype(f)
        else:
            pn = _fma32(-lr1, q, np.asarray(p, f))
    return pn, mn, vn


# ------------------------------------------------------------------------------------------- wrong steps (CPU tests)
def _mutant_p(p, m_new, v_new, k, sc, eps_inside=False):
    mk, vk = np.asarray(m_new, F32).astype(F64), np.asarray(v_new, F32).astype(F64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        B1, B2 = F64(1.0) - F64(sc.b1) ** k, F64(1.0) - F64(sc.b2) ** k
        D = np.sqrt(vk / B2 + sc.eps) if eps_inside else np.sqrt(vk) / np.sqrt(B2) + sc.eps
        return np.asarray(p, F32).astype(F64) - (sc.lr / B1) * np.where(np.isinf(D), 0.0, mk / D)


def mutant(name, p, m, v, grads, k, sc: Scalars, m_new, v_new):
    """(m', v', p') of a deliberately wrong step in float64.  Like the reference, its p' is formed from the kernel's m'
    and v' (m_new, v_new); a mutant of the moments leaves p' to the reference (None)."""
    m64, v64 = np.asarray(m, F32).astype(F64), np.asarray(v, F32).astype(F64)
    b1, b2 = sc.b1, sc.b2
    order = list(grads)[::-1] if name == "reverse_rank_order" else list(grads)
    G = grad_sum(order).astype(F64) * sc.gscale
    M, V = b1 * m64 + (1 - b1) * G, b2 * v64 + (1 - b2) * G * G
    if name == "grad_scale_after_moments":
        S = grad_sum(grads).astype(F64)
        M = sc.gscale * (b1 * m64 + (1 - b1) * S)
        V = sc.gscale ** 2 * (b2 * v64 + (1 - b2) * S * S)
    if name == "bias_correction_off_by_one":
        return M, V, _mutant_p(p, m_new, v_new, k - 1, sc)
    if name == "eps_inside_sqrt":
        return M, V, _mutant_p(p, m_new, v_new, k, sc, eps_inside=True)
    return M, V, None


MUTANTS = ("bias_correction_off_by_one", "eps_inside_sqrt", "grad_scale_after_moments", "reverse_rank_order")


def mutant_ratio(name, p, m, v, grads, k, sc, kernel_m, kernel_v):
    """Worst |mutant - reference| / bound over the entries the reference bounds."""
    ref = reference(p, m, v, grads, k, sc, kernel_m, kernel_v)
    M, V, P = mutant(name, p, m, v, grads, k, sc, kernel_m, kernel_v)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        r = [np.abs(M - ref.m) / ref.bm, np.where(ref.v_bounded, np.abs(V - ref.v) / ref.bv, 0.0)]
        if P is not None:
            r.append(np.where(ref.p_bounded, np.abs(P - ref.p) / ref.bp, 0.0))
    vals = np.concatenate([np.nan_to_num(x, nan=np.inf).ravel() for x in r])
    return float(np.max(vals))


# ------------------------------------------------------------------------------------------- inputs
# Gradient magnitudes every edge-case tensor cycles through (per entry, fixed across steps; each step draws a fresh
# mantissa in [0.5, 2) and a random sign): zero, underflowing, subnormal, tiny, ordinary, large, overflowing squares.
MAGNITUDES = (0.0, 1e-30, 1e-21, 1e-19, 1e-3, 1.0, 1e3, 1e20, 4e20)
P_SCALES = (0.0, 1e-17, 1.0)      # parameter magnitudes (p = 0 makes the underflow regime's m'/eps step visible)


def edge_gradients(rng, n, ranks=1, cancel=False):
    """[ranks, n] fp32 per-rank gradients whose sum has the entry's magnitude class; with `cancel`, every third entry
    also gets random terms of 1e4 times its magnitude that sum to zero over the ranks, so its fp32 sum depends on the
    order."""
    idx = np.arange(n)
    mag = np.asarray(MAGNITUDES)[idx % len(MAGNITUDES)]
    val = mag * rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)
    out = np.zeros((ranks, n), F64)
    if ranks == 1:
        out[0] = val
    else:
        parts = rng.uniform(0.0, 2.0, (ranks, n))
        out[:] = val * parts / parts.sum(0)
        if cancel:
            big = mag * 1e4 * rng.standard_normal((ranks, n))
            big[-1] = -big[:-1].sum(0)
            sel = (idx % 3 == 0)
            out[:, sel] += big[:, sel]
    return out.astype(F32)


def edge_state(rng, n):
    """(p, m, v) fp32 of a tensor before the first step: p at the P_SCALES magnitudes, moments zero (a fresh optimiser)."""
    idx = np.arange(n)
    ps = np.asarray(P_SCALES)[(idx // len(MAGNITUDES)) % len(P_SCALES)]
    p = (rng.standard_normal(n) * ps + 0.0).astype(F32)     # (+ 0.0: no negative zeros)
    return p, np.zeros(n, F32), np.zeros(n, F32)


CPU_STEPS = (1, 2, 10, 1_000_000)


def cpu_sequence(seed=0, n=4096, gscale=1.0, ranks=1, cancel=False, contract="kernel"):
    """The step sequence of the GPU edge-case test on one tensor, in fp32 emulation: yields (k, p, m, v, grads, p', m', v')
    for k in 1, 2, ..., 10 and then the large count."""
    rng = np.random.default_rng(seed)
    sc = Scalars(gscale=gscale)
    p, m, v = edge_state(rng, n)
    ks = list(range(1, 11)) + [1_000_000]
    for k in ks:
        grads = edge_gradients(rng, n, ranks, cancel)
        pn, mn, vn = emulate_fp32(p, m, v, grads, k, sc, contract)
        yield k, sc, p, m, v, grads, pn, mn, vn
        p, m, v = pn, mn, vn
