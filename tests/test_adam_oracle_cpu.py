"""The fused-Adam reference (tests/adam_oracle.py) on the CPU: its bound holds for fp32 emulations of the update in every
contraction order, it agrees with fp32 torch.optim.Adam (foreach) within that bound and by its underflow / overflow
rules, every deliberately wrong step exceeds twice the bound on the inputs the GPU test feeds the kernels, and the
shadow / transposed-copy rules are what they say."""
import numpy as np
import pytest
import torch

import adam_oracle as A

SEQUENCES = {   # name -> cpu_sequence arguments (the GPU test's inputs: edge_state / edge_gradients per tensor)
    "w1": dict(seed=0, n=4096),
    "w1_scaled": dict(seed=1, n=4097, gscale=1.0 / 3.0),
    "w8_cancel": dict(seed=2, n=4096, gscale=1.0 / 8.0, ranks=8, cancel=True),
}


def _merge(acc, stats):
    for k, (w, n) in stats.items():
        w0, n0 = acc.get(k, (None, 0))
        acc[k] = (w if w0 is None else (w0 if w is None else max(w0, w)), n0 + n)


def _report(title, acc):
    print(f"\n{title}")
    for k in sorted(acc):
        w, n = acc[k]
        print(f"  {k:<24} {'rule' if w is None else f'{w:.3f}':>8}  ({n} entries)")


@pytest.mark.parametrize("contract", ["kernel", "other", "none"])
@pytest.mark.parametrize("seq", sorted(SEQUENCES))
def test_bound_holds_for_fp32_emulations(seq, contract):
    """fp32 emulations of the step (the kernels' fma order, the other contraction, no contraction) stay within the bound
    at steps 1..10 and a large step count, and the inputs reach the subnormal, underflow and overflow regimes."""
    acc = {}
    for k, sc, p, m, v, grads, pn, mn, vn in A.cpu_sequence(contract=contract, **SEQUENCES[seq]):
        ref = A.reference(p, m, v, grads, k, sc, mn, vn)
        stats = A.check(pn, mn, vn, p, ref)
        assert A.worst(stats) <= 1.0, (k, stats)
        _merge(acc, stats)
    _report(f"{seq} / {contract}: max err/bound", acc)
    # (at W = 8 the 1/8 grad_scale takes the 1e-21 gradients below the subnormals: no subnormal entries there)
    for regime in ("underflow", "overflow") if seq == "w8_cancel" else ("subnormal", "underflow", "overflow"):
        assert any(key.startswith(f"m/{regime}") for key in acc), (regime, sorted(acc))


@pytest.mark.parametrize("gscale", [1.0, 1.0 / 3.0])
def test_oracle_agrees_with_torch_adam(gscale):
    """fp32 torch.optim.Adam (foreach) -- the reference project's optimiser -- with the kernel's fp32 scalars widened:
    within the bound on the bounded entries, and it follows the underflow (v' = fl(b2 v)) and overflow (v' = inf,
    p unchanged) rules exactly."""
    rng = np.random.default_rng(7)
    n = 4096
    sc = A.Scalars(gscale=gscale)
    p0, _, _ = A.edge_state(rng, n)
    w = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([w], lr=sc.lr, betas=(sc.b1, sc.b2), eps=sc.eps, foreach=True)
    p, m, v = p0, np.zeros(n, np.float32), np.zeros(n, np.float32)
    acc = {}
    for k in range(1, 13):
        grads = A.edge_gradients(rng, n)
        g32 = (grads[0] * np.float32(gscale)).astype(np.float32)   # torch takes the scaled gradient
        # the reference scales inside: feed it the same fp32 g' (a grad_scale of 1 on the pre-scaled gradient)
        sc1 = A.Scalars(gscale=1.0)
        w.grad = torch.from_numpy(g32.copy())
        opt.step()
        st = opt.state[w]
        pn, mn, vn = w.detach().numpy().copy(), st["exp_avg"].numpy().copy(), st["exp_avg_sq"].numpy().copy()
        ref = A.reference(p, m, v, [g32], k, sc1, mn, vn)
        stats = A.check(pn, mn, vn, p, ref)
        assert A.worst(stats) <= 1.0, (k, stats)
        _merge(acc, stats)
        p, m, v = pn, mn, vn
    _report(f"torch.optim.Adam, grad_scale {gscale:.4f}: max err/bound", acc)
    assert any(key.startswith("v/underflow") for key in acc) and any(key.startswith("v/overflow") for key in acc)


@pytest.mark.parametrize("name", A.MUTANTS)
def test_wrong_steps_exceed_twice_the_bound(name):
    """Each deliberately wrong step, on the GPU test's inputs, lands more than twice the bound away from the reference
    somewhere: the bias correction one step behind, eps inside the sqrt, grad_scale applied after the moments, the
    rank sum in reverse order (W = 8, cancelling gradients)."""
    seq = {"reverse_rank_order": "w8_cancel", "grad_scale_after_moments": "w1_scaled"}.get(name, "w1")
    worst = 0.0
    for k, sc, p, m, v, grads, pn, mn, vn in A.cpu_sequence(**SEQUENCES[seq]):
        worst = max(worst, A.mutant_ratio(name, p, m, v, grads, k, sc, mn, vn))
    print(f"\nmutant {name} on {seq}: worst |mutant - reference| / bound = {worst:.3g}")
    assert worst > 2.0, (name, worst)


def test_reverse_rank_order_is_harmless_without_cancellation():
    """The rank-order mutant is only visible where the order changes the fp32 sum: at W = 1 it is the reference."""
    for k, sc, p, m, v, grads, pn, mn, vn in A.cpu_sequence(**SEQUENCES["w1"]):
        assert A.mutant_ratio("reverse_rank_order", p, m, v, grads, k, sc, mn, vn) <= 1.0


@pytest.mark.parametrize("vr", [1, 5, 2048])
def test_transpose_vectors_restates_the_layout(vr):
    """vectors [axis][row][2 * level + f] -> vectors_t [axis][level][row][f], element by element."""
    rng = np.random.default_rng(vr)
    vec = rng.standard_normal(4 * vr * 32).astype(np.float32)
    vt = A.transpose_vectors(vec)
    src = vec.reshape(4, vr, 32)
    want = np.empty(4 * 16 * vr * 2, np.float32)
    for axis in range(4):
        for level in range(16):
            for f in range(2):
                base = ((axis * 16 + level) * vr) * 2 + f
                want[base:base + 2 * vr:2] = src[axis, :, 2 * level + f]
    assert np.array_equal(vt, want)


def test_bf16_copy_rounds_to_nearest_even():
    """torch's fp32 -> bf16 (the shadows' reference) rounds to nearest, ties to even, in the bits."""
    bits = np.array([0x3F808000, 0x3F818000, 0x3F80C000, 0x3F807FFF, 0xBF818000, 0x00008000, 0x7F7FFFFF], np.uint32)
    x = bits.view(np.float32)
    got = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16)
    lsb = (bits >> 16) & 1
    want = ((bits + 0x7FFF + lsb) >> 16).astype(np.uint16)
    assert np.array_equal(got, want), (got, want)
