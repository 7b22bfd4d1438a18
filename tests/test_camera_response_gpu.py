"""Per-camera colour response in the fused train step on the H100: the loss kernel (hrf_train_loss_response) against
tests/response_oracle.py and bit for bit against hrf_train_loss at identity, the per-camera sums, the error word, the
step (hrf_camera_response_step) against the float64 Adam oracle, hrf_camera_response_apply, FusedTrainer with
camera_responses, the state, and recovery of perturbed camera responses on a teacher scene.

Bars (u = 2^-24, fp32 unit roundoff), derived from the kernel's roundings:
* x = pred - gt: every rounded operation in fg, pred and gt adds at most u times its result, so
  |x - x64| <= e_x = 4u (|color| + |(1 - w) bg| + 2 |em fg| + |w b| + |rgb m| + |bg (1 - m)| + |pred|).  Rays with
  ||x| - delta| <= e_x may take the other Huber branch and are left out (counted: a handful at most).
* d_color = fl(fl(fl(h inv3r) scale) g) with h = x or +-delta: |err| <= (e_x [quad]) inv3r scale g + 4u |d_color|.
* d_wsum = the BCE term (its two quotients cancel where m = pc: 8u of the sum of their magnitudes) + sum_k dpred_k
  (em bg + b) (each product's operand error plus 4u of every term), + 2u of the result.
* per-camera sums: n 2^-23 sum|terms| (any fp32 summation order) plus the terms' own errors (e_dpred |fg| +
  |dpred| e_fg), times g for the gamma columns, plus 2u of the float64 -> float32 result.
* loss: one atomicAdd per 256 rays, fp32 tree sums: (R + 8) u sum|terms| plus the per-ray errors.
"""
import csv

import numpy as np
import pytest
import torch

import response_oracle as RO

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _batch(R, C_, rng, cams=None):
    color = rng.uniform(0, 1, (R, 3)).astype(np.float32)
    w = rng.choice([0.0, 1.0, 0.5, -1e-7, 1.0000001], R) if R else np.zeros(0)
    w = np.where(rng.uniform(0, 1, R) < 0.5, rng.uniform(0, 1, R), w).astype(np.float32)
    rgba = rng.uniform(0, 1, (R, 4)).astype(np.float32)
    rgba[:, 3] = rng.choice([0.0, 1.0, 0.5], R)
    bg = rng.uniform(0, 1, (R, 3)).astype(np.float32)
    # some rays close to their target (quadratic Huber branch), some exactly on it, -0 colours on a zero target
    near = rng.uniform(0, 1, R) < 0.5
    color[near] = (rgba[near, :3] * rgba[near, 3:] + bg[near] * (1 - rgba[near, 3:]) + rng.normal(0, 3e-3, (near.sum(), 3))).astype(np.float32)
    if R > 8:
        rgba[:4, :3], rgba[:4, 3] = color[:4], 1.0                      # x = +0
        color[4:6], rgba[4:6, :3], rgba[4:6, 3] = -0.0, 0.0, 1.0          # x = -0
        w[6:8], rgba[6:8, 3] = 0.5, 0.5                                 # BCE gradient -0
    if cams is None:
        cams = rng.integers(0, C_, R)
    return color, w, rgba, bg, np.asarray(cams, np.int32)


def _random_table(C_, rng, identity=()):
    params = np.concatenate((rng.uniform(-0.25, 0.25, (C_, 3)), rng.uniform(-0.06, 0.06, (C_, 3))), 1)
    params[list(identity)] = 0.0
    return params, RO.table_of(params)


def _loss_kernel(cuda, color, w, rgba, bg, cams, table, scale=None):
    from humanrf_b200 import _lib as L

    R, C_ = color.shape[0], table.shape[0]
    lib = L.lib()
    d = lambda a: _dev(a, cuda)   # noqa: E731
    ins = [d(color), d(w), d(rgba), d(bg), d(cams)]
    tab = d(table)
    sc = None if scale is None else torch.tensor([scale], dtype=torch.float32, device=cuda)
    d_color, d_wsum = torch.empty((R, 3), device=cuda), torch.empty(R, device=cuda)
    loss = torch.zeros(1, device=cuda)
    grad, count = torch.empty((C_, 6), device=cuda), torch.empty(C_, dtype=torch.int32, device=cuda)
    err = torch.zeros(1, dtype=torch.int32, device=cuda)
    ws = torch.empty(int(lib.hrf_train_loss_response_workspace_bytes(C_)), dtype=torch.uint8, device=cuda)
    p = lambda t: t.data_ptr() if R else None   # noqa: E731
    L.check(lib.hrf_train_loss_response(*(p(t) for t in ins[:4]), p(ins[4]), R, tab.data_ptr(), C_, 0.01, 1e-3,
                                        L.ptr(sc), p(d_color), p(d_wsum), loss.data_ptr(), grad.data_ptr(),
                                        count.data_ptr(), err.data_ptr(), ws.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    return {"d_color": d_color, "d_wsum": d_wsum, "loss": loss, "grad": grad, "count": count, "error": err}


def _train_loss(cuda, color, w, rgba, bg, scale=None):
    from humanrf_b200 import _lib as L

    R = color.shape[0]
    d = lambda a: _dev(a, cuda)   # noqa: E731
    ins = [d(color), d(w), d(rgba), d(bg)]
    sc = None if scale is None else torch.tensor([scale], dtype=torch.float32, device=cuda)
    d_color, d_wsum = torch.empty((R, 3), device=cuda), torch.empty(R, device=cuda)
    loss = torch.zeros(1, device=cuda)
    L.check(L.lib().hrf_train_loss(*(t.data_ptr() for t in ins), R, 0.01, 1e-3, L.ptr(sc), d_color.data_ptr(),
                                   d_wsum.data_ptr(), loss.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    return {"d_color": d_color, "d_wsum": d_wsum, "loss": loss}


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def _check_against_oracle(out, ref, color, w, rgba, bg, scale=1.0):
    R = color.shape[0]
    c64, w64, rgba64, bg64 = (a.astype(np.float64) for a in (color, w, rgba, bg))
    W_ = w64[:, None]
    m = rgba64[:, 3:]
    em, b, fg = ref["em"], ref["b"], ref["fg"]
    e_fg = 2 * U * (np.abs(c64) + np.abs((1 - W_) * bg64))
    e_x = 4 * U * (np.abs(c64) + np.abs((1 - W_) * bg64) + 2 * np.abs(em * fg) + np.abs(W_ * b)
                   + np.abs(rgba64[:, :3] * m) + np.abs(bg64 * (1 - m)) + np.abs(ref["pred"])) + np.abs(em) * e_fg
    ambiguous = np.abs(np.abs(ref["x"]) - 0.01) <= e_x
    assert ambiguous.sum() <= max(2, R // 1000), ambiguous.sum()
    ok = ~ambiguous.any(1)
    inv3r = 1.0 / (3 * R)
    quad = np.abs(ref["x"]) < 0.01
    g = 1.0 + em
    e_dpred = np.where(quad, e_x, 0.0) * inv3r * scale + 4 * U * np.abs(ref["dpred"])
    got = out["d_color"].double().cpu().numpy()
    bound = e_dpred * g + 4 * U * np.abs(ref["d_color"])
    assert (np.abs(got - ref["d_color"])[ok] <= bound[ok]).all(), \
        f"d_color err/bound {(np.abs(got - ref['d_color']) / np.maximum(bound, 1e-300))[ok].max():.3e}"
    resp = np.abs(em * bg64) + np.abs(b)
    pc, mm = np.clip(w64, 0, 1), m[:, 0]
    bce_terms = (np.abs(mm / (pc + 1e-10)) + np.abs((1 - mm) / (1 - pc + 1e-10))) / R * 1e-3 * scale
    bound_w = (8 * U * np.where(ref["dw_bce"] != 0, bce_terms, 0.0)
               + (e_dpred * resp + np.abs(ref["dpred"]) * 4 * U * resp).sum(1) + 2 * U * np.abs(ref["d_wsum"]))
    got_w = out["d_wsum"].double().cpu().numpy()
    assert (np.abs(got_w - ref["d_wsum"])[ok] <= bound_w[ok]).all(), \
        f"d_wsum err/bound {(np.abs(got_w - ref['d_wsum']) / np.maximum(bound_w, 1e-300))[ok].max():.3e}"
    terms = ref["huber"] * inv3r
    e_loss = ((R + 8) * U * (terms.sum() + (ref["bce"] / R * 1e-3).sum())
              + (np.where(quad, np.abs(ref["x"]), 0.01) * e_x).sum() * inv3r + 16 * U * (ref["bce"] / R * 1e-3).sum())
    assert abs(float(out["loss"][0]) - ref["loss"]) <= e_loss, (float(out["loss"][0]), ref["loss"], e_loss)
    return ok, e_dpred, e_fg


def _check_sums(out, ref, cams, e_dpred, e_fg, ok):
    C_ = ref["grad"].shape[0]
    cams = cams.astype(np.int64)
    valid = (cams >= 0) & (cams < C_)
    dpred, fg, W_ = ref["dpred"], ref["fg"], ref["w"][:, None]
    terms = np.concatenate((np.abs(dpred * fg), np.abs(dpred * W_)), 1)
    own = np.concatenate((e_dpred * np.abs(fg) + np.abs(dpred) * e_fg, e_dpred * np.abs(W_)), 1)
    n = ref["count"]
    s_terms, own_s = np.zeros((C_, 6)), np.zeros((C_, 6))
    np.add.at(s_terms, cams[valid], terms[valid])
    np.add.at(own_s, cams[valid], own[valid])
    bound = n[:, None] * 2 * U * s_terms + own_s
    bound[:, :3] *= ref["g"]
    bound += 2 * U * np.abs(ref["grad"])
    got = out["grad"].double().cpu().numpy()
    assert np.array_equal(out["count"].cpu().numpy(), n)
    err = np.abs(got - ref["grad"])
    amb = np.zeros(C_, bool)
    amb[np.unique(cams[valid & ~ok])] = True         # a ray that may take the other Huber branch: its camera is skipped
    assert (err[~amb] <= bound[~amb]).all(), f"sum err/bound {(err / np.maximum(bound, 1e-300))[~amb].max():.3e}"
    assert (got[n == 0] == 0).all()


@pytest.mark.parametrize("C_", [1, 2, 160, 1024])
@pytest.mark.parametrize("R", [1, 255, 4099, 300001])
def test_loss_kernel_matches_oracle(cuda, R, C_):
    rng = np.random.default_rng(R * 3 + C_)
    color, w, rgba, bg, cams = _batch(R, C_, rng)
    params, table = _random_table(C_, rng, identity=(0,) if C_ > 1 else ())
    scale = 1.37
    out = _loss_kernel(cuda, color, w, rgba, bg, cams, table, scale)
    again = _loss_kernel(cuda, color, w, rgba, bg, cams, table, scale)
    for k in ("d_color", "d_wsum", "grad", "count"):
        assert np.array_equal(_bits(out[k]), _bits(again[k])), k              # two runs, identical bytes
    assert int(out["error"][0]) == 0
    ref = RO.loss_and_grads(color, w, rgba, bg, cams, table, scale=scale)
    ok, e_dpred, e_fg = _check_against_oracle(out, ref, color, w, rgba, bg, scale)
    _check_sums(out, ref, cams, e_dpred, e_fg, ok)


def _lane_cams(R, C_):
    """Every camera in every lane position of a 32-ray tile: camera (r + r // 32) mod C."""
    r = np.arange(R)
    return ((r + r // 32) % C_).astype(np.int32)


@pytest.mark.parametrize("C_", [1, 2, 160, 1024])
@pytest.mark.parametrize("R", [0, 1, 31, 256, 257, 5000, 70001])
def test_identity_writes_train_loss_bytes(cuda, R, C_):
    rng = np.random.default_rng(R + 17 * C_)
    table = np.zeros((C_, 6), np.float32)
    layouts = [rng.integers(0, C_, R), np.full(R, C_ - 1), _lane_cams(max(R, 32 * C_ + 5), C_)[:R]]
    if R >= 32 * C_:
        layouts.append(_lane_cams(R, C_))
    for cams in layouts:
        color, w, rgba, bg, cams = _batch(R, C_, rng, cams)
        for scale in (None, 0.75):
            got = _loss_kernel(cuda, color, w, rgba, bg, cams, table, scale)
            if R == 0:            # hrf_train_loss takes no empty batch: the record holds zero sums and counts
                assert float(got["grad"].abs().sum()) == 0 and int(got["count"].abs().sum()) == 0
                assert float(got["loss"][0]) == 0 and int(got["error"][0]) == 0
                continue
            want = _train_loss(cuda, color, w, rgba, bg, scale)
            assert np.array_equal(_bits(got["d_color"]), _bits(want["d_color"]))
            assert np.array_equal(_bits(got["d_wsum"]), _bits(want["d_wsum"]))
            if R <= 256:          # one addend: the same bytes; more: the same addends in the atomics' order
                assert np.array_equal(_bits(got["loss"]), _bits(want["loss"]))
            else:
                assert abs(float(got["loss"][0]) - float(want["loss"][0])) <= 64 * U * abs(float(want["loss"][0]))
            assert int(got["count"].sum()) == R and int(got["error"][0]) == 0
    if R > 8:
        assert (np.signbit(got["d_color"].cpu().numpy()) & (got["d_color"].cpu().numpy() == 0)).any()   # -0 covered
        assert (np.signbit(got["d_wsum"].cpu().numpy()) & (got["d_wsum"].cpu().numpy() == 0)).any()


def test_one_camera_owns_every_ray(cuda):
    rng = np.random.default_rng(5)
    R, C_ = 300000, 8
    color, w, rgba, bg, cams = _batch(R, C_, rng, np.full(R, 5))
    params, table = _random_table(C_, rng)
    out = _loss_kernel(cuda, color, w, rgba, bg, cams, table)
    ref = RO.loss_and_grads(color, w, rgba, bg, cams, table)
    ok, e_dpred, e_fg = _check_against_oracle(out, ref, color, w, rgba, bg)
    _check_sums(out, ref, cams, e_dpred, e_fg, ok)
    assert int(out["count"][5]) == R and float(out["grad"][torch.arange(C_) != 5].abs().sum()) == 0.0


def _fake_loader(cuda, C_):
    from types import SimpleNamespace

    return SimpleNamespace(all_inverse_krs=torch.zeros((C_, 3, 3), device=cuda), camera_numbers=tuple(range(C_)))


def test_bad_camera_sets_error_and_step_writes_nothing(cuda):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    rng = np.random.default_rng(2)
    C_, R = 8, 5000
    for bad in (8, -2):
        color, w, rgba, bg, cams = _batch(R, C_, rng)
        cams[1234] = bad
        params, table = _random_table(C_, rng)
        out = _loss_kernel(cuda, color, w, rgba, bg, cams, table)
        assert int(out["error"][0]) == 1
        ref = RO.loss_and_grads(color, w, rgba, bg, cams, table)          # the bad ray: identity, out of the sums
        assert np.array_equal(out["count"].cpu().numpy(), ref["count"]) and int(out["count"].sum()) == R - 1
        ok, _, _ = _check_against_oracle(out, ref, color, w, rgba, bg)       # the bad ray's d_color: the identity's
        assert ok[1234] and np.array_equal(ref["pred"][1234], color[1234].astype(np.float64))
    resp = CameraResponses(_fake_loader(cuda, C_), fixed_cameras=())
    d = lambda a: _dev(a, cuda)   # noqa: E731
    color, w, rgba, bg, cams = _batch(R, C_, rng)
    cams[7] = 11
    dc, dw, loss = torch.empty((R, 3), device=cuda), torch.empty(R, device=cuda), torch.zeros(1, device=cuda)
    resp.loss(d(color), d(w), d(rgba), d(bg), d(cams), R, 0.01, 1e-3, None, dc, dw, loss)
    before = [t.clone() for t in (resp.params, resp.exp_avg, resp.exp_avg_sq, resp.steps, resp.table)]
    resp.step(0)
    torch.cuda.synchronize()
    for a, b in zip(before, (resp.params, resp.exp_avg, resp.exp_avg_sq, resp.steps, resp.table)):
        assert torch.equal(a, b)
    with pytest.raises(RuntimeError, match="outside"):
        resp.check()
    with pytest.raises(RuntimeError, match="outside"):
        resp.state_dict()


def test_step_matches_adam_oracle(cuda):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    C_, lr = 8, 3e-3
    resp = CameraResponses(_fake_loader(cuda, C_), lr=lr, final_lr_ratio=1.0, fixed_cameras=(0,))
    st = {"params": np.zeros((C_, 6)), "m": np.zeros((C_, 6)), "v": np.zeros((C_, 6)), "steps": np.zeros(C_, np.int64)}
    fixed = np.zeros(C_, bool)
    fixed[0] = True
    rng = np.random.default_rng(4)
    for k, touched in enumerate([[0, 1, 2, 3], [2, 3, 6], [1, 2, 3, 4, 6], [6], [0, 2, 3, 6]]):
        count = np.zeros(C_, np.int32)
        count[touched] = rng.integers(1, 1000, len(touched))
        g = (rng.standard_normal((C_, 6)) * 10.0 ** rng.uniform(-6, -1, (C_, 1))).astype(np.float32)
        g[3] = 0.0                    # camera 3 has rays but a zero gradient: Adam leaves it at identity
        resp.response_grad.copy_(torch.from_numpy(g))
        resp.ray_count.copy_(torch.from_numpy(count))
        before = {n: getattr(resp, n).clone() for n in ("params", "exp_avg", "exp_avg_sq", "steps", "table")}
        resp.step(k)
        torch.cuda.synchronize()
        RO.adam(st, g.astype(np.float64), count, fixed, lr)
        for c in range(C_):
            if c in touched and c != 0:
                continue
            for n, v in before.items():                           # untouched and fixed: bit-unchanged
                assert torch.equal(getattr(resp, n)[c], v[c]), (k, c, n)
    got = resp.params.cpu().numpy()
    assert np.allclose(got, st["params"], rtol=1e-12, atol=1e-18)
    assert np.allclose(resp.exp_avg.cpu().numpy(), st["m"], rtol=1e-12, atol=1e-30)
    assert np.allclose(resp.exp_avg_sq.cpu().numpy(), st["v"], rtol=1e-12, atol=1e-30)
    assert np.array_equal(resp.steps.cpu().numpy(), st["steps"])
    tab, want = resp.table.cpu().numpy(), RO.table_of(got)
    assert (np.abs(tab.astype(np.float64) - want) <= np.spacing(np.abs(want))).all()
    assert (tab[0] == 0).all() and (tab[3] == 0).all() and (tab[5] == 0).all() and (tab[7] == 0).all()
    assert (tab[[1, 2, 4, 6]] != 0).all()


def test_apply_matches_oracle_and_identity_is_bit_exact(cuda):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    rng = np.random.default_rng(9)
    C_, P = 5, 123457
    resp = CameraResponses(_fake_loader(cuda, C_))
    params, _ = _random_table(C_, rng, identity=(0, 3))
    resp.load_state_dict({"params": torch.from_numpy(params), "exp_avg": torch.zeros(C_, 6, dtype=torch.float64),
                          "exp_avg_sq": torch.zeros(C_, 6, dtype=torch.float64),
                          "steps": torch.zeros(C_, dtype=torch.int32), "fixed_cameras": [0]})
    color = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    color[:5] = -0.0
    alpha = rng.uniform(0, 1, P).astype(np.float32)
    alpha[:1000] = rng.choice([0.0, 1.0], 1000)
    for c in range(C_):
        for bg in (None, (0.2, 0.7, 1.0)):
            out = resp.apply(_dev(color, cuda), _dev(alpha, cuda), c, bg)
            if c in (0, 3):
                assert np.array_equal(_bits(out), color.view(np.int32))
                continue
            want = RO.apply(color, alpha, np.zeros(3) if bg is None else bg, resp.table[c].cpu().numpy())
            got = out.double().cpu().numpy()
            e = 8 * U * (np.abs(color) + 2 * np.abs(want) + 1.0)
            assert (np.abs(got - want) <= e).all()


# ------------------------------------------------------------------------------------------------ trainer
def _child_kernel_names():
    from test_camera_poses_gpu import _kernel_names
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.training import FusedTrainer

    cuda = torch.device("cuda:0")
    R = 4096
    b = synthetic_rays(R, 32, list(range(15, 21)), seed=4)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba", "cams")}
    cams = (g["cams"] % 8).contiguous()

    def names(resp):
        m, _ = make_model((6,), seed=1, device=cuda)
        tr = FusedTrainer(m, camera_responses=resp)
        for _ in range(2):
            tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams)
        return _kernel_names(lambda: tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams))

    return {"plain": names(None), "late": names(CameraResponses(_fake_loader(cuda, 8), start_step=1000)),
            "early": names(CameraResponses(_fake_loader(cuda, 8)))}


def test_default_step_unchanged(cuda):
    import json
    import subprocess
    import sys
    from pathlib import Path

    from test_camera_poses_gpu import DEFAULT_STEP_KERNELS

    here = Path(__file__).resolve().parent
    code = (f"import json, sys; sys.path[:0] = [{str(here)!r}, {str(here.parent)!r}]; import {Path(__file__).stem} as T; "
            "print('RESULT ' + json.dumps(T._child_kernel_names()))")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600,
                       cwd=str(here.parent))
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(lines[-1][len("RESULT "):])
    ours = lambda names: [n for n in names if "hrf::" in n]   # noqa: E731
    assert ours(res["plain"]) == DEFAULT_STEP_KERNELS
    assert ours(res["late"]) == DEFAULT_STEP_KERNELS
    early = ours(res["early"])
    assert not any("train_loss_kernel" in n for n in early)
    swapped = [n for n in early if "response" not in n]
    assert swapped == [n for n in DEFAULT_STEP_KERNELS if "train_loss_kernel" not in n]
    assert [n.split("(")[0] for n in early if "response" in n] == \
        ["hrf::response_loss_kernel", "hrf::response_finish_kernel", "hrf::response_step_kernel"]


def _train(cuda, resp_kw, steps, capture=None):
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.training import FusedTrainer

    R = 4096
    b = synthetic_rays(R, 32, list(range(15, 21)), seed=4)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba", "cams")}
    cams = (g["cams"] % 8).contiguous()
    m, _ = make_model((6,), seed=1, device=cuda)
    resp = None if resp_kw is None else CameraResponses(_fake_loader(cuda, 8), **resp_kw)
    if capture is not None:
        orig = resp.loss

        def loss(*a, **k):
            table = resp.table.clone()                  # enqueued before the loss kernel: the table it reads
            n = orig(*a, **k)
            torch.cuda.synchronize()
            capture.append(([x.clone() if isinstance(x, torch.Tensor) else x for x in a], table))
            return n
        resp.loss = loss
    tr = FusedTrainer(m, camera_responses=resp)
    losses = [tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams, return_loss=True)
              for _ in range(steps)]
    return tr, resp, losses


def test_frozen_responses_give_the_backward_train_loss_bytes(cuda):
    """With lr = 0 the table stays at identity: every step's loss kernel writes hrf_train_loss's d_color and d_wsum bytes
    on that step's own buffers, so the backward gets the gradient it gets without responses, and the rest of the step
    runs the default step's kernels (test_default_step_unchanged).  The field itself cannot be compared bit for bit with
    a run without responses: the backward sums with fp32 atomics, so two runs of the same default step already differ
    after the first update (test_training_gpu), and Adam turns a last-bit difference of a near-zero gradient into a
    full step; the loss value itself is summed with atomics too."""
    from humanrf_b200 import _lib as L

    cap = []
    got, resp, _ = _train(cuda, {"lr": 0.0, "fixed_cameras": ()}, 4, capture=cap)
    assert len(cap) == 4
    for (color, wsum, rgba, bg, cams, R, delta, bce_w, scale, d_color, d_wsum, loss), table in cap:
        assert float(table.abs().sum()) == 0.0
        dc, dw, lo = torch.empty_like(d_color), torch.empty_like(d_wsum), torch.zeros(1, device=cuda)
        L.check(L.lib().hrf_train_loss(color.data_ptr(), wsum.data_ptr(), rgba.data_ptr(), bg.data_ptr(), R, delta,
                                       bce_w, L.ptr(scale), dc.data_ptr(), dw.data_ptr(), lo.data_ptr(), L.stream()))
        torch.cuda.synchronize()
        assert np.array_equal(_bits(dc), _bits(d_color)) and np.array_equal(_bits(dw), _bits(d_wsum))
    assert int(resp.steps.min()) == 4 and float(resp.params.abs().sum()) == 0.0


def test_train_step_loss_matches_oracle(cuda):
    cap = []
    tr, resp, losses = _train(cuda, {"lr": 5e-2}, 3, capture=cap)
    assert float(resp.table.abs().sum()) > 0
    # the last step's own buffers and the table its loss kernel read
    (color, wsum, rgba, bg, cams, R, delta, bce_w, scale, d_color, d_wsum, loss), table = cap[-1]
    assert scale is None and float(table.abs().sum()) > 0
    c_np = [t.cpu().numpy() for t in (color, wsum.view(-1), rgba, bg, cams)]
    ref = RO.loss_and_grads(*c_np, table.cpu().numpy(), delta, bce_w)
    assert float(loss[0]) == losses[-1]
    _check_against_oracle({"d_color": d_color, "d_wsum": d_wsum, "loss": loss}, ref, *c_np[:4])


def test_state_round_trip_and_csv(cuda, tmp_path):
    from humanrf_b200.toolbox.camera_response import RESPONSE_COLUMNS, CameraResponses

    tr, resp, _ = _train(cuda, {"lr": 5e-2}, 3)
    st = resp.state_dict()
    other = CameraResponses(_fake_loader(cuda, 8))
    other.load_state_dict(st)
    for n in ("params", "exp_avg", "exp_avg_sq", "steps", "table"):
        assert torch.equal(getattr(resp, n), getattr(other, n)), n
    assert other.fixed_cameras == resp.fixed_cameras
    path = tmp_path / "response.csv"
    resp.write_response_csv(path)
    rows = list(csv.reader(open(path)))
    assert tuple(rows[0]) == RESPONSE_COLUMNS and len(rows) == 9
    vals = np.array([[float(x) for x in r[1:]] for r in rows[1:]])
    assert np.array_equal(vals[:, :3], resp.gains().cpu().numpy()) and np.array_equal(vals[:, 3:], resp.offsets().cpu().numpy())
    assert (vals[0] == [1, 1, 1, 0, 0, 0]).all()


# ------------------------------------------------------------------------------------------------ recovery
def _masked_psnr(pred, gt, mask):
    m = mask.reshape(-1).astype(bool)
    err = ((pred.reshape(-1, 3)[m] - gt.reshape(-1, 3)[m]) ** 2).mean()
    return float(10 * np.log10(1.0 / max(err, 1e-20)))


def test_joint_training_recovers_camera_responses(cuda):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.training import FusedTrainer
    from test_camera_poses_gpu import _scene8, _TeacherDataset
    from test_ray_grad_gpu import textured_teacher

    base = _scene8()
    frame, n_cams = 16, 8
    view = DL(dataset=base, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192,
              camera_numbers=tuple(range(n_cams)), frame_numbers=tuple(base.frames), max_buffer_size=1,
              render_sequence=[(0, frame)])
    teacher = textured_teacher(cuda)
    rng = np.random.default_rng(7)
    perturbed = (1, 2, 4, 5, 7)
    true = np.zeros((n_cams, 6))
    for c in perturbed:
        true[c, :3] = np.log(rng.uniform(0.8, 1.25, 3))
        true[c, 3:] = rng.uniform(-0.05, 0.05, 3)
    images, masks, fgs = {}, {}, {}
    for c in range(n_cams):
        dm = render_depth_map(teacher, view, c, frame)
        col, a = dm.color.double().cpu().numpy(), dm.alpha.double().cpu().numpy()[..., None]
        images[(c, frame)] = (np.exp(true[c, :3]) * col + a * true[c, 3:]).astype(np.float32)       # g fg + alpha b
        masks[(c, frame)] = (a > 0.5).astype(np.float32)
        fgs[c] = (col[a[..., 0] > 0.5], a[a[..., 0] > 0.5])
    psnr = {}
    for use in (False, True):
        m = textured_teacher(cuda)
        torch.manual_seed(0)
        np.random.seed(0)
        loader = DL(dataset=_TeacherDataset(base, images, masks), device="cuda", mode=DL.Mode.TRAINING,
                    dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                    space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=BATCH,
                    camera_numbers=tuple(range(n_cams)), frame_numbers=(frame,), max_buffer_size=n_cams,
                    max_num_frames_per_batch=1, use_mask=True, filter_light_bloom=False)
        for q in m.parameters():
            q.requires_grad_(True)
        resp = CameraResponses(loader, lr=RESPONSE_LR, final_lr_ratio=1e-2, max_steps=STEPS) if use else None
        if use:
            assert resp.fixed_cameras == (0,)
        trainer = FusedTrainer(m, lr=FIELD_LR, max_steps=STEPS, camera_responses=resp)
        for _ in range(STEPS):
            ib = next(loader)
            trainer.step(ib.ray_origins.contiguous(), ib.ray_directions.contiguous(),
                         ib.frame_numbers.view(-1).contiguous(), ib.sample_distances.view(-1).contiguous(),
                         ib.ray_indices.contiguous(), ib.rgba.contiguous(), ib.num_rays,
                         cameras=ib.camera_numbers.view(-1).to(torch.int32).contiguous())
        scores = []
        for c in range(n_cams):
            dm = render_depth_map(m, view, c, frame)
            color = dm.color.contiguous()
            if use:
                resp.apply(color, dm.alpha.contiguous(), c)
            scores.append(_masked_psnr(color.cpu().numpy(), images[(c, frame)], masks[(c, frame)]))
        psnr[use] = scores
        if use:
            resp.check()
            est = resp.params.cpu().numpy()
    print("masked PSNR of the training views, without / with responses: "
          f"{np.mean(psnr[False]):.2f} / {np.mean(psnr[True]):.2f} dB")
    for c in range(n_cams):
        print(f"camera {c}: PSNR {psnr[False][c]:.2f} -> {psnr[True][c]:.2f} dB")
    ok = bool((est[0] == 0).all())
    for c in range(1, n_cams):
        # A gain and an offset are told apart only through the spread of the camera's foreground colours in that
        # channel, so the error is measured where the response acts: the RMS over the camera's masked pixels of the
        # colour the learnt response adds minus the colour the true one adds, (g' - g) fg + alpha (b' - b).
        fg, a = fgs[c]
        dg, db = np.exp(est[c, :3]) - np.exp(true[c, :3]), est[c, 3:] - true[c, 3:]
        e = float(np.sqrt(((dg * fg + a * db) ** 2).mean()))
        e0 = float(np.sqrt((((np.exp(true[c, :3]) - 1) * fg + a * true[c, 3:]) ** 2).mean()))
        print(f"camera {c}: true gain {np.exp(true[c, :3]).round(4)} offset {true[c, 3:].round(4)}; learnt gain "
              f"{np.exp(est[c, :3]).round(4)} offset {est[c, 3:].round(4)}; colour error {e0:.4f} -> {e:.4f}")
        ok &= e < 0.25 * e0 if c in perturbed else e < IDENTITY_TOL
    assert ok


STEPS, BATCH, RESPONSE_LR, FIELD_LR, IDENTITY_TOL = 2000, 32768, 5e-3, 3e-5, 0.01


def test_evaluate_sequence_scores_through_the_learnt_response(cuda, tmp_path):
    """evaluate_sequence(camera_responses=...): a view whose camera has a learnt response is scored on the render with
    that response applied (alpha of the render, background 0); a camera at identity is scored as without responses."""
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.toolbox.evaluation import evaluate_sequence, quantize
    from test_evaluation_gpu import _loader, confined_teacher

    m = confined_teacher(cuda)
    ds, dl = _loader(cuda)
    resp = CameraResponses(dl)
    n = resp.num_cameras
    params = torch.zeros((n, 6), dtype=torch.float64)
    params[1] = torch.tensor([0.1, -0.05, 0.02, 0.03, -0.02, 0.01], dtype=torch.float64)
    resp.load_state_dict({"params": params, "exp_avg": torch.zeros(n, 6, dtype=torch.float64),
                          "exp_avg_sq": torch.zeros(n, 6, dtype=torch.float64), "steps": torch.zeros(n, dtype=torch.int32),
                          "fixed_cameras": [0]})
    pairs = [(0, 15), (1, 16)]
    plain = evaluate_sequence(m, dl, pairs, tmp_path / "plain", save_frames=False)
    got = evaluate_sequence(m, dl, pairs, tmp_path / "resp", save_frames=False, camera_responses=resp)
    assert (got[0].psnr, got[0].ssim) == (plain[0].psnr, plain[0].ssim)
    assert got[1].psnr != plain[1].psnr
    # the same score as image_metrics on the applied render
    from humanrf_b200.toolbox.evaluation import ground_truth, image_metrics

    dm = render_depth_map(m, dl, 1, 16)
    pred = quantize(resp.apply(dm.color.contiguous().clone(), dm.alpha.contiguous(), 1))
    gt, mask = ground_truth(dl, 1, 16)
    vals, _ = image_metrics(pred, torch.from_numpy(gt).to(cuda), torch.from_numpy(mask).to(cuda))
    assert abs(float(vals[0]) - got[1].psnr) <= 1e-9 * abs(got[1].psnr)
