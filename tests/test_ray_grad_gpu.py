"""Gradients with respect to the rays on the H100: the view-direction gradient of the MLP backward
(hrf_field_backward_mlp_dirs), the per-ray reduction (hrf_ray_gradients), render() / forward() autograd against the
float64 oracle, the frozen-model route and the unchanged no-ray-gradient route.

Bars:
* direction gradient: entrywise, the rounding-faithful MLP reference's dCin deviation bound (columns 0..15, its
  accumulation bound included) propagated through |dSH/d(x,y,z)|, plus the fp32 evaluation of the Jacobian and of the
  16-term contraction (ray_grad_oracle.direction_grad_bound).
* reduction: n 2^-23 sum|terms| per entry against the float64 sum of the kernel's own inputs.
* end to end: the norm-wise 3e-2 bar of the other end-to-end gradient tests for the per-ray tensors and the background;
  4e-2 for the per-sample d(sample distances), the one tensor not summed over a ray (measured on an H100: 2.6e-2 with
  one segment, 3.5e-2 with three).  Both sides round the MLP activations to bf16, but the kernels also round the
  gradient tiles to bf16 where the oracle passes them straight through.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import mlp_oracle as M
import position_grad_oracle as P
import ray_grad_oracle as RG
from helpers import input_batch_of, make_pair, synthetic_rays
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _sms():
    out = (C.c_int * 3)()
    L.check(L.lib().hrf_device_info(out))
    return int(out[0])


# ------------------------------------------------------------------------------------------------ MLP backward, kernel
def _mlp_dirs_case(cuda, K, n, cap, d_rgb_on=True, seed=0):
    om, m, frames = make_pair((6,), seed=123, table_std=6.0, cam_emb=(2 if K == 48 else 0), device=cuda)
    nat = m.native()
    rng = np.random.default_rng(seed + K)
    pos = rng.uniform(-0.45, 0.45, (n, 3)).astype(np.float32)
    dd = rng.standard_normal((n, 3))
    dirs = (dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(np.float32)
    dirs[: min(n, 5)] = np.eye(3, dtype=np.float32)[np.arange(min(n, 5)) % 3]
    fr = rng.choice(np.asarray(frames), n).astype(np.int32)
    if n > 10:
        k = rng.choice(n, n // 50 + 1, replace=False)
        fr[k] = rng.choice(np.array([-3, 5000, frames[0] - 1], np.int32), len(k))   # no segment
    seg_ok = (fr >= frames[0]) & (fr <= frames[-1])
    cams = rng.integers(0, 12, n).astype(np.int32) if K == 48 else None
    feat = rng.standard_normal((n, 32)) * 0.5
    featb = M.bf16(feat)
    ds = (rng.standard_normal(n) * 1e-2).astype(np.float32)
    dr = rng.standard_normal((n, 3)).astype(np.float32)
    pad = lambda a: np.concatenate([a, np.zeros((cap - n,) + a.shape[1:], a.dtype)])   # noqa: E731
    dev = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(pad(a))).to(cuda, dt)   # noqa: E731
    count = torch.tensor([n], dtype=torch.int64, device=cuda)
    samples = nat.samples_rays(dev(pos), dev(dirs), dev(fr, torch.int32), torch.zeros(cap, device=cuda),
                               torch.arange(cap, device=cuda), ray_cameras=None if cams is None else dev(cams, torch.int32),
                               count_dev=count)
    feat_dev = dev(featb.astype(np.float32)).to(torch.bfloat16).contiguous()
    ds_dev, dr_dev = dev(ds), dev(dr)
    lib = L.lib()

    def run(dirs_out):
        ws = torch.full((cap * 40,), 7.0, device=cuda)
        d_mlp = torch.zeros(m.mlp_grad_elems, device=cuda)
        d_emb = torch.zeros((160, 2), device=cuda) if K == 48 else None
        args = (C.byref(nat.field), C.byref(samples), ds_dev.data_ptr(), dr_dev.data_ptr() if d_rgb_on else None, None,
                feat_dev.data_ptr(), None, d_mlp.data_ptr(), L.ptr(d_emb))
        if dirs_out is None:
            L.check(lib.hrf_field_backward_mlp(*args, ws.data_ptr(), L.stream()))
        else:
            L.check(lib.hrf_field_backward_mlp_dirs(*args, dirs_out.data_ptr(), ws.data_ptr(), L.stream()))
        torch.cuda.synchronize()
        return ws

    out = torch.full((cap, 3), 12345.0, device=cuda)
    ws_dirs = run(out)
    ws_plain = run(None)
    F = M.Forward(np.where(seg_ok[:, None], featb, 0.0), dirs,
                  (cams if cams is not None else np.full(n, -1)).astype(np.int64), None if K == 32 else
                  m.camera_embeddings.weight.detach().cpu().numpy(),
                  M.split_params(m.sigma_net.params.detach().cpu().numpy(), m.color_net.params.detach().cpu().numpy(), K),
                  m.density_scale, K)
    B = M.Backward(F, ds, dr if d_rgb_on else None, None, m.density_scale, 160 if K == 48 else 0)
    return out, ws_dirs, ws_plain, dirs, seg_ok, B


@pytest.mark.parametrize("size", ["1tile", "multi"])
@pytest.mark.parametrize("K", [32, 48])
def test_direction_grad_kernel_matches_rounding_faithful_reference(cuda, K, size):
    n = 128 if size == "1tile" else 3 * 2 * _sms() * 128 + 77
    cap = n + 200
    out, ws_dirs, ws_plain, dirs, seg_ok, B = _mlp_dirs_case(cuda, K, n, cap)
    got = out[:n].double().cpu().numpy()
    ref = RG.direction_grad(dirs, B.dcin[:, :16])
    bound = RG.direction_grad_bound(dirs, B.dcin[:, :16], B.dcin_dev[:, :16])
    err = np.abs(got - ref)
    ok = seg_ok
    ratio = (err[ok] / np.maximum(bound[ok], 1e-300)).max()
    print(f"K={K} {size}: n={n}, ambiguous {B.amb.mean():.3f}, max |kernel - ref| {err[ok].max():.3e}, "
          f"max |ref| {np.abs(ref).max():.3e}, max err / bound {ratio:.3e}")
    assert (err[ok] <= bound[ok]).all()
    assert (got[~ok] == 0).all() and (~ok).sum() > 0
    assert (out[n:] == 12345.0).all()                     # rows past the live count untouched
    assert torch.equal(ws_dirs[: 36 * cap], ws_plain[: 36 * cap])    # d(features) and positions: the plain kernel's
    assert np.abs(ref[ok]).max() > 0.1


def test_direction_grad_without_colour_gradient_is_zero(cuda):
    n = 300
    out, *_ = _mlp_dirs_case(cuda, 32, n, n + 10, d_rgb_on=False)
    assert (out[:n] == 0).all() and (out[n:] == 12345.0).all()


# ------------------------------------------------------------------------------------------------ per-ray reduction
def test_ray_gradients_kernel(cuda):
    rng = np.random.default_rng(9)
    counts = np.array([0, 1, 7, 0, 31, 32, 33, 300, 5000, 1, 0] + list(rng.integers(0, 200, 500)))
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    n, R = int(off[-1]), len(counts)
    dp = rng.standard_normal((n, 3)).astype(np.float32)
    dd = rng.standard_normal((n, 3)).astype(np.float32)
    t = rng.uniform(0.5, 3.0, n).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    dev = lambda a: torch.from_numpy(a).to(cuda)   # noqa: E731
    dpd, ddd, td, rdd, offd = dev(dp), dev(dd), dev(t), dev(rd), dev(off)

    def run(with_dirs=True):
        g_o = torch.full((R, 3), 99.0, device=cuda)
        g_d = torch.full((R, 3), 99.0, device=cuda)
        g_t = torch.full((n,), 99.0, device=cuda)
        L.check(L.lib().hrf_ray_gradients(dpd.data_ptr(), ddd.data_ptr() if with_dirs else None, td.data_ptr(),
                                          rdd.data_ptr(), offd.data_ptr(), R, g_o.data_ptr(), g_d.data_ptr(), g_t.data_ptr(),
                                          L.stream()))
        return g_o, g_d, g_t

    a = run()
    b = run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    d_o, d_d, d_t, S_o, S_d = RG.ray_gradients(dp, dd, t, rd, off)
    cnt = np.maximum(np.diff(off), 1)[:, None]
    go, gd, gt = (x.double().cpu().numpy() for x in a)
    assert (np.abs(go - d_o) <= 2 * cnt * 2.0 ** -23 * S_o).all()
    assert (np.abs(gd - d_d) <= 3 * cnt * 2.0 ** -23 * S_d).all()
    ri = np.repeat(np.arange(R), np.diff(off))
    St = (np.abs(dp.astype(np.float64) * rd[ri])).sum(1)
    assert (np.abs(gt - d_t) <= 3 * 2.0 ** -23 * St).all()
    assert (go[counts == 0] == 0).all() and (gd[counts == 0] == 0).all()
    _, gd2, _ = run(with_dirs=False)
    d_o2, d_d2, *_ = RG.ray_gradients(dp, None, t, rd, off)
    assert (np.abs(gd2.double().cpu().numpy() - d_d2) <= 3 * cnt * 2.0 ** -23 * S_d).all()


# ------------------------------------------------------------------------------------------------ render() end to end
def _ray_batch(cuda, frames, border_frames, n_rays=192, spr=48, seed=5):
    b = synthetic_rays(n_rays, spr, frames, seed=seed, ragged=True, step=4e-3)
    rng = np.random.default_rng(seed)
    b["frames"] = torch.from_numpy(rng.choice(np.asarray(border_frames), n_rays).astype(np.int32))
    return b


def _render_grads(m, b, cuda, bg_val=(0.2, 0.5, 0.7), seed=0, want=(True, True, True, True), params=True):
    from humanrf_b200.volume_rendering import render

    ib = input_batch_of(b, cuda)
    ib.unique_frame_numbers = torch.unique(ib.frame_numbers).view(-1, 1)
    ib.ray_origins.requires_grad_(want[0])
    ib.ray_directions.requires_grad_(want[1])
    ib.sample_distances.requires_grad_(want[2])
    bg = torch.tensor(bg_val, device=cuda, requires_grad=want[3])
    for q in m.hot_parameters():
        q.grad = None
    out = render(ib, m, bg, is_training=False)
    g = torch.Generator().manual_seed(seed)
    cc = torch.randn(out.color.shape, generator=g, dtype=torch.float64)
    cw = torch.randn(out.weights_sum.shape, generator=g, dtype=torch.float64)
    loss = (out.color * cc.float().to(cuda)).sum() + (out.weights_sum * cw.float().to(cuda)).sum()
    loss.backward()
    grads = [x.grad for x in (ib.ray_origins, ib.ray_directions, ib.sample_distances, bg)]
    return out, grads, cc.numpy(), cw.numpy(), ib


@pytest.mark.parametrize("segs", [(6,), (100, 100, 50)], ids=["seg6", "seg100x2-50"])
def test_render_ray_gradients_against_oracle(cuda, segs):
    om, m, frames = make_pair(segs, table_std=1.0, device=cuda)
    border = [frames[0], frames[-1]] + ([frames[0] + 99, frames[0] + 100, frames[0] + 199, frames[0] + 200]
                                        if len(segs) > 1 else [frames[2], frames[3]])
    b = _ray_batch(cuda, frames, border)
    out, (g_o, g_d, g_t, g_bg), cc, cw, _ = _render_grads(m, b, cuda)
    segs_ = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    o, d, t, ri = (b[k].numpy() for k in ("o", "d", "t", "ri"))
    ref = RG.render_oracle(om, segs_, f2s, f2t, o, d, t, ri, b["frames"].numpy(), o.shape[0], np.array([0.2, 0.5, 0.7]),
                           cc, cw)
    for name, got, r in zip(("origins", "directions", "distances", "background"), (g_o, g_d, g_t, g_bg), ref):
        got = got.double().cpu().numpy().reshape(r.shape)
        rel = np.linalg.norm(got - r) / np.linalg.norm(r)
        print(f"{segs} d({name}): norm-wise rel {rel:.3e}, |ref| {np.linalg.norm(r):.3e}")
        assert np.linalg.norm(r) > 0 and rel < (4e-2 if name == "distances" else 3e-2), name
    assert all(q.grad is not None for q in m.hot_parameters()[-2:])


def test_forward_direction_gradient_against_oracle(cuda):
    from humanrf_b200.scene_representation.query_io import QueryInput

    om, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    segs = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    rng = np.random.default_rng(11)
    n = 3000
    pos = rng.uniform(-0.48, 0.48, (n, 3)).astype(np.float32)
    fr = rng.choice(np.asarray(frames), n).astype(np.int32)
    dd = rng.standard_normal((n, 3))
    dirs = (dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(np.float32)
    cr = rng.standard_normal((n, 3))
    feats = P.features(segs, f2s, f2t, pos, fr)
    dref = torch.from_numpy(dirs).requires_grad_(True)
    _, geo = om.sigma_head(om._q(feats.float()))
    rgb = om.color_head(dref, geo)
    (ref,) = torch.autograd.grad((rgb.double() * torch.from_numpy(cr)).sum(), dref)
    d_dev = torch.from_numpy(dirs).to(cuda).requires_grad_(True)
    out = m.forward(QueryInput(is_training=False, positions=torch.from_numpy(pos).to(cuda), directions=d_dev,
                               frame_numbers=torch.from_numpy(fr).to(cuda)))
    (out.radiance * torch.from_numpy(cr).float().to(cuda)).sum().backward()
    got = d_dev.grad.double().cpu().numpy()
    rel = np.linalg.norm(got - ref.numpy()) / np.linalg.norm(ref.numpy())
    print(f"forward d(directions): norm-wise rel {rel:.3e}")
    assert rel < 3e-2
    # the density does not depend on the direction; a frozen model gives the same gradient, without parameter grads
    d2 = torch.from_numpy(dirs).to(cuda).requires_grad_(True)
    for q in m.hot_parameters():
        q.requires_grad_(False)
        q.grad = None
    out = m.forward(QueryInput(is_training=False, positions=torch.from_numpy(pos).to(cuda), directions=d2,
                               frame_numbers=torch.from_numpy(fr).to(cuda)))
    (out.radiance * torch.from_numpy(cr).float().to(cuda)).sum().backward()
    assert torch.equal(d2.grad, d_dev.grad) and all(q.grad is None for q in m.hot_parameters())


_PROFILER_WARM = []


def _kernel_names(fn):
    """CUDA kernel names launched by fn().  The first profiler session of a process pays CUPTI's start-up; one empty
    session is run first so that the captured one sees every launch."""
    from torch.profiler import ProfilerActivity, profile

    if not _PROFILER_WARM:
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.zeros(1, device="cuda").add_(1)
            torch.cuda.synchronize()
        _PROFILER_WARM.append(True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_frozen_model_ray_gradients(cuda):
    om, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    b = _ray_batch(cuda, frames, list(frames))
    _, ref, *_ = _render_grads(m, b, cuda)
    for q in m.hot_parameters():
        q.requires_grad_(False)
        q.grad = None
    # bit-identity outside any profiler session; the kernel list from a separate frozen run
    frozen = _render_grads(m, b, cuda)[1]
    for x, y in zip(frozen, ref):
        assert torch.equal(x, y)
    names = _kernel_names(lambda: _render_grads(m, b, cuda))
    assert any("field_backward_kernel" in s for s in names)
    assert any("position_grad" in s for s in names) and any("ray_gradients" in s for s in names)
    assert not any("scatter" in s for s in names), [s for s in names if "scatter" in s]
    assert all(q.grad is None for q in m.hot_parameters())


def test_nothing_changes_without_ray_gradients(cuda):
    from humanrf_b200.volume_rendering import _ray_arrays, render, render_fused

    om, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    # 16 rays of one sample each, far apart: one atomic add per gradient entry, so parameter gradients are reproducible
    g = np.linspace(-0.3, 0.3, 4, dtype=np.float32)
    x, y = np.meshgrid(g, g, indexing="ij")
    i = np.arange(16)
    z = (0.2 * ((i + i // 4) % 4) - 0.3).astype(np.float32)
    p = np.stack([x.reshape(-1), y.reshape(-1), z], 1)
    d = np.tile(np.array([[0.0, 0.6, 0.8]], np.float32), (16, 1))
    b = dict(o=torch.from_numpy(p - 0.5 * d), d=torch.from_numpy(d), t=torch.full((16,), 0.5), ri=torch.arange(16),
             frames=torch.full((16,), frames[1], dtype=torch.int32), cams=torch.zeros(16, dtype=torch.int32),
             rgba=torch.rand(16, 4))
    runs = []
    for want in [(False,) * 4, (False,) * 4, (True,) * 4]:
        out, grads, *_ = _render_grads(m, b, cuda, want=want)
        runs.append((out, grads, [q.grad.clone() for q in m.hot_parameters()]))
    (o0, g0, p0), (o1, _, p1), (o2, g2, p2) = runs
    assert all(torch.equal(a, c) for a, c in zip(p0, p1))        # the premise: one order of adds
    assert all(torch.equal(a, c) for a, c in zip(p0, p2))        # parameter gradients unchanged by the ray gradients
    assert torch.equal(o0.color, o2.color) and torch.equal(o0.weights_sum, o2.weights_sum)
    assert all(x is None for x in g0) and all(x is not None for x in g2)
    # the backward without ray gradients launches the kernels it always did
    out, *_ = _render_grads(m, b, cuda, want=(False,) * 4)
    ib = input_batch_of(b, cuda)
    names = _kernel_names(lambda: render(ib, m, torch.zeros(3, device=cuda), False).color.sum().backward())
    assert not any(("ray_gradients" in s or "position_grad" in s or "Lb1E" in s) for s in names), names
    assert any("field_backward_kernel" in s for s in names)
    # no gradients at all: one fused render, as before
    with torch.no_grad():
        a = _kernel_names(lambda: render(ib, m, torch.zeros(3, device=cuda), False))
        c = _kernel_names(lambda: render_fused(m, *_ray_arrays(ib), ib.num_rays, torch.zeros(3, device=cuda)))
    ours = lambda names: sorted(x for x in names if "hrf::" in x)     # noqa: E731  (torch's own fills aside)
    assert ours(a) == ours(c) and len(ours(a)) > 0
    # requires_grad set on the rays, but only the parameters asked for
    ib = input_batch_of(b, cuda)
    ib.ray_origins.requires_grad_(True)
    col = render(ib, m, torch.zeros(3, device=cuda), False).color.sum()
    torch.autograd.grad(col, [m.sigma_net.params])
    assert ib.ray_origins.grad is None


def test_batch_without_samples(cuda):
    """Every ray empty (all missed or pruned): the backward returns zeros for the rays, as the parameter-only route returns
    normally; forward() with no samples and directions that require grad, likewise."""
    from humanrf_b200.scene_representation.query_io import QueryInput

    om, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    R = 8
    d = torch.nn.functional.normalize(torch.randn(R, 3), dim=1)
    b = dict(o=torch.randn(R, 3), d=d, t=torch.zeros(0), ri=torch.zeros(0, dtype=torch.int64),
             frames=torch.full((R,), frames[0], dtype=torch.int32), cams=torch.zeros(R, dtype=torch.int32), rgba=torch.rand(R, 4))
    for params in (True, False):
        for q in m.hot_parameters():
            q.requires_grad_(params)
        out, (g_o, g_d, g_t, g_bg), *_ = _render_grads(m, b, cuda)
        assert out.color.shape == (R, 3) and (out.weights_sum == 0).all()
        assert (g_o == 0).all() and (g_d == 0).all() and g_t.numel() == 0 and torch.isfinite(g_bg).all()
    dq = torch.zeros((0, 3), device=cuda, requires_grad=True)
    pq = torch.zeros((0, 3), device=cuda, requires_grad=True)
    o = m.forward(QueryInput(is_training=False, positions=pq, directions=dq,
                             frame_numbers=torch.zeros(0, dtype=torch.int32, device=cuda)))
    (o.radiance.sum() + o.density.sum()).backward()
    assert dq.grad.shape == (0, 3) and pq.grad.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ camera refinement
def _sphere(G, r=0.42):
    c = (np.arange(G) + 0.5) / G - 0.5
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    return ((x * x + y * y + z * z <= r * r) * 255).astype(np.uint8)


def textured_teacher(cuda):
    """A static model whose geometry and texture both come from the field, inside a looser spherical hull: feature 0 of
    the dense level 0 of the xyz grid is +1 inside five blobs spread over the hull and -1 outside, so
    sigma = 100 e^{+-12} away from their surfaces; feature 1 is a sum of three low-frequency sinusoids, which the sigma
    net passes to the geometry features through a ReLU pair, and the colour net (its random initialisation) turns into a
    smooth texture.  The time vector is 1 for every feature; everything else is zero.  Blobs at different depths make a
    camera's orbit about the scene visible as parallax: with a single object a rotation and the lateral shift that keeps
    the object in place are nearly indistinguishable."""
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    torch.manual_seed(0)
    m = HumanRF(sorted_frame_numbers=tuple(range(15, 21)), segment_sizes=(6,), **MODEL_KW)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        fg = m.feature_grids[0]
        for gr in fg.grids():
            gr.zero_()
        lay = fg.layout
        res, off, scale = int(lay.res[0]), int(lay.offset[0]), float(lay.scale[0])
        i = torch.arange(res, dtype=torch.float64)
        c = (i - 0.5) / scale - 0.5                     # world coordinate of vertex i (tcnn: pos = scale * x + 0.5)
        zz, yy, xx = torch.meshgrid(c, c, c, indexing="ij")
        inside = torch.zeros_like(xx, dtype=torch.bool)
        for (cx, cy, cz), (rx, ry, rz) in (((0.0, 0.0, 0.0), (0.12, 0.16, 0.1)), ((0.24, 0.08, 0.1), (0.08, 0.1, 0.08)),
                                           ((-0.22, -0.1, 0.12), (0.1, 0.08, 0.08)), ((0.05, -0.15, -0.25), (0.09, 0.08, 0.1)),
                                           ((-0.1, 0.2, -0.2), (0.08, 0.08, 0.09))):
            inside |= ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 + ((zz - cz) / rz) ** 2 <= 1.0
        tex = sum(torch.sin(2 * np.pi * (a[0] * xx + a[1] * yy + a[2] * zz) + ph)
                  for a, ph in (((2.0, 1.0, 0.5), 0.3), ((-1.0, 2.5, 1.0), 1.1), ((0.5, -1.0, 3.0), 2.0)))
        iz, iy, ix = torch.meshgrid(torch.arange(res), torch.arange(res), torch.arange(res), indexing="ij")
        idx = (ix + iy * res + iz * res * res).reshape(-1)
        t = fg.grids()[0].view(-1, 2)
        t[off + idx, 0] = torch.where(inside.reshape(-1), 1.0, -1.0).float()
        t[off + idx, 1] = (tex.reshape(-1) / 3).float()
        fg.vectors.zero_()
        fg.vectors[3] = 1.0
        w1, w2 = torch.zeros(64, 32), torch.zeros(16, 64)
        w1[0, 0], w1[1, 0], w1[2, 1], w1[3, 1] = 1.0, -1.0, 1.0, -1.0
        w2[0, 0], w2[0, 1] = 12.0, -12.0
        w2[1:, 2:4] = torch.randn(15, 2, generator=g) * 2.0
        m.sigma_net.params.copy_(torch.cat((w1.reshape(-1), w2.reshape(-1))))
    for q in m.parameters():
        q.requires_grad_(False)
    return m.to(cuda)


class _RenderedDataset:
    """A SyntheticDataset with spherical hulls whose images are a model's own renders at the true poses (mask 1)."""

    def __init__(self, base, images):
        self.base, self.images = base, images
        self.cameras, self.frames = base.cameras, base.frames

    def get_aabb(self, frame_numbers=None):
        return self.base.get_aabb()

    def get_scaled_cameras(self, scene_offset, scene_scale):
        return self.base.get_scaled_cameras(scene_offset, scene_scale)

    def get_rgb(self, camera_number, frame_number, normalize=True):
        return self.images[(camera_number, frame_number)]

    def get_mask(self, camera_number, frame_number, normalize=True):
        c = self.cameras[camera_number]
        return np.ones((c.height, c.width, 1), np.float32)

    def get_occupancy_grid(self, frame_number):
        return self.base.get_occupancy_grid(frame_number)


def _scene():
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(width=256, height=192, G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    return ds


def _loader(ds):
    from humanrf_b200.dataset.data_loader import DataLoader as DL

    return DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192, camera_numbers=(0, 1, 2),
              frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])


def _centre_shift(cam_true, rot, trans, depth):
    """Pixel distance between the true camera's image centre and the reprojection, through the pose (rot, trans), of
    the point at `depth` along the true centre ray."""
    from humanrf_b200.dataset.cameras import projection_matrix_world2pixel, rotation_from_axisangle

    W, H = cam_true.width, cam_true.height
    X = cam_true.translation + depth * rotation_from_axisangle(cam_true.rotation_axisangle)[:, 2]
    w2p = projection_matrix_world2pixel(W, H, rot, trans, cam_true.focal_length, cam_true.principal_point)
    q = w2p @ np.append(X, 1.0)
    return float(np.hypot(q[0] / q[2] - W / 2, q[1] / q[2] - H / 2))


def _rot_err(a, b):
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.toolbox.camera_refinement import axisangle_of

    return float(np.linalg.norm(axisangle_of(rotation_from_axisangle(a) @ rotation_from_axisangle(b).T)))


def test_refine_camera(cuda):
    """A camera perturbed by a rotation and a translation of >= 1 pixel each at the image centre comes back to below 0.1x
    both initial errors; the run is deterministic; the unperturbed camera moves by at most 0.05 pixel."""
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.toolbox.camera_refinement import axisangle_of, refine_camera
    from humanrf_b200.toolbox.depth_maps import render_depth_map

    m = textured_teacher(cuda)
    base = _scene()
    cam_id, fr = 1, [16, 18]
    images = {}
    for f in fr:
        dm = render_depth_map(m, _loader(base), cam_id, f)
        images[(cam_id, f)] = dm.color.cpu().numpy()
        assert 0.05 < dm.alpha.mean().item() < 0.8
    cam = base.cameras[cam_id]
    depth = float(np.linalg.norm(cam.translation - base.aabb.mean(0)))
    R = rotation_from_axisangle(cam.rotation_axisangle)
    rot_p = axisangle_of(rotation_from_axisangle(0.015 * (R[:, 0] * 0.6 + R[:, 1] * 0.8)) @ R)
    tr = 0.04 * (R[:, 0] * 0.8 - R[:, 1] * 0.6) + 0.02 * R[:, 2]
    s_rot = _centre_shift(cam, rot_p, cam.translation, depth)
    s_tr = _centre_shift(cam, cam.rotation_axisangle, cam.translation + tr, depth)
    assert s_rot >= 1.0 and s_tr >= 1.0
    pert = _scene()
    pert.cameras[cam_id].rotation_axisangle = rot_p
    pert.cameras[cam_id].translation = cam.translation + tr
    loader_p = _loader(_RenderedDataset(pert, images))
    e_rot0, e_tr0 = _rot_err(rot_p, cam.rotation_axisangle), float(np.linalg.norm(tr))
    res = refine_camera(m, loader_p, cam_id, fr, seed=3)
    e_rot = _rot_err(res.rotation_axisangle, cam.rotation_axisangle)
    e_tr = float(np.linalg.norm(res.translation - cam.translation))
    print(f"perturbation {s_rot:.2f} px (rotation) / {s_tr:.2f} px (translation); rotation error {e_rot0:.3e} -> "
          f"{e_rot:.3e}, translation error {e_tr0:.3e} -> {e_tr:.3e}, loss {res.losses[0]:.3e} -> {res.losses[-1]:.3e}")
    assert e_rot < 0.1 * e_rot0 and e_tr < 0.1 * e_tr0
    again = refine_camera(m, loader_p, cam_id, fr, seed=3)
    assert np.array_equal(again.omega, res.omega) and np.array_equal(again.tau, res.tau) and again.losses == res.losses
    assert all(not q.requires_grad and q.grad is None for q in m.parameters())
    res0 = refine_camera(m, _loader(_RenderedDataset(base, images)), cam_id, fr, seed=4)
    shift = _centre_shift(cam, res0.rotation_axisangle, res0.translation, depth)
    print(f"unperturbed: centre shift {shift:.4f} px")
    assert shift <= 0.05
