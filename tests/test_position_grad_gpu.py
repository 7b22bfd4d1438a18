"""hrf_field_position_grad on the H100 (csrc/position_grad.cu) and position gradients through HumanRF autograd, against
the float64 reference tests/position_grad_oracle.py.

Bars:
* kernel: |d_positions - J^T dF| <= 64 * 2^-23 * S per component, S = the sum of |every product term| (bound_terms), with
  the dF the MLP backward wrote read back from the workspace.  The reference uses the kernel's float32 cell offsets, so
  what remains is fp32 accumulation: 8 corners, 4 grids, 2 features, 16 levels, a chain well under 64 operations.
* affine teachers: trilinear interpolation reproduces an affine function, so the gradient is exactly parallel to the
  spatial part of the affine coefficients; its perpendicular part is bounded by the same accumulation bound.
* autograd: the norm-wise 3e-2 bar of the other end-to-end gradient tests, against the oracle MLP's d(features)
  contracted with the float64 Jacobian.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import position_grad_oracle as P
from helpers import make_pair
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu

ACC = 64 * 2.0 ** -23


def _batch(rng, n, frames, f2s):
    """Positions in the cube, on its faces and just outside it; frames on both sides of every segment border, and
    frames that map to no segment (row 0 of the result)."""
    pos = rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)
    k = rng.choice(n, n // 10, replace=False)
    edge = np.array([-0.5, 0.5, -0.5 - 1e-3, 0.5 + 1e-3, 0.52, -0.53], np.float32)
    pos[k, rng.integers(0, 3, len(k))] = rng.choice(edge, len(k))
    fr = rng.choice(np.asarray(frames), n).astype(np.int32)
    seg = f2s[np.asarray(frames)]
    borders = [f for a, f in zip(frames, frames[1:]) if seg[f - frames[0]] != seg[a - frames[0]]]
    special = [frames[0], frames[-1]] + [b for f in borders for b in (f - 1, f)] + [frames[0] - 1, -3, 5000]
    j = rng.choice(n, 4 * len(special), replace=False)
    fr[j] = np.repeat(np.asarray(special, np.int32), 4)
    return pos, fr


def _workspace_dF(ws, n_cap, n):
    w = ws[: 32 * n_cap].view(16, n_cap, 2)[:, :n]
    return w.permute(1, 0, 2).reshape(n, 32).double().cpu()


def _run(m, pos, fr, form, cuda, capacity=None, seed=0):
    """Backward MLP with random upstream gradients, then the position kernel: (d_pos, dF, pos4, kernel call)."""
    nat = m.native()
    n = pos.shape[0]
    cap = capacity or n
    g = torch.Generator().manual_seed(seed)
    pad = lambda a: np.concatenate([a, np.zeros((cap - n,) + a.shape[1:], a.dtype)]) if cap > n else a
    count = torch.tensor([n], dtype=torch.int64, device=cuda) if cap > n else None
    if form == "query":
        p_dev = torch.from_numpy(pad(pos)).to(cuda)
        d = torch.nn.functional.normalize(torch.randn(cap, 3, generator=g), dim=1).to(cuda)
        samples = nat.samples_query(p_dev, d, torch.from_numpy(pad(fr)).to(cuda))
        if count is not None:
            samples.num_samples_dev = count.data_ptr()
            samples._count = count
        pos32 = pos
    else:
        # one sample per ray at a nonzero distance: p = o + t d, mul then add in fp32, as the kernels compute it
        d = torch.nn.functional.normalize(torch.randn(cap, 3, generator=g), dim=1).numpy().astype(np.float32)
        t = np.float32(0.25) + np.zeros(cap, np.float32)
        o = (pad(pos) - t[:, None] * d).astype(np.float32)
        pos32 = (o + (t[:, None] * d).astype(np.float32)).astype(np.float32)[:n]
        dev = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        samples = nat.samples_rays(dev(o), dev(d), dev(pad(fr)), dev(t), torch.arange(cap, device=cuda),
                                   count_dev=count)
    ds = torch.randn(cap, generator=g).to(cuda)
    dr = torch.randn(cap, 3, generator=g).to(cuda)
    ws = torch.empty(cap * 40, dtype=torch.float32, device=cuda)
    d_mlp = torch.zeros(m.mlp_grad_elems, dtype=torch.float32, device=cuda)
    lib = L.lib()
    L.check(lib.hrf_field_backward_mlp(C.byref(nat.field), C.byref(samples), ds.data_ptr(), dr.data_ptr(), None, None, None,
                                       d_mlp.data_ptr(), None, ws.data_ptr(), L.stream()))

    def call(out):
        L.check(lib.hrf_field_position_grad(C.byref(nat.field), C.byref(samples), ws.data_ptr(), out.data_ptr(), L.stream()))
        return out

    out = call(torch.full((cap, 3), 12345.0, device=cuda))
    torch.cuda.synchronize()
    pos4 = ws[32 * cap:36 * cap].view(cap, 4)[:n].cpu().numpy()
    return out, _workspace_dF(ws, cap, n), pos4, pos32, call


@pytest.mark.parametrize("segs", [(50,), (100, 100, 50)], ids=["seg50-log2T18", "seg100x2-50-log2T19"])
@pytest.mark.parametrize("form", ["query", "rays"])
def test_kernel_matches_float64_jacobian(cuda, segs, form):
    _, m, frames = make_pair(segs, table_std=2.0, device=cuda)
    S_ = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    assert {int(np.log2(s.size[15])) for s in S_} == ({18} if segs == (50,) else {18, 19})
    assert any(not s.hashed[1] and s.size[1] & (s.size[1] - 1) for s in S_)     # a dense non-power-of-two level
    rng = np.random.default_rng(len(segs) * 7 + (form == "rays"))
    n = 20000
    pos, fr = _batch(rng, n, frames, f2s)
    cap = n + 333
    out, dF, pos4, pos32, call = _run(m, pos, fr, form, cuda, capacity=cap)
    u32, seg = P._normalised(pos32, fr, f2s, f2t)
    ok = seg >= 0
    assert np.array_equal(pos4[:, :3].view(np.int32), u32[:, :3].view(np.int32))
    got = out[:n].double().cpu()
    ref = P.position_grad(S_, f2s, f2t, pos32, fr, dF)
    S = P.bound_terms(S_, f2s, f2t, pos32, fr, dF)
    err = (got - ref).abs()
    ratio = (err / (ACC * S).clamp(min=1e-300)).max().item()
    print(f"{segs} {form}: max |kernel - ref| {err.max():.3e}, max |ref| {ref.abs().max():.3e}, max err / bound {ratio:.3e}")
    assert (err <= ACC * S).all()
    assert (got[~torch.from_numpy(ok)] == 0).all() and ok.sum() < n and ref.abs().max() > 1.0
    # rows past the live count are untouched; a second run writes identical bytes
    assert (out[n:] == 12345.0).all()
    again = call(torch.full((cap, 3), 12345.0, device=cuda))
    assert torch.equal(again, out)


def affine_teacher(cuda, grid, a, b, k=1.0 / 16, vector_slope=None):
    """Level 0 (dense) of grid `grid` holds a . (i0, i1, i2) + b at lattice vertex (i0, i1, i2) of the grid's own three
    dimensions (both features); every other level, grid and vector is 0 except the paired vector, constant 1 on level 0.
    The sigma net is h0 = k F_0 (two ReLU units, W1 = +-e0, W2 = (k, -k)).  With `vector_slope` = (c, d) the grid is the
    constant 1 instead and the paired vector is c * row + d."""
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    frames = tuple(range(15, 21))
    m = HumanRF(sorted_frame_numbers=frames, segment_sizes=(6,), **MODEL_KW)
    with torch.no_grad():
        fg = m.feature_grids[0]
        for g in fg.grids():
            g.zero_()
        lay = fg.layout
        res, off = int(lay.res[0]), int(lay.offset[0])
        assert not (lay.hashed_mask & 1) and res ** 3 <= int(lay.size[0])
        i2, i1, i0 = torch.meshgrid(torch.arange(res), torch.arange(res), torch.arange(res), indexing="ij")
        idx = (i0 + i1 * res + i2 * res * res).reshape(-1)
        if vector_slope is None:
            val = (a[0] * i0 + a[1] * i1 + a[2] * i2 + b).reshape(-1).float()
            assert val.abs().max() < 256        # integers, exact in bf16
        else:
            val = torch.ones(res ** 3)
        t = fg.grids()[grid].view(-1, 2)
        t[off + idx, 0] = val
        t[off + idx, 1] = val
        fg.vectors.zero_()
        ax = P.PAIRED_AXIS[grid]
        if vector_slope is None:
            fg.vectors[ax, :, 0:2] = 1.0
        else:
            c, d = vector_slope
            rows = torch.arange(fg.vectors.shape[1], dtype=torch.float32)
            fg.vectors[ax, :, 0] = c * rows + d
            fg.vectors[ax, :, 1] = c * rows + d
        w1, w2 = torch.zeros(64, 32), torch.zeros(16, 64)
        w1[0, 0], w1[1, 0] = 1.0, -1.0
        w2[0, 0], w2[0, 1] = k, -k
        m.sigma_net.params.copy_(torch.cat((w1.reshape(-1), w2.reshape(-1))))
    for p in m.parameters():
        p.requires_grad_(False)
    return m.to(cuda)


# (grid, a over the grid's three dimensions (the third is t for xyt, yzt, xzt), b): |h0| = |F0| / 16 < 4 in the cube
TEACHERS = [(0, (2, -1, 1), -32), (1, (1, 2, -3), -24), (2, (-2, 1, 2), 16), (3, (1, -1, 4), 0)]


def spatial_direction(grid, a):
    v = np.zeros(3)
    for j, d in enumerate(P.GRID_DIMS[grid]):
        if d < 3:
            v[d] += a[j]
    return v


def teacher_angle_bound(grid, a, b, res=32):
    """Perpendicular share of the gradient: per component the fp32 sum is within ACC * scale |dF| sum_c |dw_c| |T_c|,
    sum_c |dw_c / dfrac_d| = 2 and |T_c| <= Tmax; the gradient itself is scale |dF| |a_s|."""
    corners = np.stack(np.meshgrid(*[[0, res - 1]] * 3, indexing="ij"), -1).reshape(-1, 3)
    tmax = np.abs(corners @ np.asarray(a, float) + b).max()
    return ACC * np.sqrt(3) * 2 * tmax / np.linalg.norm(spatial_direction(grid, a))


def _density_grad(m, pos, frame, cuda):
    from humanrf_b200.scene_representation.query_io import QueryInput

    p = torch.from_numpy(pos).to(cuda).requires_grad_(True)
    fr = torch.full((pos.shape[0],), frame, dtype=torch.int32, device=cuda)
    sigma = m.density(QueryInput(is_training=False, positions=p, frame_numbers=fr)).density
    (g,) = torch.autograd.grad(sigma.sum(), p)
    return g.double().cpu().numpy(), sigma.detach().cpu().numpy()


@pytest.mark.parametrize("grid,a,b", TEACHERS, ids=["xyz", "xyt", "yzt", "xzt"])
def test_affine_teacher_gradient_is_parallel(cuda, grid, a, b):
    m = affine_teacher(cuda, grid, a, b)
    rng = np.random.default_rng(grid)
    pos = rng.uniform(-0.45, 0.45, (5000, 3)).astype(np.float32)
    g, sigma = _density_grad(m, pos, 16, cuda)
    assert np.isfinite(sigma).all() and sigma.min() > 0
    ahat = spatial_direction(grid, a)
    ahat /= np.linalg.norm(ahat)
    gn = np.linalg.norm(g, axis=1)
    live = gn > 0
    assert live.mean() > 0.99
    cos = (g[live] @ ahat) / gn[live]
    perp = np.linalg.norm(g[live] - np.outer(g[live] @ ahat, ahat), axis=1) / gn[live]
    bound = teacher_angle_bound(grid, a, b)
    print(f"grid {grid}: max perpendicular share {perp.max():.3e} (bound {bound:.3e})")
    assert (cos > 0).all() and (perp <= bound).all()


def test_vector_teacher_gradient_is_along_z(cuda):
    """Constant xyt grid, affine vectors[z]: only the vector term acts, and only along z."""
    c, d = 2.0 ** -9, -2.0
    m = affine_teacher(cuda, 1, None, None, k=1.0, vector_slope=(c, d))
    rng = np.random.default_rng(4)
    pos = rng.uniform(-0.45, 0.45, (5000, 3)).astype(np.float32)
    g, _ = _density_grad(m, pos, 17, cuda)
    gn = np.linalg.norm(g, axis=1)
    assert (gn > 0).all() and (g[:, 2] > 0).all()
    # x, y: the grid term sum_c dw_c * 1 cancels up to the fp32 sum (ACC * scale * 2 |dF|); |g_z| = |dF| c vec_res
    scale = float(m.feature_grids[0].layout.scale[0])
    bound = ACC * scale * 2 / (c * 2048)
    share = np.abs(g[:, :2]).max(1) / np.abs(g[:, 2])
    print(f"vector teacher: max off-axis share {share.max():.3e} (bound {bound:.3e})")
    assert (share <= bound).all()


def _oracle_dF(om, feats64, directions, want_rgb, rng):
    """d(loss)/d(features) through the oracle MLPs (bf16 rounding points of the kernels), for a fixed random loss."""
    f = feats64.float().clone().requires_grad_(True)
    sigma, geo = om.sigma_head(om._q(f))
    cs = torch.from_numpy(rng.standard_normal(sigma.shape[0])).float()
    cg = torch.from_numpy(rng.standard_normal(tuple(geo.shape))).float()
    loss = (sigma * cs / sigma.detach().clamp(min=1e-3)).sum() + (geo * cg).sum()
    if want_rgb:
        rgb = om.color_head(directions, geo)
        cr = torch.from_numpy(rng.standard_normal(tuple(rgb.shape))).float()
        loss = loss + (rgb * cr).sum()
    (d,) = torch.autograd.grad(loss, f)
    return d.double(), cs, cg, (cr if want_rgb else None)


@pytest.mark.parametrize("mode", ["density", "forward"])
def test_autograd_positions_against_oracle(cuda, mode):
    from humanrf_b200.scene_representation.query_io import QueryInput

    om, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    segs = P.segments_of(m)
    f2s, f2t = P.frame_tables(m)
    rng = np.random.default_rng(21)
    n = 4000
    pos = rng.uniform(-0.48, 0.48, (n, 3)).astype(np.float32)
    fr = rng.choice(np.asarray(frames), n).astype(np.int32)
    d = rng.standard_normal((n, 3))
    dirs = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    feats = P.features(segs, f2s, f2t, pos, fr)
    dF, cs, cg, cr = _oracle_dF(om, feats, torch.from_numpy(dirs), mode == "forward", np.random.default_rng(5))
    ref = P.position_grad(segs, f2s, f2t, pos, fr, dF).numpy()

    p = torch.from_numpy(pos).to(cuda).requires_grad_(True)
    qi = QueryInput(is_training=False, positions=p, directions=torch.from_numpy(dirs).to(cuda),
                    frame_numbers=torch.from_numpy(fr).to(cuda))
    out = m.density(qi) if mode == "density" else m.forward(qi)
    sigma = out.density
    loss = (sigma * cs.to(cuda) / sigma.detach().clamp(min=1e-3)).sum() + (out.geometry_features.float() * cg.to(cuda)).sum()
    if mode == "forward":
        loss = loss + (out.radiance * cr.to(cuda)).sum()
    loss.backward()
    got = p.grad.double().cpu().numpy()
    rel = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    print(f"{mode}: norm-wise |d_pos - oracle| / |oracle| = {rel:.3e}")
    assert rel < 3e-2
    assert all(q.grad is not None for q in m.hot_parameters())


def _separated_batch(cuda, frames):
    """16 samples far apart (no two share a table corner or a vector row at any level): one addition per gradient entry,
    so the table and vector gradients do not depend on the order of the atomic adds."""
    g = np.linspace(-0.3, 0.3, 4, dtype=np.float32)
    x, y = np.meshgrid(g, g, indexing="ij")
    i = np.arange(16)
    z = (0.2 * ((i + i // 4) % 4) - 0.3).astype(np.float32)      # distinct along every pair of axes too
    pos = np.stack([x.reshape(-1), y.reshape(-1), z], 1).astype(np.float32)
    return pos, np.full(16, frames[1], np.int32)


def _param_grads(m, pos, fr, dirs, cuda, pos_grad):
    from humanrf_b200.scene_representation.query_io import QueryInput

    for q in m.hot_parameters():
        q.grad = None
    p = torch.from_numpy(pos).to(cuda).requires_grad_(pos_grad)
    qi = QueryInput(is_training=False, positions=p, directions=torch.from_numpy(dirs).to(cuda),
                    frame_numbers=torch.from_numpy(fr).to(cuda))
    out = m.forward(qi)
    (out.density.sum() * 1e-3 + out.radiance.sum() + out.geometry_features.float().sum()).backward()
    return [q.grad.clone() for q in m.hot_parameters()], p.grad


def test_parameter_gradients_do_not_change_with_position_gradients(cuda):
    _, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    pos, fr = _separated_batch(cuda, frames)
    dirs = np.tile(np.array([[0.0, 0.6, 0.8]], np.float32), (16, 1))
    a, pa = _param_grads(m, pos, fr, dirs, cuda, False)
    b, _ = _param_grads(m, pos, fr, dirs, cuda, False)
    c, pc = _param_grads(m, pos, fr, dirs, cuda, True)
    assert pa is None and pc is not None and pc.shape == (16, 3) and (pc.abs().sum(1) > 0).all()
    assert all(torch.equal(x, y) for x, y in zip(a, b))          # the premise: this batch has one order of adds
    assert all(torch.equal(x, y) for x, y in zip(a, c))


def test_frozen_parameters_position_gradient_without_scatter(cuda):
    from torch.profiler import ProfilerActivity, profile

    from humanrf_b200.scene_representation.query_io import QueryInput

    _, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    rng = np.random.default_rng(2)
    pos = rng.uniform(-0.45, 0.45, (3000, 3)).astype(np.float32)
    fr = rng.choice(np.asarray(frames), 3000).astype(np.int32)
    qi = lambda p: QueryInput(is_training=False, positions=p, frame_numbers=torch.from_numpy(fr).to(cuda))
    # reference: the same gradient with trainable parameters
    p0 = torch.from_numpy(pos).to(cuda).requires_grad_(True)
    m.density(qi(p0)).density.sum().backward()
    for q in m.hot_parameters():
        q.requires_grad_(False)
        q.grad = None
    p1 = torch.from_numpy(pos).to(cuda).requires_grad_(True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.density(qi(p1)).density.sum().backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("position_grad" in s for s in names) and any("field_backward_kernel" in s for s in names)
    assert not any("scatter" in s for s in names), [s for s in names if "scatter" in s]
    assert torch.equal(p1.grad, p0.grad)
    assert all(q.grad is None for q in m.hot_parameters())


def test_positions_grad_stays_none_when_not_requested(cuda):
    from humanrf_b200.scene_representation.query_io import QueryInput

    _, m, frames = make_pair((6,), table_std=2.0, device=cuda)
    p = torch.zeros((64, 3), device=cuda)
    fr = torch.full((64,), frames[0], dtype=torch.int32, device=cuda)
    m.density(QueryInput(is_training=False, positions=p, frame_numbers=fr)).density.sum().backward()
    assert p.grad is None and m.sigma_net.params.grad is not None
    # requires_grad set, but only the parameters are asked for
    p2 = torch.zeros((64, 3), device=cuda, requires_grad=True)
    s = m.density(QueryInput(is_training=False, positions=p2, frame_numbers=fr)).density.sum()
    torch.autograd.grad(s, [m.sigma_net.params])
    assert p2.grad is None
