"""Data-parallel camera refinement on the H100 (DESIGN.md §3.16).

One device: W ranks simulated as in test_optimizer_gpu.py's DpWorld -- W CameraPoses (W records, descriptor sets, copies
of the tables and slot pools), each stepped by hrf_camera_pose_step_ranks / hrf_camera_calib_step_ranks over all W
records -- against tests/pose_dp_oracle.py, replica against replica, W = 1 against the single-rank kernels, the p2p
layout (W allocations) against the nccl layout (one [W, record] tensor), the error words, and the union batch.
Two or more GPUs: FusedTrainer with camera_poses at world 2 for both exchanges (skipped with fewer GPUs).

Bars: parameters and moments to 1e-6 relative of the float64 oracle fed the kernel's own reduction (the pose step's bar
in test_camera_poses_gpu.py); tables within 1 fp32 ulp of view_table / calibration_table; replicas, layouts and
reruns bit for bit.  Union batch, each rank's ray gradients from the train step's kernels at its loss_scale: bars
derived from the MLP backward's bf16 rounding (test_union_batch_on_one_device).
"""
import os
from types import SimpleNamespace

import ctypes as C
import numpy as np
import pytest
import torch

import pose_dp_oracle as DO

pytestmark = pytest.mark.gpu


def _world_loaders(cuda, C_, W, seed=0):
    """W loaders over the same C_ cameras (random well-conditioned tables, dataset cameras for the intrinsics), each
    with its own slot pool."""
    rng = np.random.default_rng((seed, C_))
    ikr = (np.eye(3) * 1e-3 + rng.standard_normal((C_, 3, 3)) * 2e-4).astype(np.float32)
    org = rng.standard_normal((C_, 3)).astype(np.float32)
    cams = [SimpleNamespace(width=96, height=72, focal_length=rng.uniform(0.8, 1.2, 2), principal_point=rng.uniform(0.4, 0.6, 2),
                            rotation_axisangle=rng.standard_normal(3)) for _ in range(C_)]
    out = []
    for r in range(W):
        B = 3 + 5 * r
        slots = rng.integers(-1, C_, B).astype(np.int32)
        out.append(SimpleNamespace(all_inverse_krs=torch.from_numpy(ikr).to(cuda).contiguous(),
                                   all_camera_origins=torch.from_numpy(org).to(cuda).contiguous(),
                                   camera_numbers=tuple(range(C_)), cameras=cams, scene_scale=1.0, scene_offset=np.zeros(3),
                                   inverse_krs_cuda=torch.full((B, 3, 3), 7.0, device=cuda),
                                   camera_origins_cuda=torch.full((B, 3), 7.0, device=cuda),
                                   camera_numbers_cuda=torch.from_numpy(slots).to(cuda)))
    return out


def _poses(loaders, calib, fixed=(0,)):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    return [CameraPoses(ld, lr=3e-3, final_lr_ratio=1.0, fixed_cameras=fixed, intrinsics=calib, intrinsics_lr=1e-3)
            for ld in loaders]


def _step_ranks(p, rank, addrs, error, t=0):
    """Rank `rank`'s ranked step over the records at `addrs` (the C entry FusedTrainer's pose step calls)."""
    from humanrf_b200 import _lib as L

    rec = L.CameraGradRecords()
    for r, a in enumerate(addrs):
        rec.record[r] = a
    rec.world, rec.rank = len(addrs), rank
    b1, b2 = p.betas
    if p.intrinsics:
        L.check(L.lib().hrf_camera_calib_step_ranks(C.byref(p._desc), C.byref(p._idesc), C.byref(rec), error.data_ptr(),
                                                    p.current_lr(t), p.current_intrinsics_lr(t), b1, b2, p.eps, L.stream()))
    else:
        L.check(L.lib().hrf_camera_pose_step_ranks(C.byref(p._desc), C.byref(rec), error.data_ptr(), p.current_lr(t), b1, b2,
                                                   p.eps, L.stream()))


def _fill(world, rng, step):
    """Writes one step's records: camera C-1 seen by the last rank only, camera 1 by none, camera 0 (fixed) by all, and
    one rank other than the last empty (W >= 2).  Returns (grads, counts) as the oracle takes them."""
    W, C_ = len(world), world[0].num_cameras
    K = 10 if world[0].intrinsics else 6
    grads, counts = [], []
    for r, p in enumerate(world):
        g = (rng.standard_normal((C_, K)) * 10.0 ** rng.uniform(-4, 1, (C_, 1))).astype(np.float32)
        n = (rng.random(C_) < 0.6).astype(np.int32) * rng.integers(1, 1000, C_).astype(np.int32)
        n[0] = 5
        if C_ > 1:
            n[1], g[1] = 0, 0.0
        if C_ > 2:
            n[C_ - 1] = 7 if r == W - 1 else 0
        if W >= 2 and r == (0 if W == 2 else W // 2):
            n[:], g[:] = 0, 0.0
        g[n == 0] = 0.0                         # what the gradient kernel writes for a camera without rays
        p.pose_grad.copy_(torch.from_numpy(g[:, :6]))
        if K == 10:
            p.intrinsics_grad.copy_(torch.from_numpy(g[:, 6:]))
        p.ray_count.copy_(torch.from_numpy(n))
        grads.append(g)
        counts.append(n)
    return grads, counts


_STATE = ("omega", "tau", "exp_avg", "exp_avg_sq", "steps")
_ISTATE = ("alpha", "beta", "intrinsics_exp_avg", "intrinsics_exp_avg_sq", "rotations")


def _snapshot(p):
    names = _STATE + (_ISTATE if p.intrinsics else ())
    out = {n: getattr(p, n).clone() for n in names}
    out["all_inverse_krs"], out["all_camera_origins"] = p.loader.all_inverse_krs.clone(), p.loader.all_camera_origins.clone()
    out["error"] = p.error.clone()
    return out


def _same(a, b):
    return [k for k in a if not torch.equal(a[k], b[k])]


def _run(cuda, calib, W, C_, layout="p2p", steps=5, seed=3):
    loaders = _world_loaders(cuda, C_, W, seed)
    world = _poses(loaders, calib)
    rng = np.random.default_rng((seed, W, C_, int(calib)))
    history = []
    gather = torch.zeros((W, world[0].record.numel()), dtype=torch.uint8, device=cuda)
    for k in range(steps):
        grads, counts = _fill(world, rng, k)
        if layout == "p2p":
            addrs = [p.record.data_ptr() for p in world]
        else:
            for r, p in enumerate(world):
                gather[r].copy_(p.record)
            addrs = [gather[r].data_ptr() for r in range(W)]
        for r, p in enumerate(world):
            _step_ranks(p, r, addrs, p.error, k)
        history.append((grads, counts))
    torch.cuda.synchronize()
    return loaders, world, history


def _oracle(world, history):
    C_ = world[0].num_cameras
    calib = world[0].intrinsics
    K = 10 if calib else 6
    st = dict(params=np.zeros((C_, K)), m=np.zeros((C_, K)), v=np.zeros((C_, K)), steps=np.zeros(C_, np.int64))
    fixed = world[0].fixed.cpu().numpy().astype(bool)
    for grads, counts in history:
        DO.ranked_step(st, grads, counts, [0] * len(grads), fixed, 3e-3, 1e-3 if calib else None)
    return st


def _ulp_close(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    return bool((np.abs(a.astype(np.float64) - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all())


@pytest.mark.parametrize("C_", [1, 8, 160, 1024])
@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("calib", [False, True], ids=["pose", "intrinsics"])
def test_step_ranks_against_oracle(cuda, calib, W, C_):
    from humanrf_b200.toolbox.camera_refinement import calibration_table, view_table

    loaders, world, history = _run(cuda, calib, W, C_)
    p0 = world[0]
    # replicas: bit for bit, their slot pools copies of their own tables
    ref = _snapshot(p0)
    for r, p in enumerate(world[1:], 1):
        assert not _same(ref, _snapshot(p)), (r, _same(ref, _snapshot(p)))
    for ld in loaders:
        cams = ld.camera_numbers_cuda.long()
        has = cams >= 0
        assert torch.equal(ld.inverse_krs_cuda[has], ld.all_inverse_krs[cams[has]])
        assert torch.equal(ld.camera_origins_cuda[has], ld.all_camera_origins[cams[has]])
        assert (ld.inverse_krs_cuda[~has] == 7.0).all()
    # against the oracle
    st = _oracle(world, history)
    params = torch.cat([p0.omega, p0.tau] + ([p0.alpha, p0.beta] if calib else []), 1).cpu().numpy()
    np.testing.assert_allclose(params, st["params"], rtol=1e-6, atol=1e-12)
    m = torch.cat([p0.exp_avg] + ([p0.intrinsics_exp_avg] if calib else []), 1).cpu().numpy()
    v = torch.cat([p0.exp_avg_sq] + ([p0.intrinsics_exp_avg_sq] if calib else []), 1).cpu().numpy()
    np.testing.assert_allclose(m, st["m"], rtol=1e-6, atol=1e-30)
    np.testing.assert_allclose(v, st["v"], rtol=1e-6, atol=1e-30)
    assert np.array_equal(p0.steps.cpu().numpy(), st["steps"])
    if C_ > 2:
        assert st["steps"][C_ - 1] == 5 and st["steps"][1] == 0 and st["steps"][0] == 0
    # tables within 1 ulp (a sample of cameras at C = 1024), untouched cameras bit for bit
    base = p0.base_inverse_krs
    for c in sorted(set(range(min(C_, 48))) | {C_ - 1}):
        if calib:
            want = calibration_table(base[c], p0.omega[c], p0.alpha[c], p0.beta[c], p0.base_intrinsics[c].tolist())
        else:
            want = view_table(base[c], p0.omega[c])
        assert _ulp_close(loaders[0].all_inverse_krs[c], want), c
        assert torch.equal(loaders[0].all_camera_origins[c], (p0.base_camera_origins[c].double() + p0.tau[c]).float())
        if st["steps"][c] == 0:
            assert torch.equal(loaders[0].all_inverse_krs[c], base[c])


@pytest.mark.parametrize("C_", [8, 1024])
@pytest.mark.parametrize("calib", [False, True], ids=["pose", "intrinsics"])
def test_one_rank_equals_single_rank_step_bit_for_bit(cuda, calib, C_):
    (la,), (lb,) = _world_loaders(cuda, C_, 1, 7), _world_loaders(cuda, C_, 1, 7)
    (a,), (b,) = _poses([la], calib), _poses([lb], calib)
    rng = np.random.default_rng(C_)
    for k in range(5):
        grads, counts = _fill([a], rng, k)
        b.record.copy_(a.record)
        a.step(k, [a.record.data_ptr()])        # the ranked entry at W = 1
        b.step(k)                               # hrf_camera_pose_step / hrf_camera_calib_step
    torch.cuda.synchronize()
    assert not _same(_snapshot(a), _snapshot(b))
    assert torch.equal(la.inverse_krs_cuda, lb.inverse_krs_cuda) and torch.equal(la.camera_origins_cuda, lb.camera_origins_cuda)
    assert int(a.steps.sum()) > 0


@pytest.mark.parametrize("calib", [False, True], ids=["pose", "intrinsics"])
def test_layouts_and_reruns_give_the_same_bits(cuda, calib):
    runs = [_run(cuda, calib, 5, 160, layout) for layout in ("p2p", "nccl", "p2p")]
    snaps = [[_snapshot(p) for p in world] for _, world, _ in runs]
    for other in snaps[1:]:
        for a, b in zip(snaps[0], other):
            assert not _same(a, b)
    for (la, _, _), (lb, _, _) in zip([runs[0]] * 2, runs[1:]):
        for x, y in zip(la, lb):
            assert torch.equal(x.inverse_krs_cuda, y.inverse_krs_cuda)


def test_reversed_rank_order_changes_the_step(cuda):
    """The kernel sums in rank order: 2^-30 + 2^30 - 2^30 is 0 from rank 0 up and 2^-30 from the top."""
    loaders = _world_loaders(cuda, 4, 8, 1)
    world = _poses(loaders, False)
    for r, p in enumerate(world):
        p.ray_count.fill_(3)
        p.pose_grad.zero_()
    for r, v in ((0, 2.0 ** -30), (1, 2.0 ** 30), (2, -(2.0 ** 30))):
        world[r].pose_grad[1] = v
    addrs = [p.record.data_ptr() for p in world]
    _step_ranks(world[0], 0, addrs, world[0].error)
    _step_ranks(world[1], 1, addrs[::-1], world[1].error)       # rank order reversed
    torch.cuda.synchronize()
    assert float(world[0].omega[1].abs().sum()) == 0.0 and int(world[0].steps[1]) == 1
    assert float(world[1].omega[1].abs().sum()) > 0.0


@pytest.mark.parametrize("calib", [False, True], ids=["pose", "intrinsics"])
def test_bad_camera_on_one_rank_stops_every_rank(cuda, calib):
    W = 3
    loaders = _world_loaders(cuda, 6, W, 2)
    world = _poses(loaders, calib)
    rng = np.random.default_rng(0)
    _fill(world, rng, 0)
    rays = torch.randn(50, 3, device=cuda)
    d = rays / rays.norm(dim=1, keepdim=True)
    cams = torch.randint(0, 6, (50,), dtype=torch.int32, device=cuda)
    cams[17] = 6                                                   # rank 1's batch holds a bad camera number
    world[1].accumulate(torch.randn(50, 3, device=cuda), torch.randn(50, 3, device=cuda), d, cams, 50)
    before = [_snapshot(p) for p in world]
    slots = [ld.inverse_krs_cuda.clone() for ld in loaders]
    addrs = [p.record.data_ptr() for p in world]
    for r, p in enumerate(world):
        _step_ranks(p, r, addrs, p.error)
    torch.cuda.synchronize()
    assert [int(p.error[0]) for p in world] == [2, 1, 2]
    for r, p in enumerate(world):
        after = _snapshot(p)
        assert _same(before[r], after) == ["error"] if r != 1 else not _same(before[r], after), r
        assert torch.equal(slots[r], loaders[r].inverse_krs_cuda)
        with pytest.raises(RuntimeError, match="outside"):
            p.check()
        with pytest.raises(RuntimeError, match="outside"):
            p.state_dict()


def _ray_gradients(tr, o, d, fr, t, ri, rgba, bg, R, loss_scale, step):
    """(g_o, g_d) of one rank's share: the kernels FusedTrainer.step runs with camera_poses and prune=False, in its
    order, the loss weighted by `loss_scale` (device float32 [1]) as a data-parallel rank's is."""
    from humanrf_b200 import _lib as L
    from humanrf_b200.volume_rendering import ray_offsets

    lib, nat, dev = L.lib(), tr.nat, o.device
    n_cap = t.shape[0]
    off = ray_offsets(ri, R)
    samples = nat.samples_rays(o, d, fr, t, ri, None, count_dev=None)
    sigma, _, rgb, feat = nat.forward(samples, 1, want_geo=False, want_feat=True)
    color = torch.empty((R, 3), device=dev)
    wsum = torch.empty((R, 1), device=dev)
    L.check(lib.hrf_composite_forward(sigma.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(), R, step, bg.data_ptr(),
                                      color.data_ptr(), wsum.data_ptr(), None, L.stream()))
    d_color, d_wsum, loss = torch.empty((R, 3), device=dev), torch.empty(R, device=dev), torch.zeros(1, device=dev)
    L.check(lib.hrf_train_loss(color.data_ptr(), wsum.data_ptr(), rgba.data_ptr(), bg.data_ptr(), R, tr.delta, tr.bce_w,
                               L.ptr(loss_scale), d_color.data_ptr(), d_wsum.data_ptr(), loss.data_ptr(), L.stream()))
    d_sigma, d_rgb = torch.empty(n_cap, device=dev), torch.empty((n_cap, 3), device=dev)
    L.check(lib.hrf_composite_backward(sigma.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(), R, step, bg.data_ptr(),
                                       d_color.data_ptr(), d_wsum.data_ptr(), d_sigma.data_ptr(), d_rgb.data_ptr(), L.stream()))
    tr.grad.zero_()
    ws = torch.empty(n_cap * 40, device=dev)
    d_dir = torch.empty((n_cap, 3), device=dev)
    L.check(lib.hrf_field_backward_mlp_dirs(C.byref(nat.field), C.byref(samples), d_sigma.data_ptr(), d_rgb.data_ptr(), None,
                                            feat.data_ptr(), None, tr.mlp_grad.data_ptr(), L.ptr(tr.emb_grad),
                                            d_dir.data_ptr(), ws.data_ptr(), L.stream()))
    L.check(lib.hrf_field_backward_tables(C.byref(nat.field), C.byref(samples), tr.sg_dev.data_ptr(),
                                          feat.data_ptr() + 64 * n_cap, None, n_cap, ws.data_ptr(), 0, 4, L.stream()))
    d_pos = torch.empty((n_cap, 3), device=dev)
    L.check(lib.hrf_field_position_grad(C.byref(nat.field), C.byref(samples), ws.data_ptr(), d_pos.data_ptr(), L.stream()))
    g_o, g_d = torch.empty((R, 3), device=dev), torch.empty((R, 3), device=dev)
    L.check(lib.hrf_ray_gradients(d_pos.data_ptr(), d_dir.data_ptr(), t.data_ptr(), d.data_ptr(), off.data_ptr(), R,
                                  g_o.data_ptr(), g_d.data_ptr(), None, L.stream()))
    return g_o, g_d


@pytest.mark.parametrize("calib", [False, True], ids=["pose", "intrinsics"])
@pytest.mark.parametrize("W", [2, 3])
def test_union_batch_on_one_device(cuda, calib, W):
    """One ray batch split over W simulated ranks at unequal shares, rank 0 empty.  Each non-empty rank runs the train
    step's kernels on its share with its loss_scale W R_r / R_total (hrf_train_loss, the composite and field backward,
    hrf_field_position_grad, hrf_ray_gradients) and accumulate(); the empty rank writes its zero record.  Against the
    single-process union batch (loss_scale 1).  The MLP backward rounds the scaled loss gradients through bf16 tiles, so
    a share scaled by W R_r / R_total (not a power of two) rounds each sample differently at 2^-9 relative: measured
    3e-3 norm-wise per share at W = 3, 0 at W = 2 (rank 1 holds the whole batch, its scale is exactly 2).  Bars:
    * per ray, g_r / W against the union's gradient: 2^-7 norm-wise over the share;
    * the reduced pose and intrinsics gradients: 2^-6 norm-wise per camera (the share's bar, doubled for the
      cancellation in a camera's sum: the bf16 rounding does not average out, 2e-3 to 7.5e-3 measured at W = 3);
    * one ranked step: Adam's first step moves each entry by lr sign(g), so every entry whose union gradient is above
      1e-1 of its camera's largest matches to 1e-9 relative, the step counters are equal, and the tables of the cameras
      with no entry below that are within 2 fp32 ulp."""
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.training import FusedTrainer
    from test_dp_gpu import _subset

    C_, R, step = 8, 512, 4e-4
    model, frames = make_model((6,), table_std=0.5, device=cuda)
    tr = FusedTrainer(model, prune=False, render_step_size=step)      # the gradient buffers the backward writes into
    b = synthetic_rays(R, 48, frames, seed=4, ragged=True)
    bg_all = torch.rand(R, 3, generator=torch.Generator().manual_seed(9)).to(cuda)
    cams = ((torch.arange(R, dtype=torch.int32) * 5) % C_).to(cuda)
    rng = np.random.default_rng(W)
    cuts = [0, 0] + sorted(rng.choice(np.arange(1, R), W - 2, replace=False).tolist()) + [R]
    (lu,) = _world_loaders(cuda, C_, 1, 4)
    (union,) = _poses([lu], calib)
    world = _poses(_world_loaders(cuda, C_, W, 4), calib)

    def share(lo, hi):
        sb = {k: v.to(cuda).contiguous() for k, v in _subset(b, lo, hi).items()}
        return sb["o"], sb["d"], sb["frames"], sb["t"].reshape(-1), sb["ri"].long(), sb["rgba"].float().contiguous()

    o, d, fr, t, ri, rgba = share(0, R)
    g_o, g_d = _ray_gradients(tr, o, d, fr, t, ri, rgba, bg_all, R, None, step)
    union.accumulate(g_o, g_d, d, cams, R)
    for r, p in enumerate(world):
        lo, hi = cuts[r], cuts[r + 1]
        if hi == lo:
            empty = torch.empty((0, 3), device=cuda)
            p.accumulate(empty, empty, empty, torch.empty(0, dtype=torch.int32, device=cuda), 0)
            continue
        scale = torch.tensor([W * (hi - lo) / R], dtype=torch.float32, device=cuda)
        so, sd, sf, st, sri, srgba = share(lo, hi)
        r_o, r_d = _ray_gradients(tr, so, sd, sf, st, sri, srgba, bg_all[lo:hi].contiguous(), hi - lo, scale, step)
        for got, want in ((r_o / W, g_o[lo:hi]), (r_d / W, g_d[lo:hi])):
            assert float((got - want).norm()) <= 2.0 ** -7 * float(want.norm()), r
        p.accumulate(r_o, r_d, sd, cams[lo:hi].contiguous(), hi - lo)
    torch.cuda.synchronize()
    assert int(world[0].ray_count.sum()) == 0 and int(world[0].error[0]) == 0
    recs = [torch.cat([p.pose_grad] + ([p.intrinsics_grad] if calib else []), 1).double().cpu().numpy() for p in world]
    red, touched = DO.reduce_records(recs, [p.ray_count.cpu().numpy() for p in world])
    ref = torch.cat([union.pose_grad] + ([union.intrinsics_grad] if calib else []), 1).double().cpu().numpy()
    assert np.array_equal(touched, union.ray_count.cpu().numpy() > 0) and touched.all()
    err = np.linalg.norm(red - ref, axis=1) / np.maximum(np.linalg.norm(ref, axis=1), 1e-30)
    assert (err <= 2.0 ** -6).all(), err
    if W == 2:                                      # the one non-empty rank holds the whole batch at scale 2: exact
        assert (err <= 1e-6).all(), err
    addrs = [p.record.data_ptr() for p in world]
    for r, p in enumerate(world):
        _step_ranks(p, r, addrs, p.error)
    union.step(0)
    torch.cuda.synchronize()
    names = ("omega", "tau") + (("alpha", "beta") if calib else ())
    a = np.concatenate([getattr(world[0], n).cpu().numpy() for n in names], 1)
    b_ = np.concatenate([getattr(union, n).cpu().numpy() for n in names], 1)
    clear = np.abs(ref) >= 1e-1 * np.abs(ref).max(axis=1, keepdims=True)      # no sign flip at the gradients' bar
    assert clear.sum() > 0.5 * clear.size
    assert (np.abs(a - b_)[clear] <= 1e-9 * np.abs(b_)[clear]).all()
    assert torch.equal(world[0].steps, union.steps)
    ok = clear.all(axis=1) & (world[0].fixed.cpu().numpy() == 0)
    assert ok.any() or calib
    for mine, theirs in ((world[0].loader.all_inverse_krs, lu.all_inverse_krs),
                         (world[0].loader.all_camera_origins, lu.all_camera_origins)):
        x, y = mine.cpu().numpy()[ok], theirs.cpu().numpy()[ok]
        assert (np.abs(x.astype(np.float64) - y) <= 2 * np.spacing(np.maximum(np.abs(x), np.abs(y)))).all()


# ------------------------------------------------------------------------------------------------ two or more GPUs
def _train_rank(rank, world, port, spans, q, exchange, plan_bad=False, steps=3):
    import torch.distributed as dist

    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.training import FusedTrainer

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    pg = None
    if world > 1:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    model, frames = make_model((6,), table_std=0.5, device=dev)
    b = synthetic_rays(512, 48, frames, seed=4, ragged=True)
    bg_all = torch.rand(512, 3, generator=torch.Generator().manual_seed(9))
    cams_all = (torch.arange(512, dtype=torch.int32) * 7) % 5
    (ld,) = _world_loaders(dev, 5, 1, 6)
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    poses = CameraPoses(ld, lr=1e-3, final_lr_ratio=1.0, intrinsics=True, world_size=world, process_group=pg)
    lo, hi = spans[rank]
    tr = FusedTrainer(model, lr=1e-2, prune=False, world_size=world, exchange=exchange, camera_poses=poses)
    from test_dp_gpu import _subset

    first = None
    for step in range(steps):
        sb = {k: v.to(dev).contiguous() for k, v in _subset(b, lo, hi).items()}
        cams = cams_all[lo:hi].clone()
        if plan_bad and rank == 1:
            cams[3] = 99
        tr.step(sb["o"], sb["d"], sb["frames"], sb["t"], sb["ri"], sb["rgba"], hi - lo, background=bg_all[lo:hi].to(dev),
                cameras=cams.to(dev))
        if step == 0:
            torch.cuda.synchronize()
            first = (poses.omega.cpu().numpy().copy(), poses.tau.cpu().numpy().copy())
    tr.gather_master_parameters()
    torch.cuda.synchronize()
    err = None
    try:
        state = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in poses.state_dict().items()}
        state["rotations"] = poses.rotations.cpu().numpy()
        state["tables"] = (ld.all_inverse_krs.cpu().numpy(), ld.all_camera_origins.cpu().numpy(),
                           ld.inverse_krs_cuda.cpu().numpy())
    except RuntimeError as e:
        state, err = None, str(e)
    q.put((rank, [p.detach().cpu().numpy() for p in model.hot_parameters()], state, first, err))
    if world > 1:
        dist.barrier()
        tr.close()
        dist.destroy_process_group()


def _spawn(world, spans, exchange, plan_bad, port_offset):
    import torch.multiprocessing as mp
    from test_dp_gpu import _collect

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + os.getpid() % 100 + port_offset
    procs = [ctx.Process(target=_train_rank, args=(r, world, port, spans, q, exchange, plan_bad)) for r in range(world)]
    for p in procs:
        p.start()
    got = {r: rest for r, *rest in _collect(q, procs, world)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return got


def test_two_rank_training_with_camera_poses(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ref = _spawn(1, [(0, 512)], "nccl", False, 0)[0]
    firsts = {}
    for i, exchange in enumerate(("nccl", "p2p")):
        got = _spawn(2, [(0, 200), (200, 512)], exchange, False, 1 + i)
        (f0, s0, first0, e0), (f1, s1, first1, e1) = got[0], got[1]
        assert e0 is None and e1 is None
        for k in s0:                                             # replicas: poses, moments, counters, rotations
            if k != "tables":
                assert np.array_equal(np.asarray(s0[k]), np.asarray(s1[k])), (exchange, k)
        assert all(np.array_equal(a, b) for a, b in zip(s0["tables"][:2], s1["tables"][:2]))
        assert all(np.array_equal(a, b) for a, b in zip(f0, f1)), exchange
        firsts[exchange] = first0
        # the field within test_dp_gpu's bar of the union batch, the poses within 1e-3 of the distance moved
        for a, b in zip(f0, ref[0]):
            assert np.linalg.norm(a - b) <= 1e-4 * max(np.linalg.norm(b), 1e-12) + 1e-6
        for k in ("omega", "tau", "alpha", "beta"):
            moved = np.linalg.norm(ref[1][k])
            assert np.linalg.norm(s0[k] - ref[1][k]) <= 1e-3 * max(moved, 1e-12), (exchange, k)
    assert all(np.array_equal(a, b) for a, b in zip(firsts["nccl"], firsts["p2p"]))


@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_two_rank_bad_camera_stops_both_ranks(cuda, exchange):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = _spawn(2, [(0, 200), (200, 512)], exchange, True, 5 + ["nccl", "p2p"].index(exchange))
    assert got[0][3] is not None and "another rank" in got[0][3]
    assert got[1][3] is not None and "outside" in got[1][3]
    assert float(np.abs(got[0][2][0]).sum()) == 0.0 and float(np.abs(got[1][2][0]).sum()) == 0.0
