"""Per-camera pose refinement in the fused train step on the H100: the pose-gradient reduction (hrf_camera_pose_grad)
and the per-camera Adam with its table rewrite (hrf_camera_pose_step) against tests/pose_oracle.py and torch, one
FusedTrainer step against render() under autograd, the unchanged default step, and recovery of perturbed cameras.

Bars:
* pose gradient: n 2^-23 sum|terms| per entry (the fp32 accumulation bound of any summation order, the cross products'
  own rounding included) against the float64 sums of the kernel's own inputs, carried through |J_l^T|.
* pose step: parameters and moments to 1e-6 relative of torch.optim.Adam run on the touched cameras only; tables within
  1 fp32 ulp of view_table (the kernel's Rodrigues exponential and torch's matrix_exp differ in the last float64 bits).
* end to end: 1e-3 norm-wise per camera.  Both routes run the same field kernels on the same rays and samples, bit for
  bit; they differ only in the loss's fp32 evaluation and in the order of the per-camera sums.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import pose_oracle as PO
from helpers import make_pair, synthetic_rays

pytestmark = pytest.mark.gpu


def _rays(R, C_, rng, cams=None):
    d = rng.standard_normal((R, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    g_d = (rng.standard_normal((R, 3)) * rng.uniform(0.1, 10.0, (R, 1))).astype(np.float32)
    g_o = rng.standard_normal((R, 3)).astype(np.float32)
    if cams is None:
        cams = rng.integers(0, C_, R).astype(np.int32)
    return g_o, g_d, d, np.asarray(cams, np.int32)


def _check_pose_grad(cuda, g_o, g_d, d, cams, omega):
    from humanrf_b200.toolbox.camera_refinement import pose_gradients

    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
    args = (dev(g_o), dev(g_d), dev(d), dev(cams), dev(omega))
    pg, cnt = pose_gradients(*args)
    pg2, cnt2 = pose_gradients(*args)
    assert torch.equal(pg, pg2) and torch.equal(cnt, cnt2)                 # bit for bit
    ref, n, bound = PO.pose_grad(g_o, g_d, d, cams, omega)
    got = pg.double().cpu().numpy()
    assert np.array_equal(cnt.cpu().numpy(), n)
    err = np.abs(got - ref)
    assert (err <= bound).all(), f"max err/bound {(err / np.maximum(bound, 1e-300)).max():.3e}"
    assert (got[n == 0] == 0).all()
    return got, n


@pytest.mark.parametrize("C_", [1, 8, 160])
@pytest.mark.parametrize("R", [1, 31, 4096, 300000])
def test_pose_grad_kernel(cuda, R, C_):
    rng = np.random.default_rng(R * 7 + C_)
    cams = None
    if C_ > 1:      # leave cameras without rays: only the even ones take part
        cams = (2 * rng.integers(0, (C_ + 1) // 2, R)).astype(np.int32)
    omega = rng.standard_normal((C_, 3)) * rng.choice([0.0, 1e-9, 1e-3, 0.4, 2.0], (C_, 1))
    g_o, g_d, d, cams = _rays(R, C_, rng, cams)
    got, n = _check_pose_grad(cuda, g_o, g_d, d, cams, omega)
    if C_ > 1:
        assert (n[1::2] == 0).all()
    assert n.sum() == R


def test_pose_grad_kernel_one_camera_owns_every_ray(cuda):
    rng = np.random.default_rng(1)
    R, C_ = 300000, 8
    omega = rng.standard_normal((C_, 3)) * 0.5
    g_o, g_d, d, cams = _rays(R, C_, rng, np.full(R, 5, np.int32))
    got, n = _check_pose_grad(cuda, g_o, g_d, d, cams, omega)
    assert n[5] == R and (np.delete(got, 5, 0) == 0).all()
    # omega != 0: J_l applied (the raw sum differs)
    raw, *_ = PO.pose_grad(g_o, g_d, d, cams, np.zeros_like(omega))
    assert np.abs(raw[5, :3] - got[5, :3]).max() > 1e-3 * np.abs(raw[5, :3]).max()


def test_pose_grad_kernel_rejects_camera_outside_range(cuda):
    from humanrf_b200.toolbox.camera_refinement import pose_gradients

    rng = np.random.default_rng(2)
    for bad in (8, -2):
        g_o, g_d, d, cams = _rays(5000, 8, rng)
        cams[1234] = bad
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
        with pytest.raises(RuntimeError, match="outside"):
            pose_gradients(dev(g_o), dev(g_d), dev(d), dev(cams), torch.zeros((8, 3), dtype=torch.float64, device=cuda))
    torch.cuda.synchronize()         # the context is healthy


def _fake_loader(cuda, C_, slot_cams, seed=0):
    """The tables CameraPoses reads and writes, as a DataLoader holds them (camera tables and pool slots)."""
    from humanrf_b200.synthetic_scene import make_scene

    sc = make_scene(num_images=C_, width=96, height=72, seed=seed, portrait_every=0)
    ikr = torch.from_numpy(sc["inverse_krs"]).to(cuda).contiguous()
    org = torch.from_numpy(sc["camera_origins"]).to(cuda).contiguous()
    B = len(slot_cams)
    return SimpleNamespace(all_inverse_krs=ikr, all_camera_origins=org, camera_numbers=tuple(range(C_)),
                           inverse_krs_cuda=torch.full((B, 3, 3), 7.0, device=cuda),
                           camera_origins_cuda=torch.full((B, 3), 7.0, device=cuda),
                           camera_numbers_cuda=torch.tensor(slot_cams, dtype=torch.int32, device=cuda))


def _ulp_close(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    return bool((np.abs(a.astype(np.float64) - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all())


def test_pose_step_kernel(cuda):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, view_table

    C_, lr = 8, 3e-3
    slot_cams = [3, -1, 0, 5, 5, -1, 7, 2, 1, 6, -1, 4]
    loader = _fake_loader(cuda, C_, slot_cams)
    poses = CameraPoses(loader, lr=lr, final_lr_ratio=1.0, fixed_cameras=(0,))
    base_ikr, base_org = loader.all_inverse_krs.clone(), loader.all_camera_origins.clone()
    ref = [torch.zeros(6, dtype=torch.float64, requires_grad=True) for _ in range(C_)]
    opts = [torch.optim.Adam([p], lr=lr, betas=(0.9, 0.99), eps=1e-15) for p in ref]
    rng = np.random.default_rng(4)
    touched_sets = [[0, 1, 2, 3], [2, 3, 6], [1, 2, 3, 4, 6], [6], [0, 2, 3, 6]]
    ever = set()
    for k, touched in enumerate(touched_sets):
        count = np.zeros(C_, np.int32)
        count[touched] = rng.integers(1, 1000, len(touched))
        g = (rng.standard_normal((C_, 6)) * 10.0 ** rng.uniform(-4, 1, (C_, 1))).astype(np.float32)
        g[3] = 0.0                    # camera 3 has rays but a zero gradient: Adam leaves omega = tau = 0
        poses.pose_grad.copy_(torch.from_numpy(g))
        poses.ray_count.copy_(torch.from_numpy(count))
        before = {n: getattr(poses, n).clone() for n in ("omega", "tau", "exp_avg", "exp_avg_sq", "steps")}
        tab_before = (loader.all_inverse_krs.clone(), loader.all_camera_origins.clone())
        poses.step(k)
        torch.cuda.synchronize()
        for c in touched:
            if c != 0:
                opts[c].zero_grad()
                ref[c].grad = torch.from_numpy(g[c].astype(np.float64))
                opts[c].step()
                ever.add(c)
        for c in range(C_):
            if c in touched and c != 0:
                continue
            for n, v in before.items():                       # untouched and fixed: bit-unchanged
                assert torch.equal(getattr(poses, n)[c], v[c]), (k, c, n)
            assert torch.equal(loader.all_inverse_krs[c], tab_before[0][c])
            assert torch.equal(loader.all_camera_origins[c], tab_before[1][c])
    params = torch.cat((poses.omega, poses.tau), 1).cpu()
    for c in range(C_):
        r = ref[c].detach()
        assert torch.allclose(params[c], r, rtol=1e-6, atol=1e-12), c
        st = opts[c].state.get(ref[c])
        if st:
            assert torch.allclose(poses.exp_avg[c].cpu(), st["exp_avg"], rtol=1e-6, atol=1e-30)
            assert torch.allclose(poses.exp_avg_sq[c].cpu(), st["exp_avg_sq"], rtol=1e-6, atol=1e-30)
            assert int(poses.steps[c]) == int(st["step"])
        else:
            assert int(poses.steps[c]) == 0
    # tables: within 1 ulp of view_table; camera 3 (rewritten at omega = 0) and never-moved cameras bit for bit
    assert 3 in ever and float(poses.omega[3].abs().sum()) == 0.0
    for c in range(C_):
        want = view_table(base_ikr[c], poses.omega[c])
        want_o = (base_org[c].double() + poses.tau[c]).float()
        assert _ulp_close(loader.all_inverse_krs[c], want) and torch.equal(loader.all_camera_origins[c], want_o), c
        if c not in ever or c == 3:
            assert torch.equal(loader.all_inverse_krs[c], base_ikr[c]) and torch.equal(loader.all_camera_origins[c], base_org[c])
    assert any(not torch.equal(loader.all_inverse_krs[c], base_ikr[c]) for c in ever)
    for s, c in enumerate(slot_cams):
        if c < 0:
            assert (loader.inverse_krs_cuda[s] == 7.0).all() and (loader.camera_origins_cuda[s] == 7.0).all()
        else:
            assert torch.equal(loader.inverse_krs_cuda[s], loader.all_inverse_krs[c])
            assert torch.equal(loader.camera_origins_cuda[s], loader.all_camera_origins[c])


def test_pose_step_skipped_after_bad_camera_number(cuda):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    loader = _fake_loader(cuda, 4, [0, 1])
    poses = CameraPoses(loader)
    rng = np.random.default_rng(0)
    g_o, g_d, d, cams = _rays(100, 4, rng)
    cams[7] = 9
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
    poses.accumulate(dev(g_o), dev(g_d), dev(d), dev(cams), 100)
    poses.step(0)
    assert int(poses.steps.sum()) == 0 and float(poses.omega.abs().sum()) == 0.0
    with pytest.raises(RuntimeError, match="outside"):
        poses.check()


# ------------------------------------------------------------------------------------------------ end to end
def test_train_step_pose_gradient_matches_autograd(cuda):
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, rotation_increment
    from humanrf_b200.training import FusedTrainer
    from humanrf_b200.utils.loss import bce_loss
    from humanrf_b200.volume_rendering import render

    om, m, frames = make_pair((6,), table_std=1.0, device=cuda)
    R, C_, step = 256, 4, 4e-3
    b = synthetic_rays(R, 48, frames, seed=11, ragged=True, step=step)
    rng = np.random.default_rng(11)
    cams = torch.from_numpy(rng.integers(0, C_, R).astype(np.int32))
    o, d, t, ri, fr = (b[k].to(cuda).contiguous() for k in ("o", "d", "t", "ri", "frames"))
    rgba = b["rgba"].to(cuda).contiguous()
    bg = torch.rand((R, 3), generator=torch.Generator().manual_seed(3)).to(cuda)
    w0 = np.zeros((C_, 3))
    w0[1:] = rng.standard_normal((3, 3)) * np.array([[0.02], [0.3], [1.5]])
    # autograd: o = o_r + tau, d = exp([w]x) exp(-[w0]x) d_r, Huber + 1e-3 BCE.  d is written d_r + (rot - I) d_r: at
    # w = w0 the increment is ~1e-16 and d rounds to d_r bit for bit, so both routes sample the same positions (a
    # near-empty ray's BCE gradient, ~1 / weights_sum, turns a 1-ulp change of a direction into a visible one).
    w = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    tau = torch.zeros((C_, 3), dtype=torch.float64, requires_grad=True)
    rot = torch.stack([rotation_increment(w[c]) @ rotation_increment(-torch.from_numpy(w0[c])) - torch.eye(3, dtype=torch.float64)
                       for c in range(C_)])
    cl = cams.long()
    dd = (d.double() + (rot.to(cuda)[cl] @ d.double()[:, :, None])[:, :, 0]).float()
    assert torch.equal(dd, d)
    oo = (o.double() + tau.to(cuda)[cl]).float()
    ib = InputBatch(ray_origins=oo, ray_directions=dd, frame_numbers=fr.view(-1, 1), sample_distances=t.view(-1, 1),
                    ray_indices=ri, unique_frame_numbers=torch.unique(fr).view(-1, 1))
    # mask targets from the model's own opacity: a ray whose weights sum is ~0 against a mask of 1 (or ~1 against 0) gets
    # a BCE gradient ~1 / (1 - |mask - weights_sum|) that dwarfs every other ray and leaves the per-camera sums to cancel
    with torch.no_grad():
        rgba[:, 3] = (render(ib, m, bg, is_training=False, render_step_size=step).weights_sum[:, 0] > 0.5).float()
    out = render(ib, m, bg, is_training=True, render_step_size=step)
    mask = rgba[:, 3:]
    gt = rgba[:, :3] * mask + bg * (1 - mask)
    loss = torch.nn.HuberLoss(delta=0.01)(out.color, gt) + 1e-3 * bce_loss(out.weights_sum, mask).mean()
    loss.backward()
    ref = torch.cat((w.grad, tau.grad), 1).numpy()
    for q in m.hot_parameters():
        q.grad = None
    # the fused step with the same rays (d_r = exp([w0]x) d0 as sampled)
    loader = _fake_loader(cuda, C_, [0, 1])
    poses = CameraPoses(loader, fixed_cameras=(0,))
    poses.omega.copy_(torch.from_numpy(w0))
    tr = FusedTrainer(m, prune=False, render_step_size=step, camera_poses=poses)
    tr.step(o, d, fr, t, ri, rgba, R, background=bg, cameras=cams.to(cuda))
    got = poses.pose_grad.double().cpu().numpy()
    assert np.array_equal(poses.ray_count.cpu().numpy(), np.bincount(cams.numpy(), minlength=C_))
    for c in range(C_):
        rel = np.linalg.norm(got[c] - ref[c]) / np.linalg.norm(ref[c])
        print(f"camera {c}: |omega0| {np.linalg.norm(w0[c]):.3f}, |grad| {np.linalg.norm(ref[c]):.3e}, norm-wise rel {rel:.3e}")
        assert np.linalg.norm(ref[c]) > 0 and rel < 1e-3, c
    assert float(poses.omega[1:].sub(torch.from_numpy(w0[1:]).to(cuda)).abs().min()) > 0      # the step moved them
    assert torch.equal(poses.omega[0], torch.zeros(3, dtype=torch.float64, device=cuda))


# ------------------------------------------------------------------------------------------------ default path
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


def _step_kernel_names():
    """Kernel names of one FusedTrainer step after two warm steps: without camera_poses, with camera_poses before its
    start step, and with camera_poses from step 0.  Also the pose step counters of the late-start poses."""
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.training import FusedTrainer

    cuda = torch.device("cuda:0")
    R = 4096
    b = synthetic_rays(R, 32, list(range(15, 21)), seed=4)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba", "cams")}
    cams = (g["cams"] % 8).contiguous()

    def names(poses):
        m, _ = make_model((6,), seed=1, device=cuda)
        tr = FusedTrainer(m, camera_poses=poses)
        for _ in range(2):
            tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams)
        return _kernel_names(lambda: tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams))

    late = CameraPoses(_fake_loader(cuda, 8, [0, 1]), start_step=1000)
    out = {"plain": names(None), "late": names(late)}
    out["late_steps"] = int(late.steps.sum())
    out["early"] = names(CameraPoses(_fake_loader(cuda, 8, [0, 1]), start_step=0))
    return out


def _in_child(fn_name):
    """Runs this module's fn_name() in a fresh Python process and returns its JSON result.  The profiler sessions stay out
    of the test process: once CUPTI has been started in a process, a later profiler session there can miss kernels, and
    other test files profile their own launches."""
    import json
    import subprocess
    import sys
    from pathlib import Path

    here = Path(__file__).resolve().parent
    code = (f"import json, sys; sys.path[:0] = [{str(here)!r}, {str(here.parent)!r}]; import {Path(__file__).stem} as T; "
            f"print('RESULT ' + json.dumps(T.{fn_name}()))")
    flags = (["-s"] if sys.flags.no_user_site else []) + (["-E"] if sys.flags.ignore_environment else [])
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600,
                       cwd=str(here.parent))
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(lines[-1][len("RESULT "):])


# The library's kernels of one default FusedTrainer step (one segment, prune, reuse="feat"), in launch order, as
# recorded before pose refinement existed.
DEFAULT_STEP_KERNELS = [
    "hrf::ray_offsets_kernel(long const*, long, long, int*)",
    "hrf::ray_max_chunks_kernel(int const*, long, int*)",
    "void hrf::field_forward_kernel<false, 5, false, 1, false, false, false>(hrf::FieldArgs)",
    "hrf::visibility_kernel(float const*, int const*, long, float, float, float, unsigned char*, int*)",
    "hrf::scan_i32_kernel(int const*, long, int*, long*)",
    "hrf::prune_compact_kernel(unsigned char const*, float const*, int const*, int const*, long, float*, long*, int*)",
    "void hrf::field_forward_kernel<false, 5, false, 1, true, false, false>(hrf::FieldArgs)",
    "hrf::composite_fwd_kernel(float const*, float const*, float const*, int const*, long, float, float const*, float*, float*, "
    "float*)",
    "hrf::train_loss_kernel(float const*, float const*, float const*, float const*, long, float, float, float const*, float*, "
    "float*, float*)",
    "hrf::composite_bwd_kernel(float const*, float const*, float const*, int const*, long, float, float const*, float const*, "
    "float const*, float*, float*)",
    "void hrf::field_backward_kernel<4, false>(hrf::BwdArgs)",
    "void hrf::grid_scatter_v6_kernel<true>(hrf::ScatterV5Args)",
    "hrf::adam_steps_kernel(hrf_adam_tensor const*, int)",
    "hrf::adam_multi_kernel(hrf_adam_tensor const*, int, float, float, float, float, float, int)",
]


def _ours(names):
    return [n for n in names if "hrf::" in n]


def test_default_step_unchanged(cuda):
    res = _in_child("_step_kernel_names")
    plain, late, early = res["plain"], res["late"], res["early"]
    assert _ours(plain) == DEFAULT_STEP_KERNELS
    assert late == plain
    assert res["late_steps"] == 0
    extra = [n for n in _ours(early) if n not in _ours(plain)]
    assert any("position_grad" in n for n in extra) and any("ray_gradients" in n for n in extra)
    assert any("pose_partials" in n for n in extra) and any("pose_step" in n for n in extra)


# ------------------------------------------------------------------------------------------------ recovery
class _TeacherDataset:
    """A SyntheticDataset whose images are a teacher's renders at the true poses (BGR, as the dataset gives them) and
    whose masks are the renders' alpha > 0.5; its cameras may be perturbed."""

    def __init__(self, base, images, masks):
        self.base, self.images, self.masks = base, images, masks
        self.cameras, self.frames = base.cameras, base.frames

    def get_aabb(self, frame_numbers=None):
        return self.base.get_aabb()

    def get_scaled_cameras(self, scene_offset, scene_scale):
        return self.base.get_scaled_cameras(scene_offset, scene_scale)

    def get_rgb(self, camera_number, frame_number, normalize=True):
        return self.images[(camera_number, frame_number)][..., ::-1].copy()

    def get_mask(self, camera_number, frame_number, normalize=True):
        return self.masks[(camera_number, frame_number)]

    def get_occupancy_grid(self, frame_number):
        return self.base.get_occupancy_grid(frame_number)


def _scene8():
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from test_ray_grad_gpu import _sphere

    ds = SyntheticDataset(num_cameras=8, width=256, height=192, G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    return ds


def test_joint_training_recovers_perturbed_cameras(cuda):
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, axisangle_of
    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.training import FusedTrainer
    from test_ray_grad_gpu import _centre_shift, _rot_err, textured_teacher

    m = textured_teacher(cuda)
    base = _scene8()
    frame, n_cams = 16, 8
    view = DL(dataset=base, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192,
              camera_numbers=tuple(range(n_cams)), frame_numbers=tuple(base.frames), max_buffer_size=1,
              render_sequence=[(0, frame)])
    images, masks = {}, {}
    for c in range(n_cams):
        dm = render_depth_map(m, view, c, frame)
        images[(c, frame)] = dm.color.cpu().numpy()
        masks[(c, frame)] = (dm.alpha.cpu().numpy() > 0.5).astype(np.float32).reshape(192, 256, 1)
        assert 0.02 < masks[(c, frame)].mean() < 0.9
    pert = _scene8()
    perturbed = (1, 3, 6)
    init = {}
    for k, c in enumerate(perturbed):
        cam = base.cameras[c]
        R = rotation_from_axisangle(cam.rotation_axisangle)
        a = 0.6 + 0.3 * k
        rot_p = axisangle_of(rotation_from_axisangle(0.012 * (R[:, 0] * np.cos(a) + R[:, 1] * np.sin(a))) @ R)
        tr = 0.035 * (R[:, 0] * np.sin(a) - R[:, 1] * np.cos(a)) + 0.02 * R[:, 2]
        depth = float(np.linalg.norm(cam.translation - base.aabb.mean(0)))
        s_rot = _centre_shift(cam, rot_p, cam.translation, depth)
        s_tr = _centre_shift(cam, cam.rotation_axisangle, cam.translation + tr, depth)
        assert s_rot >= 1.0 and s_tr >= 1.0, (c, s_rot, s_tr)
        pert.cameras[c].rotation_axisangle = rot_p
        pert.cameras[c].translation = cam.translation + tr
        init[c] = (_rot_err(rot_p, cam.rotation_axisangle), float(np.linalg.norm(tr)), s_rot, s_tr)
    torch.manual_seed(0)
    np.random.seed(0)
    loader = DL(dataset=_TeacherDataset(pert, images, masks), device="cuda", mode=DL.Mode.TRAINING,
                dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=STEPS_BATCH,
                camera_numbers=tuple(range(n_cams)), frame_numbers=(frame,), max_buffer_size=n_cams,
                max_num_frames_per_batch=1, use_mask=True, filter_light_bloom=False)
    anchor_ikr, anchor_org = loader.all_inverse_krs[0].clone(), loader.all_camera_origins[0].clone()
    for q in m.parameters():
        q.requires_grad_(True)
    poses = CameraPoses(loader, lr=POSE_LR, final_lr_ratio=1e-2, max_steps=STEPS)
    assert poses.fixed_cameras == (0,)
    trainer = FusedTrainer(m, lr=FIELD_LR, max_steps=STEPS, camera_poses=poses)
    for _ in range(STEPS):
        ib = next(loader)
        trainer.step(ib.ray_origins.contiguous(), ib.ray_directions.contiguous(), ib.frame_numbers.view(-1).contiguous(),
                     ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous(), ib.rgba.contiguous(),
                     ib.num_rays, cameras=ib.camera_numbers.view(-1).to(torch.int32).contiguous())
    poses.check()
    refined = poses.refined_cameras()
    assert torch.equal(loader.all_inverse_krs[0], anchor_ikr) and torch.equal(loader.all_camera_origins[0], anchor_org)
    ok = True
    for c in range(1, n_cams):
        cam = base.cameras[c]
        e_rot = _rot_err(refined[c].rotation_axisangle, cam.rotation_axisangle)
        e_tr = float(np.linalg.norm(refined[c].translation - cam.translation))
        depth = float(np.linalg.norm(cam.translation - base.aabb.mean(0)))
        shift = _centre_shift(cam, refined[c].rotation_axisangle, refined[c].translation, depth)
        if c in perturbed:
            r0, t0, s_rot, s_tr = init[c]
            print(f"camera {c}: perturbed {s_rot:.2f} px / {s_tr:.2f} px; rotation error {r0:.3e} -> {e_rot:.3e} "
                  f"({e_rot / r0:.3f}), translation error {t0:.3e} -> {e_tr:.3e} ({e_tr / t0:.3f}), centre shift {shift:.3f} px")
            ok &= e_rot < 0.25 * r0 and e_tr < 0.25 * t0
        else:
            print(f"camera {c}: unperturbed, centre shift {shift:.4f} px")
            ok &= shift <= 0.1
    assert ok


STEPS, STEPS_BATCH, POSE_LR, FIELD_LR = 2000, 32768, 5e-3, 3e-5
