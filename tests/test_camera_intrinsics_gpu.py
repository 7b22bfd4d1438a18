"""Per-camera intrinsics refinement in the fused train step on the H100: hrf_camera_calib_grad and hrf_camera_calib_step
against tests/intrinsics_oracle.py, torch and the pose-only kernels, one FusedTrainer step against render() under
autograd, the step's kernel list, and recovery of perturbed focal lengths and principal points.

Bars:
* gradient: (n + 12) 2^-23 sum|terms| per entry against the float64 sums of the kernel's own inputs; the pose columns
  bit-identical to hrf_camera_pose_grad's.
* step: parameters and moments to 1e-6 relative of torch.optim.Adam with two parameter groups, run on the touched
  cameras only; tables within 1 fp32 ulp of the float64 table; at alpha = beta = 0 bit-identical to the pose-only step.
* end to end: 1e-3 norm-wise per camera, the pose test's bar.
* recovery: RMS reprojection error over points inside the teacher's blobs, perturbed cameras to <= 25 % of their initial
  error, unperturbed cameras <= 0.15 px (measured 0.074-0.104 px on an H100 80GB HBM3, 700 W: the intrinsics' extra
  freedom lets the field and the free cameras settle slightly off the truth), the anchor camera's tables bit for bit.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import intrinsics_oracle as IO
import pose_oracle as PO
from helpers import make_pair, synthetic_rays
from test_camera_poses_gpu import _kernel_names, _rays, _TeacherDataset, _scene8

pytestmark = pytest.mark.gpu


def _dev(cuda):
    return lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _random_rotations(C_, rng):
    return np.stack([PO.so3_exp(rng.standard_normal(3) * rng.uniform(0, 3)) for _ in range(C_)]).astype(np.float32)


@pytest.mark.parametrize("C_", [1, 8, 160])
@pytest.mark.parametrize("R", [1, 31, 4096, 300000])
def test_calib_grad_kernel(cuda, R, C_):
    from humanrf_b200.toolbox.camera_refinement import calibration_gradients, pose_gradients

    rng = np.random.default_rng(R * 11 + C_)
    cams = None
    if C_ > 1:      # only the even cameras have rays
        cams = (2 * rng.integers(0, (C_ + 1) // 2, R)).astype(np.int32)
    omega = rng.standard_normal((C_, 3)) * rng.choice([0.0, 1e-3, 0.4, 2.0], (C_, 1))
    alpha = rng.standard_normal((C_, 2)) * rng.choice([0.0, 0.05], (C_, 1))
    rot = _random_rotations(C_, rng)
    g_o, g_d, d, cams = _rays(R, C_, rng, cams)
    dev = _dev(cuda)
    args = (dev(g_o), dev(g_d), dev(d), dev(cams), dev(omega), dev(alpha), dev(rot))
    pg, ig, cnt = calibration_gradients(*args)
    pg2, ig2, cnt2 = calibration_gradients(*args)
    assert torch.equal(pg, pg2) and torch.equal(ig, ig2) and torch.equal(cnt, cnt2)      # bit for bit
    pp, pc = pose_gradients(*args[:5])
    assert torch.equal(pg.view(torch.int32), pp.view(torch.int32)) and torch.equal(cnt, pc)
    ref, n, bound = IO.intrinsics_grad(g_d, d, cams, alpha, rot)
    got = ig.double().cpu().numpy()
    assert np.array_equal(cnt.cpu().numpy(), n) and n.sum() == R
    err = np.abs(got - ref)
    assert (err <= bound).all(), f"max err/bound {(err / np.maximum(bound, 1e-300)).max():.3e}"
    assert (got[n == 0] == 0).all()
    if C_ > 1:
        assert (n[1::2] == 0).all()


def test_calib_grad_kernel_rejects_camera_outside_range(cuda):
    from humanrf_b200.toolbox.camera_refinement import calibration_gradients

    rng = np.random.default_rng(2)
    dev = _dev(cuda)
    for bad in (8, -2):
        g_o, g_d, d, cams = _rays(5000, 8, rng)
        cams[777] = bad
        with pytest.raises(RuntimeError, match="outside"):
            calibration_gradients(dev(g_o), dev(g_d), dev(d), dev(cams), torch.zeros((8, 3), dtype=torch.float64, device=cuda),
                                  torch.zeros((8, 2), dtype=torch.float64, device=cuda), dev(_random_rotations(8, rng)))
    torch.cuda.synchronize()         # the context is healthy


def _loader_with_cameras(cuda, C_, slot_cams):
    """The tables CameraPoses reads and writes, as a DataLoader holds them on the device, and its cameras."""
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(num_cameras=C_, width=96, height=72)
    ld = DL(dataset=ds, device="cpu", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS,
            space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=64, camera_numbers=tuple(range(C_)),
            frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])
    B = len(slot_cams)
    return SimpleNamespace(all_inverse_krs=ld.all_inverse_krs.to(cuda).contiguous(),
                           all_camera_origins=ld.all_camera_origins.to(cuda).contiguous(), camera_numbers=tuple(range(C_)),
                           inverse_krs_cuda=torch.full((B, 3, 3), 7.0, device=cuda),
                           camera_origins_cuda=torch.full((B, 3), 7.0, device=cuda),
                           camera_numbers_cuda=torch.tensor(slot_cams, dtype=torch.int32, device=cuda),
                           cameras=ld.cameras, scene_scale=ld.scene_scale, scene_offset=ld.scene_offset)


def test_calib_step_kernel(cuda):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    C_, lr, lr_i = 8, 3e-3, 1e-3
    slot_cams = [3, -1, 0, 5, 5, -1, 7, 2, 1, 6, -1, 4]
    loader = _loader_with_cameras(cuda, C_, slot_cams)
    poses = CameraPoses(loader, lr=lr, final_lr_ratio=1.0, fixed_cameras=(0,), intrinsics=True, intrinsics_lr=lr_i)
    # the pose-only step on a copy of the tables, fed the same pose gradients: equal tables while alpha = beta = 0
    loader_p = _loader_with_cameras(cuda, C_, slot_cams)
    pose_only = CameraPoses(loader_p, lr=lr, final_lr_ratio=1.0, fixed_cameras=(0,))
    base_ikr, base_org = loader.all_inverse_krs.clone(), loader.all_camera_origins.clone()
    ref = [(torch.zeros(6, dtype=torch.float64, requires_grad=True), torch.zeros(4, dtype=torch.float64, requires_grad=True))
           for _ in range(C_)]
    opts = [torch.optim.Adam([{"params": [p], "lr": lr}, {"params": [q], "lr": lr_i}], betas=(0.9, 0.99), eps=1e-15)
            for p, q in ref]
    rng = np.random.default_rng(4)
    touched_sets = [[0, 1, 2, 3], [2, 3, 6], [1, 2, 3, 4, 6], [6], [0, 2, 3, 6]]
    names = ("omega", "tau", "exp_avg", "exp_avg_sq", "steps", "alpha", "beta", "intrinsics_exp_avg",
             "intrinsics_exp_avg_sq", "rotations")
    for k, touched in enumerate(touched_sets):
        count = np.zeros(C_, np.int32)
        count[touched] = rng.integers(1, 1000, len(touched))
        g = (rng.standard_normal((C_, 6)) * 10.0 ** rng.uniform(-4, 1, (C_, 1))).astype(np.float32)
        gi = (rng.standard_normal((C_, 4)) * 10.0 ** rng.uniform(-4, 1, (C_, 1))).astype(np.float32)
        gi[2] = 0.0                   # camera 2: intrinsics without gradient stay at zero, its pose moves
        for p_ in (poses, pose_only):
            p_.pose_grad.copy_(torch.from_numpy(g))
            p_.ray_count.copy_(torch.from_numpy(count))
        poses.intrinsics_grad.copy_(torch.from_numpy(gi))
        before = {n: getattr(poses, n).clone() for n in names}
        tab_before = (loader.all_inverse_krs.clone(), loader.all_camera_origins.clone())
        poses.step(k)
        pose_only.step(k)
        torch.cuda.synchronize()
        for c in touched:
            if c != 0:
                opts[c].zero_grad()
                ref[c][0].grad = torch.from_numpy(g[c].astype(np.float64))
                ref[c][1].grad = torch.from_numpy(gi[c].astype(np.float64))
                opts[c].step()
        for c in range(C_):
            if c in touched and c != 0:
                continue
            for n, v in before.items():                       # untouched and fixed: bit-unchanged
                assert torch.equal(getattr(poses, n)[c], v[c]), (k, c, n)
            assert torch.equal(loader.all_inverse_krs[c], tab_before[0][c])
            assert torch.equal(loader.all_camera_origins[c], tab_before[1][c])
        # camera 2 (alpha = beta = 0, pose moved): the pose-only step's table bit for bit
        assert float(poses.alpha[2].abs().sum() + poses.beta[2].abs().sum()) == 0.0
        assert torch.equal(loader.all_inverse_krs[2].view(torch.int32), loader_p.all_inverse_krs[2].view(torch.int32))
        assert torch.equal(loader.all_camera_origins, loader_p.all_camera_origins)
    params = torch.cat((poses.omega, poses.tau, poses.alpha, poses.beta), 1).cpu()
    moments = (torch.cat((poses.exp_avg, poses.intrinsics_exp_avg), 1).cpu(),
               torch.cat((poses.exp_avg_sq, poses.intrinsics_exp_avg_sq), 1).cpu())
    for c in range(C_):
        r = torch.cat([p.detach() for p in ref[c]])
        assert torch.allclose(params[c], r, rtol=1e-6, atol=1e-12), c
        sts = [opts[c].state.get(p) for p in ref[c]]
        if sts[0]:
            assert torch.allclose(moments[0][c], torch.cat([s["exp_avg"] for s in sts]), rtol=1e-6, atol=1e-30)
            assert torch.allclose(moments[1][c], torch.cat([s["exp_avg_sq"] for s in sts]), rtol=1e-6, atol=1e-30)
            assert int(poses.steps[c]) == int(sts[0]["step"])
        else:
            assert int(poses.steps[c]) == 0
    moved = 0
    for c in range(C_):
        K = poses.base_intrinsics[c].tolist()
        want = IO.calibration_table(base_ikr[c].cpu().numpy(), poses.omega[c].cpu().numpy(), poses.alpha[c].cpu().numpy(),
                                    poses.beta[c].cpu().numpy(), K)
        got = loader.all_inverse_krs[c].cpu().numpy().astype(np.float64)
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all(), c
        want_o = (base_org[c].double() + poses.tau[c]).float()
        assert torch.equal(loader.all_camera_origins[c], want_o)
        rot = (PO.so3_exp(poses.omega[c].cpu().numpy()) @ poses.base_rotations[c].cpu().numpy())
        assert np.abs(poses.rotations[c].cpu().numpy() - rot).max() <= 2.0 ** -23
        moved += int(float(poses.alpha[c].abs().sum()) > 0)
        if int(poses.steps[c]) == 0:
            assert torch.equal(loader.all_inverse_krs[c], base_ikr[c]) and torch.equal(loader.all_camera_origins[c], base_org[c])
    assert moved >= 4
    for s, c in enumerate(slot_cams):
        if c < 0:
            assert (loader.inverse_krs_cuda[s] == 7.0).all() and (loader.camera_origins_cuda[s] == 7.0).all()
        else:
            assert torch.equal(loader.inverse_krs_cuda[s], loader.all_inverse_krs[c])
            assert torch.equal(loader.camera_origins_cuda[s], loader.all_camera_origins[c])


def test_calib_step_skipped_after_bad_camera_number(cuda):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    poses = CameraPoses(_loader_with_cameras(cuda, 4, [0, 1]), intrinsics=True)
    rng = np.random.default_rng(0)
    g_o, g_d, d, cams = _rays(100, 4, rng)
    cams[7] = 9
    dev = _dev(cuda)
    poses.accumulate(dev(g_o), dev(g_d), dev(d), dev(cams), 100)
    poses.step(0)
    assert int(poses.steps.sum()) == 0 and float(poses.alpha.abs().sum() + poses.omega.abs().sum()) == 0.0
    with pytest.raises(RuntimeError, match="outside"):
        poses.check()


# ------------------------------------------------------------------------------------------------ end to end
def test_train_step_intrinsics_gradient_matches_autograd(cuda):
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, rotation_increment
    from humanrf_b200.training import FusedTrainer
    from humanrf_b200.utils.loss import bce_loss
    from humanrf_b200.volume_rendering import render

    om, m, frames = make_pair((6,), table_std=1.0, device=cuda)
    R, C_, step = 256, 4, 4e-3
    b = synthetic_rays(R, 48, frames, seed=11, ragged=True, step=step)
    rng = np.random.default_rng(12)
    cams = torch.from_numpy(rng.integers(0, C_, R).astype(np.int32))
    o, d, t, ri, fr = (b[k].to(cuda).contiguous() for k in ("o", "d", "t", "ri", "frames"))
    rgba = b["rgba"].to(cuda).contiguous()
    bg = torch.rand((R, 3), generator=torch.Generator().manual_seed(3)).to(cuda)
    loader = _loader_with_cameras(cuda, C_, [0, 1])
    poses = CameraPoses(loader, fixed_cameras=(0,), intrinsics=True)
    w0 = np.zeros((C_, 3))
    w0[1:] = rng.standard_normal((3, 3)) * np.array([[0.02], [0.3], [1.5]])
    a0 = rng.standard_normal((C_, 2)) * 0.04
    b0 = rng.standard_normal((C_, 2)) * 0.02
    with torch.no_grad():
        poses.omega.copy_(torch.from_numpy(w0))
        poses.alpha.copy_(torch.from_numpy(a0))
        poses.beta.copy_(torch.from_numpy(b0))
        poses.rotations.copy_(poses.current_rotations())
    Rp = poses.rotations.double().cpu()                          # R'_c as the kernel reads it
    # autograd: a ray of camera c is u' = R'^T d_r / (R'^T d_r)_z in camera coordinates, u0 = A(a0, b0)^-1 u' its base
    # coordinates; d = normalize(exp([w]x) exp(-[w0]x) R' A(a, b) u0) and o = o_r + tau.  Written d_r + (f - f.detach())
    # so that d equals d_r bit for bit (both routes sample the same positions) while the gradient is f's.
    w = torch.tensor(w0, requires_grad=True)
    tau = torch.zeros((C_, 3), dtype=torch.float64, requires_grad=True)
    a = torch.tensor(a0, requires_grad=True)
    bb = torch.tensor(b0, requires_grad=True)
    cl = cams.long()
    dr = d.double().cpu()
    q = torch.einsum("rij,ri->rj", Rp[cl], dr)
    u = q / q[:, 2:3]
    x0 = u[:, 0] * torch.exp(torch.from_numpy(a0[:, 0]))[cl] + torch.from_numpy(b0[:, 0])[cl]
    y0 = u[:, 1] * torch.exp(torch.from_numpy(a0[:, 1]))[cl] + torch.from_numpy(b0[:, 1])[cl]
    up = torch.stack([(x0 - bb[cl, 0]) * torch.exp(-a[cl, 0]), (y0 - bb[cl, 1]) * torch.exp(-a[cl, 1]), torch.ones_like(x0)], 1)
    rot = torch.stack([rotation_increment(w[c]) @ rotation_increment(-torch.from_numpy(w0[c])) @ Rp[c] for c in range(C_)])
    v = torch.einsum("rij,rj->ri", rot[cl], up)
    # a ray behind its camera (q_z < 0) is -R' u' / |u'|; the kernel's q_z h covers both signs
    f = torch.sign(q[:, 2:3]) * v / torch.linalg.vector_norm(v, dim=1, keepdim=True)
    dd = (dr + (f - f.detach())).float().to(cuda)
    assert torch.equal(dd, d)
    oo = (o.double() + tau.to(cuda)[cl.to(cuda)]).float()
    ib = InputBatch(ray_origins=oo, ray_directions=dd, frame_numbers=fr.view(-1, 1), sample_distances=t.view(-1, 1),
                    ray_indices=ri, unique_frame_numbers=torch.unique(fr).view(-1, 1))
    with torch.no_grad():
        rgba[:, 3] = (render(ib, m, bg, is_training=False, render_step_size=step).weights_sum[:, 0] > 0.5).float()
    out = render(ib, m, bg, is_training=True, render_step_size=step)
    mask = rgba[:, 3:]
    gt = rgba[:, :3] * mask + bg * (1 - mask)
    loss = torch.nn.HuberLoss(delta=0.01)(out.color, gt) + 1e-3 * bce_loss(out.weights_sum, mask).mean()
    loss.backward()
    ref = torch.cat((w.grad, tau.grad, a.grad, bb.grad), 1).numpy()
    for p_ in m.hot_parameters():
        p_.grad = None
    tr = FusedTrainer(m, prune=False, render_step_size=step, camera_poses=poses)
    tr.step(o, d, fr, t, ri, rgba, R, background=bg, cameras=cams.to(cuda))
    got = torch.cat((poses.pose_grad, poses.intrinsics_grad), 1).double().cpu().numpy()
    assert np.array_equal(poses.ray_count.cpu().numpy(), np.bincount(cams.numpy(), minlength=C_))
    for c in range(C_):
        rel = np.linalg.norm(got[c] - ref[c]) / np.linalg.norm(ref[c])
        rel_i = np.linalg.norm(got[c, 6:] - ref[c, 6:]) / np.linalg.norm(ref[c, 6:])
        print(f"camera {c}: |grad| {np.linalg.norm(ref[c]):.3e}, norm-wise rel {rel:.3e}, intrinsics alone {rel_i:.3e}")
        assert np.linalg.norm(ref[c, 6:]) > 0 and rel < 1e-3 and rel_i < 1e-3, c
    assert float(poses.alpha[1:].sub(torch.from_numpy(a0[1:]).to(cuda)).abs().min()) > 0      # the step moved them
    assert torch.equal(poses.alpha[0], torch.from_numpy(a0[0]).to(cuda))


# ------------------------------------------------------------------------------------------------ kernel list
def _step_kernel_lists():
    """Kernel names of one FusedTrainer step after two warm steps, with pose-only and with intrinsics refinement."""
    from humanrf_b200.synthetic import make_model
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.training import FusedTrainer

    cuda = torch.device("cuda:0")
    R = 4096
    b = synthetic_rays(R, 32, list(range(15, 21)), seed=4)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba", "cams")}
    cams = (g["cams"] % 8).contiguous()

    def names(intrinsics):
        m, _ = make_model((6,), seed=1, device=cuda)
        tr = FusedTrainer(m, camera_poses=CameraPoses(_loader_with_cameras(cuda, 8, [0, 1]), intrinsics=intrinsics))
        for _ in range(2):
            tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams)
        return _kernel_names(lambda: tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], R, cameras=cams))

    return {"pose": names(False), "calib": names(True)}


def _in_child(fn_name):
    """This module's fn_name() in a fresh Python process (the profiler stays out of the test process), its JSON result."""
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


def test_intrinsics_step_replaces_only_the_pose_kernels(cuda):
    res = _in_child("_step_kernel_lists")
    ours = lambda names: [n for n in names if "hrf::" in n]    # noqa: E731
    pose, calib = ours(res["pose"]), ours(res["calib"])
    swap = {"pose_partials_kernel": "calib_partials_kernel", "pose_finish_kernel": "calib_finish_kernel",
            "pose_step_kernel": "calib_step_kernel"}
    assert len(pose) == len(calib)
    replaced = 0
    for p_, c_ in zip(pose, calib):
        key = next((k for k in swap if k in p_), None)
        if key is None:
            assert p_ == c_
        else:
            assert swap[key] in c_, (p_, c_)
            replaced += 1
    assert replaced == 3


# ------------------------------------------------------------------------------------------------ recovery
_BLOBS = (((0.0, 0.0, 0.0), (0.12, 0.16, 0.1)), ((0.24, 0.08, 0.1), (0.08, 0.1, 0.08)),
          ((-0.22, -0.1, 0.12), (0.1, 0.08, 0.08)), ((0.05, -0.15, -0.25), (0.09, 0.08, 0.1)),
          ((-0.1, 0.2, -0.2), (0.08, 0.08, 0.09)))      # textured_teacher's blobs, normalised scene units


def _blob_points(loader, n=2000, seed=0):
    """World points inside the teacher's blobs (seeded)."""
    rng = np.random.default_rng(seed)
    pts = []
    for k in range(n):
        c, r = _BLOBS[k % len(_BLOBS)]
        u = rng.standard_normal(3)
        u *= rng.uniform() ** (1 / 3) / np.linalg.norm(u)
        pts.append(np.asarray(c) + np.asarray(r) * u)
    return np.asarray(pts) / float(loader.scene_scale) - np.asarray(loader.scene_offset)


def _perturb_intrinsics(cam, k):
    s = np.array([1.03, 0.97]) if k % 2 == 0 else np.array([0.97, 1.03])
    cam.focal_length = np.asarray(cam.focal_length) * s
    a = 0.7 + 1.3 * k
    cam.principal_point = np.asarray(cam.principal_point) + 4.0 * np.array([np.cos(a) / cam.width, np.sin(a) / cam.height])


def _teacher_images(m, base, n_cams, frame):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.depth_maps import render_depth_map

    view = DL(dataset=base, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192,
              camera_numbers=tuple(range(n_cams)), frame_numbers=tuple(base.frames), max_buffer_size=1,
              render_sequence=[(0, frame)])
    images, masks = {}, {}
    for c in range(n_cams):
        dm = render_depth_map(m, view, c, frame)
        images[(c, frame)] = dm.color.cpu().numpy()
        masks[(c, frame)] = (dm.alpha.cpu().numpy() > 0.5).astype(np.float32).reshape(192, 256, 1)
    return images, masks


def _recover(cuda, with_pose):
    from humanrf_b200.dataset.cameras import rotation_from_axisangle
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, axisangle_of
    from humanrf_b200.training import FusedTrainer
    from test_ray_grad_gpu import textured_teacher

    m = textured_teacher(cuda)
    base = _scene8()
    frame, n_cams = 16, 8
    images, masks = _teacher_images(m, base, n_cams, frame)
    pert = _scene8()
    perturbed = (1, 3, 6)
    for k, c in enumerate(perturbed):
        _perturb_intrinsics(pert.cameras[c], k)
        if with_pose:            # the pose test's perturbation
            cam = base.cameras[c]
            R = rotation_from_axisangle(cam.rotation_axisangle)
            a = 0.6 + 0.3 * k
            pert.cameras[c].rotation_axisangle = axisangle_of(
                rotation_from_axisangle(0.012 * (R[:, 0] * np.cos(a) + R[:, 1] * np.sin(a))) @ R)
            pert.cameras[c].translation = cam.translation + 0.035 * (R[:, 0] * np.sin(a) - R[:, 1] * np.cos(a)) + 0.02 * R[:, 2]
    torch.manual_seed(0)
    np.random.seed(0)
    loader = DL(dataset=_TeacherDataset(pert, images, masks), device="cuda", mode=DL.Mode.TRAINING,
                dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=STEPS_BATCH,
                camera_numbers=tuple(range(n_cams)), frame_numbers=(frame,), max_buffer_size=n_cams,
                max_num_frames_per_batch=1, use_mask=True, filter_light_bloom=False)
    pts = _blob_points(loader)
    init = {c: IO.reprojection_rms(pts, pert.cameras[c], base.cameras[c]) for c in perturbed}
    anchor_ikr, anchor_org = loader.all_inverse_krs[0].clone(), loader.all_camera_origins[0].clone()
    for q in m.parameters():
        q.requires_grad_(True)
    steps = STEPS_POSE if with_pose else STEPS
    poses = CameraPoses(loader, lr=POSE_LR, final_lr_ratio=1e-2, max_steps=steps, intrinsics=True, intrinsics_lr=INTR_LR)
    trainer = FusedTrainer(m, lr=FIELD_LR, max_steps=steps, camera_poses=poses)
    for _ in range(steps):
        ib = next(loader)
        trainer.step(ib.ray_origins.contiguous(), ib.ray_directions.contiguous(), ib.frame_numbers.view(-1).contiguous(),
                     ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous(), ib.rgba.contiguous(),
                     ib.num_rays, cameras=ib.camera_numbers.view(-1).to(torch.int32).contiguous())
    poses.check()
    assert torch.equal(loader.all_inverse_krs[0], anchor_ikr) and torch.equal(loader.all_camera_origins[0], anchor_org)
    refined = poses.refined_cameras()
    ok = True
    for c in range(1, n_cams):
        e = IO.reprojection_rms(pts, refined[c], base.cameras[c])
        if c in perturbed:
            print(f"camera {c}: RMS reprojection error {init[c]:.3f} px -> {e:.3f} px ({e / init[c]:.3f}); "
                  f"alpha {poses.alpha[c].tolist()}, beta {poses.beta[c].tolist()}")
            ok &= e <= 0.25 * init[c]
        else:
            print(f"camera {c}: unperturbed, RMS reprojection error {e:.4f} px")
            ok &= e <= UNPERTURBED_PX
    assert ok


def test_joint_training_recovers_perturbed_intrinsics(cuda):
    _recover(cuda, with_pose=False)


def test_joint_training_recovers_perturbed_intrinsics_and_poses(cuda):
    _recover(cuda, with_pose=True)


def test_refine_camera_recovers_intrinsics(cuda):
    from test_ray_grad_gpu import _RenderedDataset, _loader, _scene, textured_teacher
    from humanrf_b200.toolbox.camera_refinement import refine_camera
    from humanrf_b200.toolbox.depth_maps import render_depth_map

    m = textured_teacher(cuda)
    base = _scene()
    cam_id, fr = 1, [16, 18]
    images = {}
    for f in fr:
        images[(cam_id, f)] = render_depth_map(m, _loader(base), cam_id, f).color.cpu().numpy()
    pert = _scene()
    _perturb_intrinsics(pert.cameras[cam_id], 0)
    loader_p = _loader(_RenderedDataset(pert, images))
    pts = _blob_points(loader_p)
    e0 = IO.reprojection_rms(pts, pert.cameras[cam_id], base.cameras[cam_id])
    res = refine_camera(m, loader_p, cam_id, fr, seed=3, intrinsics=True)
    got = SimpleNamespace(width=base.cameras[cam_id].width, height=base.cameras[cam_id].height,
                          rotation_axisangle=res.rotation_axisangle, translation=res.translation,
                          focal_length=res.focal_length, principal_point=res.principal_point)
    e = IO.reprojection_rms(pts, got, base.cameras[cam_id])
    print(f"RMS reprojection error {e0:.3f} px -> {e:.3f} px ({e / e0:.3f}); alpha {res.alpha}, beta {res.beta}, "
          f"loss {res.losses[0]:.3e} -> {res.losses[-1]:.3e}")
    assert e <= 0.1 * e0
    assert all(not q.requires_grad and q.grad is None for q in m.parameters())


STEPS, STEPS_POSE, STEPS_BATCH, POSE_LR, INTR_LR, FIELD_LR = 2000, 2000, 32768, 5e-3, 2e-3, 3e-5
UNPERTURBED_PX = 0.15
