"""Per-camera intrinsics refinement without a GPU: the float64 references of tests/intrinsics_oracle.py against torch
autograd and torch.optim.Adam, the refined sampler tables at and away from zero, CameraPoses(intrinsics=True)'s
calibration export against the loader's own table path, and its state."""
import copy
import csv

import numpy as np
import pytest
import torch

import intrinsics_oracle as IO
import pose_oracle as PO


def _camera(portrait: bool, seed: int):
    """(R camera-to-world, (fx0, fy0, cx0, cy0), W, H) of a look-at camera with an off-centre principal point."""
    from humanrf_b200.dataset.cameras import rotation_from_axisangle

    rng = np.random.default_rng(seed)
    W, H = (72, 96) if portrait else (96, 72)
    R = rotation_from_axisangle(rng.standard_normal(3))
    f = 1.77 * W * np.array([1.0, 1.02])
    c = np.array([W, H]) * (0.5 + 0.05 * rng.standard_normal(2))
    return R, np.array([f[0], f[1], c[0], c[1]]), W, H


@pytest.mark.parametrize("portrait", [False, True])
@pytest.mark.parametrize("theta", [0.0, 0.3, 2.5])
@pytest.mark.parametrize("ab", [0.0, 0.05, -0.05])
def test_intrinsics_gradient_matches_autograd(portrait, theta, ab):
    from humanrf_b200.toolbox.camera_refinement import intrinsics_matrix, rotation_increment

    R, K, W, H = _camera(portrait, seed=int(theta * 10) + 3 * portrait)
    rng = np.random.default_rng(7 + int(100 * ab))
    axis = rng.standard_normal(3)
    w0 = theta * axis / np.linalg.norm(axis)
    a0 = np.array([ab, -0.5 * ab])
    b0 = np.array([-ab, 0.7 * ab])
    K0inv = np.linalg.inv(np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1.0]]))
    M0 = torch.from_numpy(R @ K0inv)                   # exactly R K0^-1: the gradient's premise
    P = 300
    px = torch.from_numpy(rng.uniform(0, W, P))
    py = torch.from_numpy(rng.uniform(0, H, P))
    g = rng.standard_normal((P, 3)) * rng.uniform(0.1, 10, (P, 1))
    w = torch.tensor(w0, requires_grad=True)
    a = torch.tensor(a0, requires_grad=True)
    b = torch.tensor(b0, requires_grad=True)
    T = (rotation_increment(w) @ (M0 @ intrinsics_matrix(a, b, K))).T      # the sampler's formula, float64
    v = px[:, None] * T[0] + py[:, None] * T[1] + T[2]
    d = v / torch.linalg.vector_norm(v, dim=1, keepdim=True)
    ga, gb = torch.autograd.grad((d * torch.from_numpy(g)).sum(), (a, b))
    Rp = (rotation_increment(torch.from_numpy(w0)) @ torch.from_numpy(R)).numpy()
    got, n, _ = IO.intrinsics_grad(g, d.detach().numpy(), np.zeros(P, np.int64), a0[None], Rp[None])
    assert n[0] == P
    ref = torch.cat((ga, gb)).numpy()
    scale = np.abs(ref).max()
    np.testing.assert_allclose(got[0], ref, rtol=1e-10, atol=1e-10 * scale)
    assert scale > 0


def test_intrinsics_matrix_at_zero_is_identity():
    from humanrf_b200.toolbox.camera_refinement import intrinsics_matrix

    K = (170.0, 171.0, 48.3, 35.9)
    z = torch.zeros(2, dtype=torch.float64)
    assert torch.equal(intrinsics_matrix(z, z, K), torch.eye(3, dtype=torch.float64))
    assert np.array_equal(IO.intrinsics_matrix((0.0, 0.0), (0.0, 0.0), K), np.eye(3))
    a, b = np.array([0.03, -0.02]), np.array([0.01, 0.004])
    np.testing.assert_allclose(intrinsics_matrix(torch.from_numpy(a), torch.from_numpy(b), K).numpy(),
                               IO.intrinsics_matrix(a, b, K), rtol=1e-15, atol=1e-13)
    # R K0^-1 B = R K'^-1: the refined camera's K' = B^-1 K0 has fx0 e^ax, cx0 + fx0 bx
    K0 = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1.0]])
    K1 = np.linalg.inv(IO.intrinsics_matrix(a, b, K)) @ K0
    np.testing.assert_allclose(K1, [[K[0] * np.exp(a[0]), 0, K[2] + K[0] * b[0]],
                                    [0, K[1] * np.exp(a[1]), K[3] + K[1] * b[1]], [0, 0, 1]], rtol=1e-14, atol=1e-12)


def _cpu_loader(num_cameras=6):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(num_cameras=num_cameras, width=64, height=48)
    loader = DL(dataset=ds, device="cpu", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS,
                space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=64, camera_numbers=tuple(range(num_cameras)),
                frame_numbers=tuple(ds.frames), max_buffer_size=2, render_sequence=[(2, 15), (4, 16)])
    return ds, loader


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_tables_at_zero_and_pose_only():
    from humanrf_b200.toolbox.camera_refinement import CameraPoses, calibration_table, view_table

    _, loader = _cpu_loader()
    poses = CameraPoses(loader, intrinsics=True)
    ikr, org = poses.tables()
    assert torch.equal(_bits(ikr), _bits(loader.all_inverse_krs)) and torch.equal(org, loader.all_camera_origins)
    rng = np.random.default_rng(2)
    z = torch.zeros(2, dtype=torch.float64)
    for c in range(poses.num_cameras):
        for th in (0.0, 1e-3, 0.3, 2.5):
            w = torch.from_numpy(rng.standard_normal(3) * th)
            K = poses.base_intrinsics[c].tolist()
            got = calibration_table(poses.base_inverse_krs[c], w, z, z, K)
            assert torch.equal(_bits(got), _bits(view_table(poses.base_inverse_krs[c], w))), (c, th)
        # away from zero: the float64 reference, one rounding
        a, b = rng.standard_normal(2) * 0.05, rng.standard_normal(2) * 0.05
        got = calibration_table(poses.base_inverse_krs[c], w, torch.from_numpy(a), torch.from_numpy(b), K).numpy()
        want = IO.calibration_table(poses.base_inverse_krs[c].numpy(), w.numpy(), a, b, K)
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all()


def test_per_camera_adam_two_learning_rates():
    C, lr, lr_i = 5, 1e-2, 3e-3
    rng = np.random.default_rng(3)
    fixed = np.array([1, 0, 0, 0, 0], bool)
    st = dict(params=rng.standard_normal((C, 10)), m=np.zeros((C, 10)), v=np.zeros((C, 10)), steps=np.zeros(C, int))
    ref = [(torch.tensor(st["params"][c, :6], requires_grad=True), torch.tensor(st["params"][c, 6:], requires_grad=True))
           for c in range(C)]
    opts = [torch.optim.Adam([{"params": [p], "lr": lr}, {"params": [q], "lr": lr_i}], betas=(0.9, 0.99), eps=1e-15)
            for p, q in ref]
    for touched in ([0, 1, 2], [2, 3], [0, 1, 2, 3, 4], [4], [1, 2]):
        count = np.zeros(C, int)
        count[touched] = 7
        g = rng.standard_normal((C, 10)) * 10.0 ** rng.uniform(-3, 1, (C, 1))
        before = {k: v.copy() for k, v in st.items()}
        IO.adam(st, g, count, fixed, lr, lr_i)
        for c in range(C):
            if c in touched and not fixed[c]:
                opts[c].zero_grad()
                ref[c][0].grad, ref[c][1].grad = torch.from_numpy(g[c, :6].copy()), torch.from_numpy(g[c, 6:].copy())
                opts[c].step()
            else:
                for k in st:
                    assert np.array_equal(st[k][c], before[k][c]), (c, k)
    for c in range(C):
        want = torch.cat([p.detach() for p in ref[c]]).numpy()
        np.testing.assert_allclose(st["params"][c], want, rtol=1e-13, atol=1e-15)
    assert list(st["steps"]) == [0, 3, 4, 2, 2]


def _moved(poses, seed=5):
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        poses.omega.copy_(torch.from_numpy(rng.standard_normal(poses.omega.shape) * 1e-2))
        poses.tau.copy_(torch.from_numpy(rng.standard_normal(poses.tau.shape) * 1e-2))
        poses.alpha.copy_(torch.from_numpy(rng.standard_normal(poses.alpha.shape) * 3e-2))
        poses.beta.copy_(torch.from_numpy(rng.standard_normal(poses.beta.shape) * 1e-2))
    return poses


def _read_csv(path):
    with open(path, newline="") as fh:
        return list(csv.DictReader(fh))


def test_exported_calibration_rebuilds_the_tables(tmp_path):
    from humanrf_b200.dataset.cameras import projection_matrix_world2pixel
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    ds, loader = _cpu_loader()
    poses = _moved(CameraPoses(loader, intrinsics=True))
    ikr, org = poses.tables()
    refined = poses.refined_cameras()
    for c, cam in enumerate(refined):
        # the loader's path: normalised centre, world-to-pixel projection, inverse, transpose, float32
        t = (np.asarray(cam.translation) + loader.scene_offset) * loader.scene_scale
        P = projection_matrix_world2pixel(cam.width, cam.height, cam.rotation_axisangle, t, cam.focal_length,
                                          cam.principal_point)
        table = torch.from_numpy(np.linalg.inv(P))[:3, :3].T.float()
        got = ikr[c].numpy()
        ulp = np.spacing(np.maximum(np.abs(got), np.abs(table.numpy())))
        assert (np.abs(got.astype(np.float64) - table.numpy()) <= 2 * ulp).all(), c
        np.testing.assert_allclose(t, org[c].numpy(), rtol=0, atol=2e-7)
        base = ds.cameras[c]
        np.testing.assert_allclose(cam.focal_length, base.focal_length * np.exp(poses.alpha[c].numpy()), rtol=1e-15)
        np.testing.assert_allclose(cam.principal_point, base.principal_point + base.focal_length * poses.beta[c].numpy(),
                                   rtol=1e-15)
    path = tmp_path / "calibration.csv"
    poses.write_calibration_csv(path)
    for r, cam in zip(_read_csv(path), refined):       # reads back to the same cameras
        assert (int(r["w"]), int(r["h"])) == (cam.width, cam.height)
        assert [float(r[k]) for k in ("rx", "ry", "rz")] == list(cam.rotation_axisangle)
        assert [float(r[k]) for k in ("tx", "ty", "tz")] == list(cam.translation)
        assert [float(r[k]) for k in ("fx", "fy")] == list(cam.focal_length)
        assert [float(r[k]) for k in ("px", "py")] == list(cam.principal_point)


def test_state_round_trip_and_pose_only_state():
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    _, loader = _cpu_loader()
    poses = _moved(CameraPoses(loader, intrinsics=True))
    rng = np.random.default_rng(9)
    with torch.no_grad():
        for name in ("exp_avg", "exp_avg_sq", "intrinsics_exp_avg", "intrinsics_exp_avg_sq"):
            getattr(poses, name).copy_(torch.from_numpy(rng.random(getattr(poses, name).shape)))
        poses.steps.copy_(torch.arange(6, dtype=torch.int32))
    state = poses.state_dict()
    _, loader2 = _cpu_loader()
    other = CameraPoses(loader2, intrinsics=True, fixed_cameras=(3,))
    other.load_state_dict(state)
    names = ("omega", "tau", "exp_avg", "exp_avg_sq", "steps", "fixed", "alpha", "beta", "intrinsics_exp_avg",
             "intrinsics_exp_avg_sq")
    for name in names:
        assert torch.equal(getattr(other, name), getattr(poses, name)), name
    ikr, org = poses.tables()
    assert torch.equal(loader2.all_inverse_krs, ikr) and torch.equal(loader2.all_camera_origins, org)
    for s, c in enumerate(loader2.camera_numbers_cuda.tolist()):
        assert torch.equal(loader2.inverse_krs_cuda[s], ikr[c])
    assert torch.equal(other.rotations, poses.current_rotations())
    # a pose-only state: the intrinsics and their moments stay at zero
    pose_only = CameraPoses(_cpu_loader()[1])
    with torch.no_grad():
        pose_only.omega.copy_(poses.omega)
    pose_state = pose_only.state_dict()
    assert not any(k in pose_state for k in ("alpha", "beta", "intrinsics_exp_avg", "base_intrinsics"))
    other.load_state_dict(pose_state)
    for name in ("alpha", "beta", "intrinsics_exp_avg", "intrinsics_exp_avg_sq"):
        assert float(getattr(other, name).abs().sum()) == 0.0, name
    assert torch.equal(other.tables()[0], pose_only.tables()[0])
    # refined intrinsics do not load into a pose-only object
    with pytest.raises(RuntimeError, match="intrinsics=True"):
        CameraPoses(_cpu_loader()[1]).load_state_dict(state)


def test_pose_only_object_is_unchanged():
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    poses = CameraPoses(_cpu_loader()[1])
    assert not poses.intrinsics and not hasattr(poses, "alpha")
    assert sorted(poses.state_dict()) == sorted(["omega", "tau", "exp_avg", "exp_avg_sq", "steps", "fixed_cameras",
                                                 "base_inverse_krs", "base_camera_origins"])


def test_intrinsics_need_the_loader_cameras():
    from types import SimpleNamespace

    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    _, loader = _cpu_loader()
    fake = SimpleNamespace(**{k: getattr(loader, k) for k in ("all_inverse_krs", "all_camera_origins", "camera_numbers",
                                                              "inverse_krs_cuda", "camera_origins_cuda",
                                                              "camera_numbers_cuda")})
    with pytest.raises(RuntimeError, match="loader.cameras"):
        CameraPoses(fake, intrinsics=True)


def test_refined_camera_projection_matches_the_table():
    """A point seen through the refined table's ray lands on the refined camera's pixel (world units)."""
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    ds, loader = _cpu_loader()
    poses = _moved(CameraPoses(loader, intrinsics=True), seed=11)
    ikr, org = poses.tables()
    refined = poses.refined_cameras()
    for c in range(poses.num_cameras):
        cam = copy.deepcopy(refined[c])
        T = ikr[c].double().numpy()
        px, py = 20.5, 31.5
        v = px * T[0] + py * T[1] + T[2]
        point_n = org[c].double().numpy() + 1.3 * v / np.linalg.norm(v)
        point = point_n / loader.scene_scale - loader.scene_offset
        np.testing.assert_allclose(IO.project(point[None], cam)[0], [px, py], atol=2e-4)
    assert PO.so3_exp(np.zeros(3)).tolist() == np.eye(3).tolist()
