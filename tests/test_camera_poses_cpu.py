"""Per-camera pose refinement without a GPU: the float64 references of tests/pose_oracle.py against torch autograd and
torch.optim.Adam, CameraPoses' state and calibration export, and FusedTrainer's refusal of data-parallel poses."""
import csv

import numpy as np
import pytest
import torch

import pose_oracle as PO


@pytest.mark.parametrize("theta", [0.0, 1e-9, 1e-4, 0.3, 2.5])
def test_left_jacobian_pose_gradient_matches_autograd(theta):
    from humanrf_b200.toolbox.camera_refinement import rotation_increment

    rng = np.random.default_rng(int(theta * 1e3) + 1)
    axis = rng.standard_normal(3)
    w0 = theta * axis / np.linalg.norm(axis)
    d0 = rng.standard_normal((50, 3))
    d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
    g = rng.standard_normal((50, 3))
    w = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    d = (rotation_increment(w) @ torch.from_numpy(d0).T).T
    (ref,) = torch.autograd.grad((d * torch.from_numpy(g)).sum(), w)
    d_np = d.detach().numpy()                      # the sampled directions, d = exp([w]x) d0
    got, n, _ = PO.pose_grad(np.zeros_like(g), g, d_np, np.zeros(50, np.int64), w0[None])
    assert n[0] == 50
    np.testing.assert_allclose(got[0, :3], ref.numpy(), rtol=1e-12, atol=1e-13 * np.abs(g).sum())
    if theta == 0.0:
        assert np.array_equal(PO.left_jacobian(w0), np.eye(3))


def test_oracle_exponential_matches_matrix_exp():
    from humanrf_b200.toolbox.camera_refinement import rotation_increment

    for th in (0.0, 1e-9, 1e-4, 5e-3, 0.3, 2.5):
        w = np.array([0.6, -0.8, 0.0]) * th
        np.testing.assert_allclose(PO.so3_exp(w), rotation_increment(torch.from_numpy(w)).numpy(), rtol=0, atol=1e-14)


def test_per_camera_adam_skips_untouched_and_fixed_cameras():
    C, lr = 5, 1e-2
    rng = np.random.default_rng(3)
    fixed = np.array([1, 0, 0, 0, 0], bool)
    st = dict(params=rng.standard_normal((C, 6)), m=np.zeros((C, 6)), v=np.zeros((C, 6)), steps=np.zeros(C, int))
    ref = [torch.tensor(st["params"][c], requires_grad=True) for c in range(C)]
    opts = [torch.optim.Adam([p], lr=lr, betas=(0.9, 0.99), eps=1e-15) for p in ref]
    touched_sets = [[0, 1, 2], [2, 3], [0, 1, 2, 3, 4], [4], [1, 2]]
    for touched in touched_sets:
        count = np.zeros(C, int)
        count[touched] = 7
        g = rng.standard_normal((C, 6))
        before = {k: v.copy() for k, v in st.items()}
        PO.adam(st, g, count, fixed, lr)
        for c in range(C):
            if c in touched and not fixed[c]:
                opts[c].zero_grad()
                ref[c].grad = torch.from_numpy(g[c].copy())
                opts[c].step()
            else:
                for k in st:
                    assert np.array_equal(st[k][c], before[k][c]), (c, k)
    for c in range(C):
        np.testing.assert_allclose(st["params"][c], ref[c].detach().numpy(), rtol=1e-13, atol=1e-15)
        s = opts[c].state.get(ref[c])
        assert st["steps"][c] == (int(s["step"]) if s else 0)
    assert list(st["steps"]) == [0, 3, 4, 2, 2]


def _cpu_loader():
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(num_cameras=6, width=64, height=48)
    loader = DL(dataset=ds, device="cpu", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS,
                space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=64, camera_numbers=tuple(range(6)),
                frame_numbers=tuple(ds.frames), max_buffer_size=2, render_sequence=[(2, 15), (4, 16)])
    return ds, loader


def test_state_dict_round_trip():
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    _, loader = _cpu_loader()
    poses = CameraPoses(loader)
    assert poses.fixed_cameras == (0,)
    rng = np.random.default_rng(5)
    with torch.no_grad():
        for name in ("omega", "tau", "exp_avg", "exp_avg_sq"):
            getattr(poses, name).copy_(torch.from_numpy(rng.standard_normal(getattr(poses, name).shape) * 1e-2))
        poses.steps.copy_(torch.arange(6, dtype=torch.int32))
    state = poses.state_dict()
    _, loader2 = _cpu_loader()
    other = CameraPoses(loader2, fixed_cameras=(3,))
    other.load_state_dict(state)
    for name in ("omega", "tau", "exp_avg", "exp_avg_sq", "steps", "fixed"):
        assert torch.equal(getattr(other, name), getattr(poses, name)), name
    assert other.fixed_cameras == (0,)
    # the loader's tables now hold the refined views, the pool slots their cameras' copies
    ikr, org = poses.tables()
    assert torch.equal(loader2.all_inverse_krs, ikr) and torch.equal(loader2.all_camera_origins, org)
    for s, c in enumerate(loader2.camera_numbers_cuda.tolist()):
        assert torch.equal(loader2.inverse_krs_cuda[s], ikr[c]) and torch.equal(loader2.camera_origins_cuda[s], org[c])
    # omega = tau = 0 gives the loader's tables bit for bit
    zero = CameraPoses(_cpu_loader()[1])
    assert torch.equal(zero.tables()[0], zero.base_inverse_krs) and torch.equal(zero.tables()[1], zero.base_camera_origins)


def _read_csv(path):
    with open(path, newline="") as fh:
        return list(csv.DictReader(fh))


def test_write_calibration_csv(tmp_path):
    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    ds, loader = _cpu_loader()
    poses = CameraPoses(loader)
    path = tmp_path / "calibration.csv"
    poses.write_calibration_csv(path)
    with open(path) as fh:
        assert fh.readline().strip() == "name,w,h,rx,ry,rz,tx,ty,tz,fx,fy,px,py"
    rows = _read_csv(path)
    assert [r["name"] for r in rows] == [f"Cam{c + 1:03d}" for c in range(6)]
    for r, cam in zip(rows, ds.cameras):          # omega = tau = 0: the input calibration within float64 noise
        assert (int(r["w"]), int(r["h"])) == (cam.width, cam.height)
        np.testing.assert_allclose([float(r[k]) for k in ("rx", "ry", "rz")], cam.rotation_axisangle, rtol=0, atol=1e-12)
        np.testing.assert_allclose([float(r[k]) for k in ("tx", "ty", "tz")], cam.translation, rtol=0, atol=1e-12)
        assert [float(r[k]) for k in ("fx", "fy")] == list(cam.focal_length)
        assert [float(r[k]) for k in ("px", "py")] == list(cam.principal_point)
    # a moved camera: rotation exp([w]x) R and centre (c_n + tau) / scale - offset
    from humanrf_b200.dataset.cameras import rotation_from_axisangle

    w, tau = np.array([0.01, -0.02, 0.005]), np.array([0.003, 0.001, -0.002])
    with torch.no_grad():
        poses.omega[2] = torch.from_numpy(w)
        poses.tau[2] = torch.from_numpy(tau)
    poses.write_calibration_csv(path)
    r = _read_csv(path)[2]
    cam = ds.cameras[2]
    R = rotation_from_axisangle([float(r[k]) for k in ("rx", "ry", "rz")])
    np.testing.assert_allclose(R, PO.so3_exp(w) @ rotation_from_axisangle(cam.rotation_axisangle), atol=1e-12)
    np.testing.assert_allclose([float(r[k]) for k in ("tx", "ty", "tz")], cam.translation + tau / loader.scene_scale,
                               atol=1e-12)


def test_fused_trainer_rejects_camera_poses_with_data_parallel():
    from humanrf_b200.training import FusedTrainer

    with pytest.raises(ValueError, match="world_size"):
        FusedTrainer(None, world_size=2, camera_poses=object())
