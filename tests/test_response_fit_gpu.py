"""Held-out response fit on the H100: hrf_response_fit_accumulate against tests/response_fit_oracle.py (correctly
rounded sums), hrf_response_fit_solve against the oracle's solve and its refusals, recovery of known responses of
held-out cameras on the teacher scene of DESIGN.md §3.14/§3.17, evaluate_sequence with fitted responses, and the
refusals of CameraResponses.fit_held_out.

Bars:
* accumulate: every addend is exact in float64, so a sum of m addends in any order is within (m - 1) 2^-53 sum|addends|
  of the correctly rounded sum; n and S_yy are sums of integers below 2^53 and exact.
* solve: the kernel and the oracle take the same float64 operations in the same order, so gains, offsets and SSEs
  agree within 1e-12 relative (log may differ in the last bits).
"""
import csv
import re
import types

import numpy as np
import pytest
import torch

import response_fit_oracle as FO
import response_oracle as RO

pytestmark = pytest.mark.gpu

EXACT = (0, 6, 11, 16)       # n and S_yy of each channel


def _fake_loader(cuda, C_):
    from types import SimpleNamespace

    return SimpleNamespace(all_inverse_krs=torch.zeros((C_, 3, 3), device=cuda), camera_numbers=tuple(range(C_)))


def _view(P, kind, rng):
    color = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    alpha = rng.uniform(0, 1, P).astype(np.float32)
    alpha[rng.uniform(0, 1, P) < 0.3] = 1.0
    alpha[rng.uniform(0, 1, P) < 0.1] = 0.0
    gt = rng.integers(0, 256, (P, 3), dtype=np.uint8)
    if kind == "empty":
        mask = np.zeros(P, np.uint8)
    elif kind == "full":
        mask = np.full(P, 7, np.uint8)                # any non-zero byte is inside
    elif kind == "random":
        mask = (rng.uniform(0, 1, P) < 0.5).astype(np.uint8)
    else:
        mask = np.zeros(P, np.uint8)
        if P:
            mask[rng.integers(0, P)] = 1
    return color, alpha, gt, mask


def _accumulate(resp, views, camera, moments, cuda):
    error = torch.zeros(1, dtype=torch.int32, device=cuda)
    for color, alpha, gt, mask in views:
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
        resp.accumulate_fit(d(color), d(alpha), d(gt), d(mask), camera, moments, error)
    torch.cuda.synchronize()
    return error


def _bytes(t):
    return t.cpu().numpy().tobytes()


@pytest.mark.parametrize("kind", ["empty", "full", "random", "single"])
@pytest.mark.parametrize("P", [0, 1, 31, 4099, 1028 * 752, 4112 * 3008])
def test_accumulate_matches_oracle(cuda, P, kind):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    rng = np.random.default_rng(P + len(kind))
    view = _view(P, kind, rng)
    want, mag, m = FO.moments(*view)
    for C_ in (1, 160, 1024):
        resp = CameraResponses(_fake_loader(cuda, C_), fixed_cameras=())
        camera = C_ - 1 if C_ > 1 else 0
        sentinel = torch.from_numpy(rng.uniform(-1, 1, (C_, FO.ROW))).to(cuda)
        moments = sentinel.clone()
        moments[camera] = 0.0
        err = _accumulate(resp, [view], camera, moments, cuda)
        assert int(err[0]) == 0
        got = moments.cpu().numpy()
        others = np.arange(C_) != camera
        assert got[others].tobytes() == sentinel.cpu().numpy()[others].tobytes()
        bound = max(m - 1, 0) * 2.0 ** -53 * mag
        assert (np.abs(got[camera] - want) <= bound).all(), (got[camera], want, bound)
        assert (got[camera][list(EXACT)] == want[list(EXACT)]).all()
        assert got[camera][0] == int((view[3] != 0).sum())
        again = sentinel.clone()
        again[camera] = 0.0
        _accumulate(resp, [view], camera, again, cuda)
        assert _bytes(again) == _bytes(moments)                      # a rerun writes the same bytes


def test_views_add_in_order_and_bad_camera_writes_nothing(cuda):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    rng = np.random.default_rng(11)
    C_ = 160
    resp = CameraResponses(_fake_loader(cuda, C_), fixed_cameras=())
    views = [_view(P, "random", rng) for P in (5000, 70001, 123)]
    moments = torch.zeros((C_, FO.ROW), dtype=torch.float64, device=cuda)
    _accumulate(resp, views, 7, moments, cuda)
    rows = [FO.moments(*v) for v in views]
    m = sum(r[2] for r in rows)
    want = FO.moments(*(np.concatenate([v[i] for v in views]) for i in range(4)))[0]
    mag = sum(r[1] for r in rows)
    got = moments[7].cpu().numpy()
    assert (np.abs(got - want) <= (m - 1) * 2.0 ** -53 * mag).all()
    # each view's own sums added in the given order
    seq = torch.zeros((C_, FO.ROW), dtype=torch.float64, device=cuda)
    total = np.zeros(FO.ROW)
    for v in views:
        one = torch.zeros((C_, FO.ROW), dtype=torch.float64, device=cuda)
        _accumulate(resp, [v], 7, one, cuda)
        total = total + one[7].cpu().numpy()
    _accumulate(resp, views, 7, seq, cuda)
    assert seq[7].cpu().numpy().tobytes() == total.tobytes()
    for bad in (C_, -1, 5000):
        before = _bytes(moments)
        err = _accumulate(resp, [views[0]], bad, moments, cuda)
        assert int(err[0]) == 1 and _bytes(moments) == before
    with pytest.raises(RuntimeError):
        resp.accumulate_fit(torch.zeros(4, 3, device=cuda), torch.zeros(4, device=cuda),
                            torch.zeros(4, 3, dtype=torch.uint8, device=cuda), torch.zeros(5, dtype=torch.uint8, device=cuda),
                            0, moments, torch.zeros(1, dtype=torch.int32, device=cuda))


# ------------------------------------------------------------------------------------------------ solve
def _state(resp):
    return {n: _bytes(getattr(resp, n)) for n in ("params", "exp_avg", "exp_avg_sq", "steps", "table")}


def _fit_data(P, rng, gain, offset):
    a = np.where(rng.uniform(0, 1, P) < 0.7, 1.0, rng.uniform(0, 1, P)).astype(np.float32)
    f = (rng.uniform(0.05, 0.85, (P, 3)) * a[:, None]).astype(np.float32)
    y = np.asarray(gain) * f + a[:, None] * np.asarray(offset) + rng.normal(0, 2e-3, (P, 3))
    gt = np.rint(np.clip(y, 0, 1) * 255).astype(np.uint8)
    return f, a, gt, (rng.uniform(0, 1, P) < 0.8).astype(np.uint8)


def _loaded(cuda, C_, rng):
    """CameraResponses with random params, moments of Adam and steps on every camera (so that stray writes show)."""
    from humanrf_b200.toolbox.camera_response import CameraResponses

    resp = CameraResponses(_fake_loader(cuda, C_), fixed_cameras=(0,))
    params = np.concatenate((rng.uniform(-0.2, 0.2, (C_, 3)), rng.uniform(-0.05, 0.05, (C_, 3))), 1)
    resp.load_state_dict({"params": torch.from_numpy(params), "exp_avg": torch.from_numpy(rng.normal(0, 1e-3, (C_, 6))),
                          "exp_avg_sq": torch.from_numpy(rng.uniform(0, 1e-6, (C_, 6))),
                          "steps": torch.from_numpy(rng.integers(0, 50, C_).astype(np.int32)),
                          "fixed_cameras": [0]})
    return resp


def test_solve_matches_oracle_and_writes_only_listed_cameras(cuda):
    rng = np.random.default_rng(3)
    C_ = 160
    resp = _loaded(cuda, C_, rng)
    listed = [3, 17, 42, 159]
    moments = torch.zeros((C_, FO.ROW), dtype=torch.float64, device=cuda)
    truth = {}
    for c in listed:
        gain, off = rng.uniform(0.8, 1.2, 3), rng.uniform(-0.05, 0.05, 3)
        truth[c] = (gain, off)
        _accumulate(resp, [_fit_data(int(rng.integers(3000, 60000)), rng, gain, off) for _ in range(3)], c, moments,
                    cuda)
    moments[5] = moments[3]                  # moments of a camera that is not listed: never read, never written
    before, mom = _state(resp), _bytes(moments)
    report, status = resp.solve_fit(moments, listed, 1e-6, 1024)
    torch.cuda.synchronize()
    gains, offs, rep, st = FO.solve(moments.cpu().numpy(), listed, 1e-6, 1024)
    assert (status.cpu().numpy() == 0).all() and (st == 0).all()
    got_rep = report.cpu().numpy()
    assert np.allclose(got_rep, rep, rtol=1e-12, atol=0)
    params = resp.params.cpu().numpy()
    for k, c in enumerate(listed):
        assert np.allclose(params[c, :3], np.log(gains[k]), rtol=1e-12, atol=1e-15)
        assert np.allclose(params[c, 3:], offs[k], rtol=1e-12, atol=1e-15)
        assert np.allclose(np.exp(params[c, :3]), truth[c][0], atol=5e-3)
        assert np.allclose(params[c, 3:], truth[c][1], atol=5e-3)
    tab, want = resp.table.cpu().numpy(), RO.table_of(params)
    assert (np.abs(tab[listed].astype(np.float64) - want[listed]) <= np.spacing(np.abs(want[listed]))).all()
    after = _state(resp)
    for n in ("exp_avg", "exp_avg_sq", "steps"):
        assert after[n] == before[n], n
    unlisted = np.setdiff1d(np.arange(C_), listed)
    p0 = np.frombuffer(before["params"], np.float64).reshape(C_, 6)
    t0 = np.frombuffer(before["table"], np.float32).reshape(C_, 6)
    assert params[unlisted].tobytes() == p0[unlisted].tobytes() and tab[unlisted].tobytes() == t0[unlisted].tobytes()
    assert _bytes(moments) == mom


def test_solve_refusals_write_nothing(cuda):
    rng = np.random.default_rng(4)
    C_ = 8
    resp = _loaded(cuda, C_, rng)
    moments = torch.zeros((C_, FO.ROW), dtype=torch.float64, device=cuda)
    _accumulate(resp, [_fit_data(20000, rng, (0.9, 1.0, 1.1), (0.02, 0.0, -0.02))], 1, moments, cuda)
    # gain <= 0: gt = 255 - round(255 f) at alpha 1
    f = rng.uniform(0.05, 0.95, (20000, 3)).astype(np.float32)
    a = np.ones(20000, np.float32)
    gt = (255 - np.rint(f * 255)).astype(np.uint8)
    _accumulate(resp, [(f, a, gt, np.ones(20000, np.uint8))], 2, moments, cuda)
    # too few pixels
    _accumulate(resp, [_fit_data(100, rng, (1, 1, 1), (0, 0, 0))], 3, moments, cuda)
    # non-finite: no spread at all (every f = alpha = 1) and no ridge: a singular system
    _accumulate(resp, [(np.ones((5000, 3), np.float32), np.ones(5000, np.float32),
                        np.full((5000, 3), 200, np.uint8), np.ones(5000, np.uint8))], 4, moments, cuda)
    mom = _bytes(moments)
    for listed, lam, want in (([1, 2], 1e-6, [0, 3]), ([3, 1], 1e-6, [1, 0]), ([1, 4], 0.0, [0, 2]),
                              ([1, C_], 1e-6, [0, 4]), ([1, -3], 1e-6, [0, 4])):
        before = _state(resp)
        report, status = resp.solve_fit(moments, listed, lam, 1024)
        torch.cuda.synchronize()
        assert status.cpu().numpy().tolist() == want, (listed, status)
        _, _, rep, st = FO.solve(moments.cpu().numpy(), listed, lam, 1024, num_cameras=C_)
        assert st.tolist() == want
        assert report.cpu().numpy()[:, 7].tolist() == want
        assert _state(resp) == before and _bytes(moments) == mom
    # the same cameras solved alone are accepted: the refusal was the other camera's
    report, status = resp.solve_fit(moments, [1], 1e-6, 1024)
    assert status.cpu().numpy().tolist() == [0]


# ------------------------------------------------------------------------------------------------ teacher scene
HELD_OUT = {3: ((0.85, 0.95, 0.9), (0.03, -0.04, 0.02)), 5: ((0.98, 0.82, 0.93), (-0.03, 0.05, 0.0)),
            6: ((0.9, 0.88, 1.0), (0.01, 0.02, -0.05)), 1: ((1.0, 1.0, 1.0), (0.0, 0.0, 0.0)),
            7: ((1.0, 1.0, 1.0), (0.0, 0.0, 0.0))}
SCORED_FRAME = 16


@pytest.fixture(scope="module")
def scene(cuda):
    """The teacher scene: 8 cameras, frames 15..20 of the static textured teacher.  Camera c's images are
    g_c f + alpha b_c of the teacher's render (HELD_OUT: cameras 1 and 7 at identity; 0, 2, 4 recorded as rendered),
    with every offset kept where no masked pixel of any frame leaves [0, 1]."""
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from test_camera_poses_gpu import _scene8, _TeacherDataset
    from test_ray_grad_gpu import textured_teacher

    base = _scene8()
    teacher = textured_teacher(cuda)
    view = DL(dataset=base, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192,
              camera_numbers=tuple(range(8)), frame_numbers=tuple(base.frames), max_buffer_size=1,
              render_sequence=[(0, 15)])
    renders = {}
    for c in range(8):
        for f in base.frames:
            dm = render_depth_map(teacher, view, c, f)
            renders[(c, f)] = (dm.color.double().cpu().numpy(), dm.alpha.double().cpu().numpy()[..., None])
    true = {c: (np.ones(3), np.zeros(3)) for c in range(8)}
    for c, (g, b) in HELD_OUT.items():
        g, b = np.asarray(g, np.float64), np.asarray(b, np.float64).copy()
        for col, a in (renders[(c, f)] for f in base.frames):
            m = a[..., 0] > 0.5
            gf, am = g * col[m], a[m]
            b = np.maximum(b, (-gf / am).max(0))
            b = np.minimum(b, ((1 - gf) / am).min(0))
        true[c] = (g, b)
    images, masks = {}, {}
    for (c, f), (col, a) in renders.items():
        g, b = true[c]
        images[(c, f)] = (g * col + a * b).astype(np.float32)
        masks[(c, f)] = (a > 0.5).astype(np.float32)
    ds = _TeacherDataset(base, images, masks)
    loader = DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=256 * 192,
                camera_numbers=tuple(range(8)), frame_numbers=tuple(base.frames), max_buffer_size=1,
                render_sequence=[(0, 15)])
    return {"teacher": teacher, "loader": loader, "true": true, "renders": renders, "frames": list(base.frames)}


def _fitted(scene, cameras, per_camera=4):
    from humanrf_b200.toolbox.camera_response import CameraResponses, held_out_fit_pairs

    resp = CameraResponses(scene["loader"])
    score = [(c, SCORED_FRAME) for c in cameras]
    pairs = held_out_fit_pairs(score, scene["frames"], per_camera=per_camera)
    fits = resp.fit_held_out(scene["teacher"], scene["loader"], pairs)
    return resp, score, pairs, fits


def _colour_error(scene, c, est_g, est_b):
    col, a = scene["renders"][(c, SCORED_FRAME)]
    m = a[..., 0] > 0.5
    g, b = scene["true"][c]
    return float(np.sqrt((((np.asarray(est_g) - g) * col[m] + a[m] * (np.asarray(est_b) - b)) ** 2).mean()))


def test_fit_recovers_held_out_responses(cuda, scene):
    resp, score, pairs, fits = _fitted(scene, sorted(HELD_OUT))
    assert not set(pairs) & set(score)
    assert [f.camera for f in fits] == sorted(HELD_OUT)
    for fit in fits:
        c = fit.camera
        assert SCORED_FRAME not in fit.frames and len(fit.frames) == 4
        e = _colour_error(scene, c, fit.gain, fit.offset)
        g, b = scene["true"][c]
        print(f"camera {c}: true gain {g.round(4)} offset {b.round(4)}; fitted gain {np.round(fit.gain, 4)} offset "
              f"{np.round(fit.offset, 4)}; colour error {e:.2e} ({e * 255:.3f} / 255); n {fit.n}; PSNR "
              f"{fit.psnr_before:.2f} -> {fit.psnr_after:.2f} dB")
        assert e < 1.0 / 255
        assert fit.psnr_after >= fit.psnr_before
        assert fit.n > 1024
    assert resp.fitted_pairs == {c: [(c, f) for f in fits[k].frames] for k, c in enumerate(sorted(HELD_OUT))}
    assert int(resp.steps.abs().sum()) == 0 and float(resp.exp_avg.abs().sum()) == 0.0
    assert (resp.params[[0, 2, 4]] == 0).all()
    # fitting a camera again replaces its fit
    other = [(3, 15), (3, 20)]
    again = resp.fit_held_out(scene["teacher"], scene["loader"], other)
    assert [f.camera for f in again] == [3] and resp.fitted_pairs[3] == other
    assert _colour_error(scene, 3, again[0].gain, again[0].offset) < 1.0 / 255


def test_evaluate_sequence_with_fitted_responses(cuda, scene, tmp_path):
    from humanrf_b200.toolbox.camera_response import FIT_COLUMNS, CameraResponses
    from humanrf_b200.toolbox.depth_maps import camera_name
    from humanrf_b200.toolbox.evaluation import evaluate_sequence

    teacher, loader = scene["teacher"], scene["loader"]
    held = [3, 5, 6]
    resp, score, pairs, fits = _fitted(scene, held)
    scored = score + [(0, SCORED_FRAME), (2, SCORED_FRAME)]
    plain = evaluate_sequence(teacher, loader, scored, tmp_path / "plain", save_frames=False)
    got = evaluate_sequence(teacher, loader, scored, tmp_path / "fit", save_frames=False, camera_responses=resp)
    for s, p in zip(got[3:], plain[3:]):                            # unfitted cameras: the scores without responses
        assert (s.psnr, s.ssim) == (p.psnr, p.ssim)
    true = CameraResponses(loader)
    params = torch.zeros((8, 6), dtype=torch.float64)
    for c in held:
        g, b = scene["true"][c]
        params[c, :3], params[c, 3:] = torch.from_numpy(np.log(g)), torch.from_numpy(b)
    true.load_state_dict({"params": params, "exp_avg": torch.zeros(8, 6, dtype=torch.float64),
                          "exp_avg_sq": torch.zeros(8, 6, dtype=torch.float64), "steps": torch.zeros(8, dtype=torch.int32),
                          "fixed_cameras": [0]})
    ref = evaluate_sequence(teacher, loader, score, tmp_path / "true", save_frames=False, camera_responses=true)
    for s, r, p in zip(got, ref, plain):
        print(f"camera {s.camera} frame {s.frame}: PSNR unfitted {p.psnr:.2f}, fitted {s.psnr:.2f}, true response "
              f"{r.psnr:.2f} dB; SSIM {p.ssim:.4f} / {s.ssim:.4f} / {r.ssim:.4f}")
        assert abs(s.psnr - r.psnr) <= 0.5
        assert s.psnr >= p.psnr + 3.0
    assert not (tmp_path / "true" / "response_fit.csv").exists() and not (tmp_path / "plain" / "response_fit.csv").exists()
    rows = list(csv.reader(open(tmp_path / "fit" / "response_fit.csv", newline="")))
    assert tuple(rows[0]) == FIT_COLUMNS and len(rows) == 1 + len(held)
    for row, fit in zip(rows[1:], fits):
        assert row[0] == camera_name(loader, fit.camera)
        assert int(row[1]) == len(fit.frames) and int(row[2]) == fit.n
        assert [float(x) for x in row[3:9]] == [*fit.gain, *fit.offset]
        assert (float(row[9]), float(row[10])) == (fit.psnr_before, fit.psnr_after)
    # a scored pair among the fit pairs raises before anything is written
    out = tmp_path / "leak"
    with pytest.raises(ValueError, match=re.escape(str(pairs[-1]))):
        evaluate_sequence(teacher, loader, [(0, 16), pairs[-1]], out, camera_responses=resp)
    assert not out.exists()


def test_saturating_gain_scores_as_the_clamped_render(cuda, scene, tmp_path):
    """A fitted gain above 1 pushes bright pixels past 1: the score is the one of the render clamped to [0, 1] before
    quantising (quantize alone wraps such values on the CPU; on the GPU its result is not pinned)."""
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.toolbox.evaluation import evaluate_sequence, ground_truth, image_metrics, quantize

    teacher, loader = scene["teacher"], scene["loader"]
    resp = CameraResponses(loader)
    # camera 4 records the render as it is.  Fitted against its images brightened channel by channel so that each
    # channel's brightest masked pixel reaches 1.2 (clipped at 255 by ground_truth), a gain comes out above 1.  (A
    # channel whose colours sit close to its brightest clips on most pixels and trades gain for offset instead.)
    frames = [15, 17, 18]
    brightest = np.max([col[a[..., 0] > 0.5].max(0) for col, a in (scene["renders"][(4, f)] for f in frames)], 0)
    scale = (1.2 / brightest)[::-1].astype(np.float32)             # get_rgb's channel order is BGR
    bright = types.SimpleNamespace(**{k: getattr(loader, k) for k in ("all_inverse_krs", "all_camera_origins", "aabb",
                                                                      "scene_scale", "cameras", "camera_numbers")})
    bright.dataset = types.SimpleNamespace(get_occupancy_grid=loader.dataset.get_occupancy_grid,
                                           get_mask=loader.dataset.get_mask,
                                           get_rgb=lambda c, f, normalize=True: loader.dataset.get_rgb(c, f) * scale)
    fits = resp.fit_held_out(teacher, bright, [(4, f) for f in frames])
    print(f"brightened {scale[::-1].round(3)} times: fitted gain {np.round(fits[0].gain, 4)} offset "
          f"{np.round(fits[0].offset, 4)}")
    assert max(fits[0].gain) > 1.0
    got = evaluate_sequence(teacher, loader, [(4, SCORED_FRAME)], tmp_path / "sat", save_frames=False,
                            camera_responses=resp)
    dm = render_depth_map(teacher, loader, 4, SCORED_FRAME)
    applied = resp.apply(dm.color.contiguous().clone(), dm.alpha.contiguous(), 4)
    assert float(applied.max()) > 1.0                                # pixels saturate
    gt, mask = ground_truth(loader, 4, SCORED_FRAME)
    vals, _ = image_metrics(quantize(applied.clamp(0, 1)), torch.from_numpy(gt).to(cuda),
                            torch.from_numpy(mask).to(cuda))
    assert (float(vals[0]), float(vals[1])) == (got[0].psnr, got[0].ssim)


def test_fit_held_out_refusals(cuda, scene):
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from test_evaluation_gpu import _loader

    teacher, loader = scene["teacher"], scene["loader"]
    resp = CameraResponses(loader)
    before = _state(resp)
    with pytest.raises(ValueError, match="fixed"):
        resp.fit_held_out(teacher, loader, [(3, 15), (0, 15)])
    steps = resp.steps.clone()
    resp.steps[5] = 1
    with pytest.raises(ValueError, match="trained"):
        resp.fit_held_out(teacher, loader, [(5, 15)])
    resp.steps.copy_(steps)
    with pytest.raises(ValueError, match="frame 99"):
        resp.fit_held_out(teacher, loader, [(3, 15), (3, 99)])
    _, small = _loader(cuda)
    with pytest.raises(ValueError, match="cameras"):
        resp.fit_held_out(teacher, small, [(1, 15)])
    with pytest.raises(ValueError, match="camera 3"):                  # refused by the solve: nothing written
        resp.fit_held_out(teacher, loader, [(3, 15), (6, 15)], min_pixels=10 ** 7)
    assert _state(resp) == before and resp.fits == {}
