"""Depth-map export on the CPU (humanrf_b200/toolbox/depth_maps.py): the distance -> camera z conversion against a
projection through world2pixel, the EXR / PNG writers and the ActorsHQ renderer's file layout."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from humanrf_b200.dataset.cameras import inverse_kr
from humanrf_b200.synthetic_scene import look_at_camera, make_scene
from humanrf_b200.toolbox import depth_maps as D


def _make_scene_world2pixel(num_images, width, height, seed=0, portrait_every=3):
    """The world2pixel matrices behind make_scene's inverse_krs (same camera ring, same generator draws)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(num_images):
        a = 2 * np.pi * i / num_images + 0.3
        pos = np.array([2.0 * np.cos(a), rng.uniform(-0.4, 0.4), 2.0 * np.sin(a)])
        ls = not (portrait_every and i % portrait_every == portrait_every - 1)
        w, h = (width, height) if ls else (height, width)
        out.append((look_at_camera(pos, w, h), pos, w, h, ls))
    return out


def test_distance_to_z_matches_a_projection_through_world2pixel():
    W, H = 40, 30
    sc = make_scene(num_images=3, width=W, height=H)
    cams = _make_scene_world2pixel(3, W, H)
    assert [c[4] for c in cams] == list(sc["landscape"]) and not cams[2][4]     # one portrait view
    rng = np.random.default_rng(3)
    for k, (w2p, pos, w, h, _) in enumerate(cams):
        np.testing.assert_array_equal(inverse_kr(w2p), sc["inverse_krs"][k])
        T = sc["inverse_krs"][k]
        norms = D.pixel_ray_norms(torch.from_numpy(T), w, h).numpy()
        assert norms.shape == (w * h,)
        x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
        v = np.stack([x, y, np.ones_like(x)], -1).reshape(-1, 3) @ T.astype(np.float64)   # the sampler's M [px,py,1]
        np.testing.assert_allclose(np.linalg.norm(v, axis=1), norms, rtol=1e-15)
        s = rng.uniform(1.0, 3.0, w * h)                                             # distance along the unit ray
        p = pos + s[:, None] * v / np.linalg.norm(v, axis=1, keepdims=True)
        q = (w2p @ np.concatenate([p, np.ones((w * h, 1))], 1).T).T
        z = s / norms
        np.testing.assert_allclose(q[:, 2], z, rtol=2e-6)                            # camera z (K's last row is 0 0 1)
        np.testing.assert_allclose(q[:, 0] / q[:, 2], x.reshape(-1), atol=2e-4)      # lands on the pixel centre ...
        np.testing.assert_allclose(q[:, 1] / q[:, 2], y.reshape(-1), atol=2e-4)      # ... in row-major order


def test_exr_and_png_round_trip_exactly(tmp_path):
    D.write_depth_exr(tmp_path / "probe.exr", np.zeros((1, 1), np.float32))          # enables OpenCV's EXR codec first
    import cv2

    rng = np.random.default_rng(0)
    z = (rng.random((23, 37)) * 5).astype(np.float32)
    z[rng.random(z.shape) < 0.3] = 0.0
    z[0, 0] = np.float32(1e-30)
    z[0, 1] = np.nextafter(np.float32(2.0), np.float32(3.0))
    D.write_depth_exr(tmp_path / "z.exr", torch.from_numpy(z))
    back = cv2.imread(str(tmp_path / "z.exr"), cv2.IMREAD_UNCHANGED)
    assert back.dtype == np.float32 and back.shape == z.shape
    assert np.array_equal(back.view(np.uint32), z.view(np.uint32))
    m = rng.random((23, 37)) >= 0.5
    D.write_mask_png(tmp_path / "m.png", torch.from_numpy(m))
    mb = cv2.imread(str(tmp_path / "m.png"), cv2.IMREAD_UNCHANGED)
    assert mb.dtype == np.uint8 and mb.shape == m.shape
    assert np.array_equal(mb, m.astype(np.uint8) * 255)


def test_writers_raise_on_failure(tmp_path):
    with pytest.raises(RuntimeError):
        D.write_depth_exr(tmp_path / "missing_dir" / "z.exr", np.zeros((2, 2), np.float32))
    with pytest.raises(RuntimeError):
        D.write_mask_png(tmp_path / "missing_dir" / "m.png", np.zeros((2, 2), bool))


def test_file_names_and_layout():
    named = SimpleNamespace(cameras=[SimpleNamespace(name="Cam042"), SimpleNamespace()])
    assert D.camera_name(named, 0) == "Cam042"
    assert D.camera_name(named, 1) == "Cam002"          # 1-based, as actorshq/evaluation numbers cameras
    unnamed = SimpleNamespace(cameras=[SimpleNamespace() for _ in range(12)])
    assert [D.camera_name(unnamed, c) for c in (0, 9, 11)] == ["Cam001", "Cam010", "Cam012"]
    assert D.depth_path("out", "Cam007", 15) == os.path.join("out", "depths", "Cam007", "Cam007_depth000015.exr")
    assert D.mask_path("out", "Cam007", 123456) == os.path.join("out", "masks", "Cam007", "Cam007_mask123456.png")
