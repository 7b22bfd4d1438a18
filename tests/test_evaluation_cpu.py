"""Image scores on the CPU: the float64 oracle (tests/eval_oracle.py) against a brute-force window loop and closed forms,
the ROI against cv2.boundingRect, and the files of humanrf_b200/toolbox/evaluation.py."""
import csv
import os

import numpy as np
import pytest

from eval_oracle import bounding_rect, evaluate_pair, psnr, ssim, ssim_channel
from humanrf_b200.toolbox import evaluation as E

C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2


def _brute_ssim_channel(x, y):
    """Mean of S over every 7x7 window lying inside the image, each window's statistics summed directly."""
    x, y = x.astype(np.float64), y.astype(np.float64)
    h, w = x.shape
    out = []
    for i in range(h - 6):
        for j in range(w - 6):
            a, b = x[i:i + 7, j:j + 7].ravel(), y[i:i + 7, j:j + 7].ravel()
            ux, uy = a.mean(), b.mean()
            vx, vy = a.var(ddof=1), b.var(ddof=1)
            vxy = ((a - ux) * (b - uy)).sum() / 48
            out.append((2 * ux * uy + C1) * (2 * vxy + C2) / ((ux * ux + uy * uy + C1) * (vx + vy + C2)))
    return float(np.mean(out))


@pytest.mark.parametrize("shape", [(7, 7), (8, 11), (20, 9)])
def test_oracle_ssim_equals_brute_force_windows(shape):
    rng = np.random.default_rng(sum(shape))
    x = rng.integers(0, 256, shape + (3,), dtype=np.uint8)
    y = np.clip(x.astype(int) + rng.integers(-40, 41, x.shape), 0, 255).astype(np.uint8)
    y[0, 0] = 255
    x[-1, -1] = 0
    for c in range(3):
        assert abs(ssim_channel(x[..., c], y[..., c]) - _brute_ssim_channel(x[..., c], y[..., c])) <= 1e-12
    ref = np.mean([_brute_ssim_channel(x[..., c], y[..., c]) for c in range(3)])
    assert abs(ssim(x, y) - ref) <= 1e-12


def test_closed_forms():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 256, (12, 10, 3), dtype=np.uint8)
    mask = np.ones((12, 10), bool)
    assert ssim(x, x) == pytest.approx(1.0, abs=1e-12) and psnr(x, x, mask) == float("inf")
    for a, b in ((0, 255), (17, 200), (128, 128)):
        ia, ib = np.full((9, 8, 3), a, np.uint8), np.full((9, 8, 3), b, np.uint8)
        assert ssim(ia, ib) == pytest.approx((2 * a * b + C1) / (a * a + b * b + C1), abs=1e-12)
    # an error of 1 in one channel on every masked pixel: MSE = 1 / (3 * 255^2)
    y = x.copy()
    y[..., 1] = np.where(y[..., 1] < 255, y[..., 1] + 1, 254)
    m = rng.random((12, 10)) < 0.5
    assert psnr(y, x, m) == pytest.approx(10 * np.log10(3 * 255 ** 2), abs=1e-12)
    # undefined cases
    assert np.isnan(ssim(x[:6], x[:6])) and np.isnan(ssim(x[:, :6], x[:, :6]))
    p, s, roi = evaluate_pair(x, y, np.zeros((12, 10), np.uint8))
    assert np.isnan(p) and np.isnan(s) and roi == (0, 0, 0, 0)


def test_roi_equals_cv2_bounding_rect():
    import cv2

    rng = np.random.default_rng(2)
    H, W = 23, 31
    masks = [rng.random((H, W)) < 0.05, np.zeros((H, W), bool)]
    for side in ("top", "bottom", "left", "right"):
        m = np.zeros((H, W), bool)
        m[{"top": (0, 5), "bottom": (H - 1, 7), "left": (4, 0), "right": (9, W - 1)}[side]] = True
        m[12, 13] = True
        masks.append(m)
    single = np.zeros((H, W), bool)
    single[6, 29] = True
    full = np.ones((H, W), bool)
    masks += [single, full]
    for m in masks:
        u8 = m.astype(np.uint8) * 255
        assert bounding_rect(u8) == tuple(cv2.boundingRect(u8[..., None])), m.nonzero()
    assert bounding_rect(single) == (29, 6, 1, 1) and bounding_rect(full) == (0, 0, W, H)


def test_crop_follows_the_roi():
    rng = np.random.default_rng(4)
    pred = rng.integers(0, 256, (30, 40, 3), dtype=np.uint8)
    gt = rng.integers(0, 256, (30, 40, 3), dtype=np.uint8)
    m = np.zeros((30, 40), np.uint8)
    m[5:20, 8:30] = rng.random((15, 22)) < 0.6
    m[5, 8] = m[19, 29] = 1
    p, s, roi = evaluate_pair(pred, gt, m)
    assert roi == (8, 5, 22, 15)
    assert s == ssim(gt[5:20, 8:30], pred[5:20, 8:30])
    assert p == psnr(pred, gt, m)          # every masked pixel is inside the ROI


def test_tables_and_file_names(tmp_path):
    scores = [E.ViewScore(0, 15, 30.5, 0.9, (0, 0, 8, 8)), E.ViewScore(2, 15, float("inf"), 1.0, (1, 2, 9, 9)),
              E.ViewScore(0, 16, 20.25, 0.75, (0, 0, 7, 7))]
    E.write_metric_tables(tmp_path, scores)
    with open(tmp_path / "metrics.csv", newline="") as f:
        rows = list(csv.reader(f))
    assert rows[0] == ["camera", "frame", "PSNR", "SSIM"]
    assert [r[:2] for r in rows[1:]] == [["1", "15"], ["3", "15"], ["1", "16"]]
    assert [float(r[2]) for r in rows[1:]] == [30.5, float("inf"), 20.25]
    assert [float(r[3]) for r in rows[1:]] == [0.9, 1.0, 0.75]
    with open(tmp_path / "averages.csv", newline="") as f:
        avg = list(csv.reader(f))
    assert avg[0] == ["PSNR", "SSIM"]
    assert float(avg[1][0]) == float("inf") and float(avg[1][1]) == pytest.approx((0.9 + 1.0 + 0.75) / 3, abs=1e-15)
    assert E.frame_path("out", "Cam007", 15) == os.path.join("out", "test_frames", "Cam007_rgb000015.png")


def test_png_round_trip_and_quantize(tmp_path):
    import cv2
    import torch

    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (13, 17, 3), dtype=np.uint8)
    E.write_frame_png(tmp_path / "f.png", torch.from_numpy(img))
    back = cv2.imread(str(tmp_path / "f.png"), cv2.IMREAD_UNCHANGED)
    assert np.array_equal(back[..., ::-1], img)                     # stored BGR, as Trainer.test writes it
    with pytest.raises(RuntimeError):
        E.write_frame_png(tmp_path / "missing_dir" / "f.png", img)
    c = torch.tensor([0.0, 0.5, 1.0, 0.999, 1 / 255, 2 / 255 - 1e-7])
    assert E.quantize(c).tolist() == (c.numpy() * 255).astype(np.uint8).tolist() == [0, 127, 255, 254, 1, 1]


def test_image_metrics_rejects_cpu_tensors():
    import torch

    x = torch.zeros(8, 8, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        E.image_metrics(x, x, torch.ones(8, 8, dtype=torch.uint8))
