"""float64 restatement of the ActorsHQ evaluation's image scores (actorshq/evaluation/evaluate.py:76-85,117-125): the
mask's bounding rectangle, the crop, the masked PSNR, and scikit-image's ``structural_similarity(gt, pred,
channel_axis=2)`` with its defaults for uint8 images, written out with ``scipy.ndimage.uniform_filter`` as scikit-image
implements it (scikit-image itself is not a dependency of the project)."""
import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
K1, K2 = 0.01, 0.03


def bounding_rect(mask):
    """cv2.boundingRect of the non-zero pixels of an [H,W] mask: (x, y, w, h), (0, 0, 0, 0) when there are none."""
    ys, xs = np.nonzero(np.asarray(mask))
    if len(xs) == 0:
        return (0, 0, 0, 0)
    return (int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1))


def psnr(pred, gt, mask):
    """-10 log10 of the mean over masked pixels of the channel mean of ((p - g) / 255)^2; NaN without masked pixels."""
    m = np.asarray(mask) != 0
    if not m.any():
        return float("nan")
    e = (((pred.astype(np.float64) - gt.astype(np.float64)) / 255.0) ** 2).mean(axis=2)
    mse = e[m].mean()
    return float("inf") if mse == 0 else float(-10.0 * np.log10(mse))


def ssim_channel(x, y, data_range=255.0):
    """scikit-image's structural_similarity of two 2-D images (gaussian_weights False, use_sample_covariance True)."""
    x, y = x.astype(np.float64), y.astype(np.float64)
    np_ = WIN ** 2
    cov_norm = np_ / (np_ - 1)
    ux, uy = uniform_filter(x, size=WIN), uniform_filter(y, size=WIN)
    uxx, uyy, uxy = uniform_filter(x * x, size=WIN), uniform_filter(y * y, size=WIN), uniform_filter(x * y, size=WIN)
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    A1, A2, B1, B2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
    S = (A1 * A2) / (B1 * B2)
    pad = (WIN - 1) // 2
    return float(S[pad:-pad, pad:-pad].mean(dtype=np.float64))


def ssim(gt, pred):
    """Mean over the 3 channels of ssim_channel; NaN where scikit-image raises (an image under 7 pixels either way)."""
    if gt.shape[0] < WIN or gt.shape[1] < WIN:
        return float("nan")
    return float(np.mean([ssim_channel(gt[..., c], pred[..., c]) for c in range(gt.shape[2])]))


def evaluate_pair(pred, gt, mask):
    """(PSNR, SSIM, roi) of uint8 [H,W,3] images under an [H,W] mask, cropped to the mask's bounding rectangle."""
    roi = bounding_rect(mask)
    x, y, w, h = roi
    if w == 0:
        return float("nan"), float("nan"), roi
    crop = lambda a: a[y:y + h, x:x + w]
    return psnr(crop(pred), crop(gt), crop(np.asarray(mask))), ssim(crop(gt), crop(pred)), roi
