"""Float64 reference of LPIPS (lpips.LPIPS(net="alex", version="0.1"), normalize=True), test-only.

The trunk is torchvision's own ``alexnet(weights=None).features``; the input scaling and the tail are restated from
lpips' published v0.1 source (``ScalingLayer``, ``normalize_tensor``, ``NetLinLayer``, ``spatial_average``), which is
not installable here.  With ``tf32=True`` every convolution operand is rounded to TF32 (nearest, ties away from zero)
exactly where csrc/lpips.cu rounds: the scaled input, the packed weights and each ReLU output; everything else is exact
float64.  The product never imports this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

CONV_KEYS = ("features.0", "features.3", "features.6", "features.8", "features.10")
CONV_SPECS = ((4, 2), (1, 2), (1, 1), (1, 1), (1, 1))          # stride, padding
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
LIN_CHANNELS = (64, 192, 384, 256, 256)


def rna_tf32(x):
    """fp32 -> tf32 (10 mantissa bits), nearest with ties away from zero, as ``cvt.rna.tf32.f32``: add half an ulp to
    the magnitude bits and truncate.  Inf and NaN pass unchanged; a finite value that rounds past the largest finite
    float becomes inf.  numpy float32 arrays or torch float32 tensors."""
    if isinstance(x, torch.Tensor):
        assert x.dtype == torch.float32
        u = x.view(torch.int32)
        finite = torch.isfinite(x)
        r = ((u + 0x1000) & -8192).view(torch.float32)
        return torch.where(finite, r, x)
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32)
    r = ((u.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)
    return np.where(np.isfinite(x), r, x)


def scale_input(img) -> np.ndarray:
    """Step 1 in numpy float32: [H,W,3] uint8 (v = u / 255, correctly rounded) or float32 (v as given) -> x = 2v - 1 ->
    (x - shift) / scale, returned [3,H,W] float32, RGB."""
    img = np.asarray(img)
    v = img.astype(np.float32) / np.float32(255.0) if img.dtype == np.uint8 else img.astype(np.float32)
    x = v * np.float32(2.0) - np.float32(1.0)
    shift = np.array(SHIFT, np.float32)[:, None, None]
    scale = np.array(SCALE, np.float32)[:, None, None]
    return np.ascontiguousarray((x.transpose(2, 0, 1) - shift) / scale)


def seeded_state_dicts(seed: int = 0):
    """torchvision ``alexnet(weights=None)``'s state dict from a seeded init and seeded non-negative lin weights in
    lpips' layout (``lin{k}.model.1.weight``, [1,C,1,1]): the two weight files' formats, with random values."""
    import torchvision

    torch.manual_seed(seed)
    alex = torchvision.models.alexnet(weights=None).state_dict()
    g = torch.Generator().manual_seed(seed + 1)
    # a distinct scale per layer, as trained lin weights have: exchangeable layers would hide a swapped layer
    lin = {f"lin{k}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) * (0.1 * 2 ** k)
           for k, c in enumerate(LIN_CHANNELS)}
    return alex, lin


class Oracle:
    """LPIPS in float64 on `device` (CPU, or a GPU through torch to keep the large cases fast)."""

    def __init__(self, alex_state, lin_state, device="cpu", tf32=False):
        import torchvision

        self.device, self.tf32, self.specs = torch.device(device), tf32, list(CONV_SPECS)
        feats = torchvision.models.alexnet(weights=None).features[:12]
        feats.load_state_dict({k[len("features."):]: v for k, v in alex_state.items() if k.startswith("features.")})
        self.features = feats.double().to(self.device).eval()
        self.w, self.b = [], []
        for k in CONV_KEYS:
            w = alex_state[k + ".weight"].float()
            self.w.append((rna_tf32(w) if tf32 else w).double().to(self.device))
            self.b.append(alex_state[k + ".bias"].float().double().to(self.device))
        self.lin = [lin_state[f"lin{k}.model.1.weight"].float().double().reshape(-1).to(self.device) for k in range(5)]

    def trunk_torchvision(self, x):
        """The five ReLU outputs of torchvision's module itself, applied layer by layer."""
        out = []
        for i, m in enumerate(self.features):
            x = m(x)
            if i in (1, 4, 7, 9, 11):
                out.append(x)
        return out

    def trunk(self, x):
        """The five ReLU outputs for a float64 [N,3,H,W] input, restated with F.conv2d so that each output can be
        rounded where the kernel rounds it."""
        out = []
        for k in range(5):
            if k in (1, 2):
                x = F.max_pool2d(x, 3, 2)
            s, p = self.specs[k]
            x = torch.relu(F.conv2d(x, self.w[k], self.b[k], stride=s, padding=p))
            if self.tf32:
                x = rna_tf32(x.float()).double()      # the fp32 epilogue output, rounded
            out.append(x)
        return out

    def prepare(self, img, roi=None):
        """Scaled float64 [1,3,h,w] input of an [H,W,3] uint8 / float32 image cropped to roi (x, y, w, h)."""
        img = np.asarray(img)
        if roi is not None:
            x, y, w, h = roi
            img = img[y:y + h, x:x + w]
        s = scale_input(img)
        if self.tf32:
            s = rna_tf32(s)
        return torch.from_numpy(s.astype(np.float64))[None].to(self.device)

    def layer_scores(self, feats0, feats1):
        """The five spatial means of sum_c lin (f0 - f1)^2."""
        d = []
        for k, (a, b) in enumerate(zip(feats0, feats1)):
            na = a / (torch.sqrt((a * a).sum(1, keepdim=True)) + 1e-10)
            nb = b / (torch.sqrt((b * b).sum(1, keepdim=True)) + 1e-10)
            d.append(float((self.lin[k][None, :, None, None] * (na - nb) ** 2).sum(1).mean()))
        return d

    def __call__(self, pred, gt, roi=None) -> float:
        """LPIPS of two [H,W,3] images (uint8 or float32) over roi; NaN when the crop is under 31x31 pixels."""
        w, h = (np.asarray(pred).shape[1], np.asarray(pred).shape[0]) if roi is None else roi[2:]
        if w < 31 or h < 31:
            return float("nan")
        with torch.no_grad():
            f0 = self.trunk(self.prepare(pred, roi))
            f1 = self.trunk(self.prepare(gt, roi))
            return float(sum(self.layer_scores(f0, f1)))


# ---- test pairs shared by the CPU and GPU tests ---------------------------------------------------------------------------
def _blur(img):
    from scipy.ndimage import uniform_filter

    return np.clip(np.rint(uniform_filter(img.astype(np.float64), size=(5, 5, 1), mode="reflect")), 0, 255).astype(np.uint8)


def base_image(W, H, seed):
    """Smooth colour gradients plus texture and a few hard edges: a stand-in for a rendered view."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.empty((H, W, 3))
    for c in range(3):
        fx, fy, ph = rng.uniform(2, 9), rng.uniform(2, 9), rng.uniform(0, 6.3)
        img[..., c] = 127 + 90 * np.sin(2 * np.pi * fx * x / W + ph) * np.cos(2 * np.pi * fy * y / H)
    img += rng.normal(0, 12, img.shape)
    img[H // 3:H // 2, W // 4:W // 2] = rng.uniform(0, 255, 3)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


PAIR_KINDS = ("noise", "blur", "quantised", "saturated", "unrelated")


def make_pair(kind, W, H, seed=0):
    """(pred, gt) [H,W,3] of one kind; "quantised" is a float32 render against its own 8-bit truncation."""
    rng = np.random.default_rng(seed + 17)
    gt = base_image(W, H, seed)
    if kind == "noise":
        pred = np.clip(gt.astype(np.int32) + np.rint(rng.normal(0, 8, gt.shape)).astype(np.int32), 0, 255).astype(np.uint8)
    elif kind == "blur":
        pred = _blur(gt)
    elif kind == "quantised":
        f = (gt.astype(np.float32) + rng.random(gt.shape, dtype=np.float32)) / np.float32(256.0)
        return f, ((f * 255).astype(np.uint8).astype(np.float32) / np.float32(255.0))
    elif kind == "saturated":
        pred = gt.copy()
        bh, bw = max(1, H // 4), max(1, W // 4)
        pred[:bh, :bw] = 255
        gt = gt.copy()
        gt[H - bh:, W - bw:] = 0
        pred[H - bh:, :bw] = 0
        pred[H // 2:H // 2 + bh, W // 2:W // 2 + bw] = 255
    elif kind == "unrelated":
        pred = base_image(W, H, seed + 1000)
    else:
        raise ValueError(kind)
    return pred, gt
