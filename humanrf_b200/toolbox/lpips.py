"""LPIPS (AlexNet, v0.1) of rendered views on the GPU, as the ActorsHQ evaluation and the reference trainer compute it.

``lpips`` scores one image pair with ``hrf_lpips`` (csrc/lpips.cu, contract in include/humanrf_b200.h): the number
``lpips.LPIPS(net="alex", version="0.1")(gt, pred, normalize=True)`` gives on the ROI crop of both images, with every
convolution on TF32 tensor cores (torch's own default for cuDNN convolutions on Ampere and later GPUs).
``load_lpips_alex`` reads the two weight files the reference's evaluation downloads: torchvision's AlexNet checkpoint
and lpips' ``weights/v0.1/alex.pth``.  The ``lpips`` package itself is not needed.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import torch

from .. import _lib as L

CONV_KEYS = ("features.0", "features.3", "features.6", "features.8", "features.10")
CONV_SHAPES = ((64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3))
LIN_KEYS = tuple(f"lin{k}.model.1.weight" for k in range(5))
# the eight tensors of the workspace (include/humanrf_b200.h, hrf_lpips): name and channels
TENSORS = (("input", 4), ("conv1", 64), ("pool1", 64), ("conv2", 192), ("pool2", 192), ("conv3", 384), ("conv4", 256),
           ("conv5", 256))


@dataclass
class LpipsAlex:
    """Packed AlexNet convolution weights plus the fp32 biases and lin weights, on one CUDA device."""
    packed: torch.Tensor        # uint8 [hrf_lpips_packed_bytes()]
    bias: tuple                 # 5 x fp32 [C]
    lin: tuple                  # 5 x fp32 [C]

    @property
    def device(self) -> torch.device:
        return self.packed.device

    def _struct(self) -> L.LpipsWeights:
        return L.LpipsWeights(self.packed.data_ptr(), (L.vp * 5)(*[b.data_ptr() for b in self.bias]),
                              (L.vp * 5)(*[w.data_ptr() for w in self.lin]))


def _tensor(sd, key, shape, what):
    if key not in sd:
        raise RuntimeError(f"{what}: missing key {key}")
    t = sd[key]
    if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape):
        got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise RuntimeError(f"{what}: {key} has shape {got}, expected {tuple(shape)}")
    if not t.is_floating_point():
        raise RuntimeError(f"{what}: {key} has dtype {t.dtype}, expected a floating-point tensor")
    return t


def lpips_alex_from_state_dicts(alexnet_state, lin_state, device="cuda") -> LpipsAlex:
    """``LpipsAlex`` from torchvision's AlexNet state dict (``features.{0,3,6,8,10}.{weight,bias}``; other keys are
    ignored) and lpips' v0.1 lin state dict (``lin{0..4}.model.1.weight``, ``[1,C,1,1]``).  Every key and shape is
    checked before anything reaches the device."""
    convs, biases, lins = [], [], []
    for key, shape in zip(CONV_KEYS, CONV_SHAPES):
        convs.append(_tensor(alexnet_state, key + ".weight", shape, "alexnet weights"))
        biases.append(_tensor(alexnet_state, key + ".bias", shape[:1], "alexnet weights"))
    for key, shape in zip(LIN_KEYS, CONV_SHAPES):
        lins.append(_tensor(lin_state, key, (1, shape[0], 1, 1), "lpips lin weights"))
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("LPIPS weights must go to a CUDA device")
    f32 = dict(dtype=torch.float32, device=dev)
    convs = [w.detach().to(**f32).contiguous() for w in convs]
    packed = torch.empty(int(L.lib().hrf_lpips_packed_bytes()), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(L.lib().hrf_lpips_pack_weights((L.vp * 5)(*[w.data_ptr() for w in convs]), packed.data_ptr(),
                                               L.stream()))
    return LpipsAlex(packed, tuple(b.detach().to(**f32).contiguous() for b in biases),
                     tuple(w.detach().to(**f32).reshape(-1).contiguous() for w in lins))


def load_lpips_alex(alexnet_path, lin_path, device="cuda") -> LpipsAlex:
    """Loads torchvision's ``alexnet-owt-7be5be79.pth`` and lpips' ``weights/v0.1/alex.pth`` (``torch.load`` with
    ``weights_only=True``) and packs them for ``lpips`` on `device`."""
    alexnet_state = torch.load(os.path.expanduser(str(alexnet_path)), map_location="cpu", weights_only=True)
    lin_state = torch.load(os.path.expanduser(str(lin_path)), map_location="cpu", weights_only=True)
    return lpips_alex_from_state_dicts(alexnet_state, lin_state, device)


def _check_image(t, name):
    if (not isinstance(t, torch.Tensor) or t.dim() != 3 or t.shape[2] != 3 or t.dtype not in (torch.uint8, torch.float32)
            or t.device.type != "cuda" or not t.is_contiguous()):
        raise RuntimeError(f"{name} must be a contiguous uint8 or float32 [H,W,3] CUDA tensor")


def workspace_bytes(width: int, height: int) -> int:
    """Device scratch ``lpips`` needs for a `width` x `height` image (any ROI): about 1.6 GB at 4112x3008."""
    return int(L.lib().hrf_lpips_workspace_bytes(width, height))


def lpips(pred: torch.Tensor, gt: torch.Tensor, weights: LpipsAlex, roi: torch.Tensor | None = None,
          out: torch.Tensor | None = None, workspace: torch.Tensor | None = None) -> torch.Tensor:
    """LPIPS (AlexNet, v0.1, normalize=True) of `pred` against `gt`: contiguous [H,W,3] RGB tensors of one dtype on one
    CUDA device, uint8 (scaled by 1/255) or float32 in [0, 1].  `roi` is a device int32 [4] (x, y, w, h), e.g. the one
    ``image_metrics`` returns; ``None`` scores the whole image.  Returns a float64 device scalar without synchronising;
    `out` (a float64 one-element tensor, e.g. an element of a larger one) is written in place when given.  The score is
    NaN when the ROI is under 31 pixels wide or tall (lpips raises there) or does not lie inside the image.  `workspace`
    (uint8, at least ``workspace_bytes(W, H)``) may be given to keep the layer outputs (``workspace_tensors``)."""
    _check_image(pred, "pred")
    _check_image(gt, "gt")
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if gt.shape != pred.shape or gt.dtype != pred.dtype:
        raise RuntimeError(f"gt is {gt.dtype} {tuple(gt.shape)}, pred {pred.dtype} {tuple(pred.shape)}: they must match")
    dev = pred.device
    if gt.device != dev or weights.device != dev:
        raise RuntimeError("pred, gt and the LPIPS weights must be on one device")
    if W * H * 3 >= 1 << 31:
        raise RuntimeError(f"{W}x{H} image too large (width * height * 3 must be under 2^31)")
    if roi is not None and (not isinstance(roi, torch.Tensor) or roi.dtype != torch.int32 or roi.device != dev
                            or roi.numel() != 4 or not roi.is_contiguous()):
        raise RuntimeError(f"roi must be a contiguous int32 [4] tensor on {dev}")
    if out is None:
        out = torch.empty((), dtype=torch.float64, device=dev)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float64 or out.device != dev or out.numel() != 1):
        raise RuntimeError(f"out must be a one-element float64 tensor on {dev}")
    need = workspace_bytes(W, H)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.uint8, device=dev)
    elif (not isinstance(workspace, torch.Tensor) or workspace.dtype != torch.uint8 or workspace.device != dev
          or not workspace.is_contiguous() or workspace.numel() < need or workspace.data_ptr() % 256):
        raise RuntimeError(f"workspace must be a contiguous, 256-byte aligned uint8 tensor of >= {need} bytes on {dev}")
    with torch.cuda.device(dev):
        L.check(L.lib().hrf_lpips(C.byref(weights._struct()), pred.data_ptr(), gt.data_ptr(),
                                  0 if pred.dtype == torch.uint8 else 1, W, H, L.ptr(roi), out.data_ptr(),
                                  workspace.data_ptr(), L.stream()))
    return out


def _conv1(n):
    return (n - 7) // 4 + 1 if n >= 7 else 0


def _pool(n):
    return (n - 3) // 2 + 1 if n >= 3 else 0


def tensor_sizes(w: int, h: int):
    """(h, w) of the workspace's eight tensors for a w x h crop, in the order of ``TENSORS``."""
    d = [(h, w), (_conv1(h), _conv1(w))]
    d += [(_pool(d[1][0]), _pool(d[1][1]))] * 2
    d += [(_pool(d[3][0]), _pool(d[3][1]))] * 4
    return d


def workspace_tensors(workspace: torch.Tensor, width: int, height: int, roi_w: int, roi_h: int) -> dict:
    """Views of the eight fp32 NHWC tensors ``lpips`` left in `workspace` for a `width` x `height` image and a
    `roi_w` x `roi_h` ROI: name -> [2, h, w, C] (image 0 = pred, 1 = gt), laid out as include/humanrf_b200.h states."""
    full, crop = tensor_sizes(width, height), tensor_sizes(roi_w, roi_h)
    views, off = {}, 0
    for (name, c), (fh, fw), (h, w) in zip(TENSORS, full, crop):
        views[name] = workspace[off:off + 2 * h * w * c * 4].view(torch.float32).view(2, h, w, c)
        off += -(-2 * fh * fw * c * 4 // 256) * 256
    return views
