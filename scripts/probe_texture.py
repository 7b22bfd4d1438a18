"""GPU experiment (test infrastructure): dump raw hardware tex3D values for controlled sub-texel offsets so the
1.8 fixed-point emulation can be fitted exactly.  usage: python scripts/probe_texture.py <output .npz>"""
import ctypes
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
lib = ctypes.CDLL(str(ROOT / "oracle/_build/libtexprobe.so"))
lib.tex_probe.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
dev = torch.device("cuda:0")


def hw(grid, pts):
    g = torch.from_numpy(grid).to(dev).contiguous()
    p = torch.from_numpy(pts.astype(np.float32)).to(dev).contiguous()
    out = torch.empty(p.shape[0], device=dev)
    torch.cuda.synchronize()
    assert lib.tex_probe(g.data_ptr(), grid.shape[0], p.data_ptr(), p.shape[0], out.data_ptr()) == 0
    return out.cpu().numpy()


out = {}
for G in (8, 64, 256):
    grid = np.zeros((G, G, G), np.uint8)
    c = G // 2
    grid[c, c, c] = 255
    ctr = (c + 0.5) / G
    # A: 1-D sweep along x in steps of 1/4096 texel
    s = np.arange(-5000, 5001) / 4096.0
    pts = np.stack([(c + 0.5 + s) / G, np.full_like(s, ctr), np.full_like(s, ctr)], 1)
    out[f"A_s_{G}"], out[f"A_v_{G}"] = s, hw(grid, pts)
    pts = np.stack([np.full_like(s, ctr), np.full_like(s, ctr), (c + 0.5 + s) / G], 1)
    out[f"Az_v_{G}"] = hw(grid, pts)
    # B: 2-D small weights: offsets 1 - (i+0.5)/256 (centre of the i-th weight bin)
    i = np.arange(0, 48)
    sx = 1.0 - (i + 0.5) / 256.0
    X, Y = np.meshgrid(sx, sx, indexing="ij")
    pts = np.stack([(c + 0.5 + X.ravel()) / G, (c + 0.5 + Y.ravel()) / G, np.full(X.size, ctr)], 1)
    out[f"B_v_{G}"] = hw(grid, pts).reshape(48, 48)
    # C: 3-D small weights
    i3 = np.arange(0, 24)
    s3 = 1.0 - (i3 + 0.5) / 256.0
    X, Y, Z = np.meshgrid(s3, s3, s3, indexing="ij")
    pts = np.stack([(c + 0.5 + X.ravel()) / G, (c + 0.5 + Y.ravel()) / G, (c + 0.5 + Z.ravel()) / G], 1)
    out[f"C_v_{G}"] = hw(grid, pts).reshape(24, 24, 24)
    # D: one small weight (bin i) times mid weights on the other axes
    mids = np.array([0.5, 0.25, 0.75, 0.1, 0.9])
    I, M1, M2 = np.meshgrid(1.0 - (np.arange(0, 32) + 0.5) / 256.0, mids, mids, indexing="ij")
    pts = np.stack([(c + 0.5 + I.ravel()) / G, (c + 0.5 + M1.ravel()) / G, (c + 0.5 + M2.ravel()) / G], 1)
    out[f"D_v_{G}"] = hw(grid, pts).reshape(32, 5, 5)
    # E: random points around the voxel + raw values
    rng = np.random.default_rng(0)
    r = rng.uniform(-1.1, 1.1, (200000, 3))
    pts = ((c + 0.5 + r) / G).astype(np.float32)
    out[f"E_p_{G}"], out[f"E_v_{G}"] = pts, hw(grid, pts)
# F: a 2x2x2 block of occupied voxels (sums of several small weights)
G = 64
grid = np.zeros((G, G, G), np.uint8)
grid[32:34, 32:34, 32:34] = 255
rng = np.random.default_rng(1)
r = rng.uniform(-1.2, 2.2, (300000, 3))
pts = ((32 + 0.5 + r) / G).astype(np.float32)
out["F_p"], out["F_v"] = pts, hw(grid, pts)
np.savez_compressed(sys.argv[1], **out)
print("wrote", sys.argv[1])
