"""CPU restatement of the learned occupancy bake (include/humanrf_b200.h, hrf_bake_occupancy) on the oracle field.

TEST INFRASTRUCTURE ONLY: the reference has no learned occupancy, so this module states the contract itself, in fp32
on OracleModel.density, with torch.nn.functional.max_pool3d for the dilation."""
import numpy as np
import torch

f32 = np.float32


def bake_positions(x, y, z, G):
    """The 8 sub-sample positions of voxels (x, y, z) of a G^3 grid, float32 [n, 8, 3]; sub-sample a + 2b + 4c is offset
    by (a, b, c) / 2 of a voxel: p = fl(fl((i + 0.25 + 0.5 a) / G) - 0.5) in float32 (correctly rounded divide)."""
    s = np.arange(8)
    halves = [(s & 1), (s >> 1) & 1, (s >> 2) & 1]
    out = []
    for i, h in zip((x, y, z), halves):
        num = (np.asarray(i, f32)[:, None] + f32(0.25) + f32(0.5) * h.astype(f32)[None, :]).astype(f32)
        out.append(((num / f32(G)).astype(f32) - f32(0.5)).astype(f32))
    return np.stack(out, -1)


def bake_occupancy_grid(oracle_model, frame_number, hull, step=4e-4, alpha_thre=1e-4):
    """Learned occupancy grid (include/humanrf_b200.h, hrf_bake_occupancy) on OracleModel.density in fp32:
    every hull voxel's 8 sub-sample densities -> m = max -> live = 1 - exp(-m step) >= alpha_thre ->
    out = hull AND 26-neighbourhood dilation of live by one voxel.  hull: uint8 [G,G,G] ([z][y][x], non-zero =
    occupied).  Returns (out uint8 {0,255}, max_sigma float32, 0 outside the hull), numpy arrays."""
    hull = np.asarray(hull)
    G = hull.shape[0]
    z, y, x = np.nonzero(hull)
    max_sigma = np.zeros((G, G, G), f32)
    live = np.zeros((G, G, G), bool)
    if x.size:
        pos = torch.from_numpy(bake_positions(x, y, z, G).reshape(-1, 3))
        frames = torch.full((pos.shape[0],), int(frame_number), dtype=torch.int32)
        with torch.no_grad():
            sigma, _ = oracle_model.density(pos, frames)
        m = sigma.reshape(-1, 8).amax(1)
        max_sigma[z, y, x] = m.numpy()
        live[z, y, x] = ((1 - torch.exp(-m * step)) >= alpha_thre).numpy()
    dil = torch.nn.functional.max_pool3d(torch.from_numpy(live).float()[None, None], 3, stride=1, padding=1)[0, 0] > 0
    out = (hull != 0) & dil.numpy()
    return np.where(out, 255, 0).astype(np.uint8), max_sigma
