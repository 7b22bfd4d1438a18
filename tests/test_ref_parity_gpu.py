"""Differential tests against builds of the reference's first-party CUDA (oracle/build_ref.py compiles its unmodified
sources; ray_sampler.cu through oracle/glm_shim).  What those builds compute on the seeded inputs below is stored in
tests/golden/ref_parity.npz by tests/golden/make_ref_parity_golden.py, which runs every `reference_*` function of this
module and of test_occupancy_tools_gpu.py on a GPU where oracle/_ref was built; the tests run our kernels on the same
inputs and compare."""
from pathlib import Path

import numpy as np
import pytest
import torch

from scene import make_scene

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden" / "ref_parity.npz"


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _composition_inputs(cuda):
    g = torch.Generator().manual_seed(0)
    n, F, VR = 5000, 32, 2048
    feats = [torch.randn(n, F, generator=g).half().to(cuda) for _ in range(4)]
    vec = (torch.randn(4, VR, F, generator=g) * 0.1).to(cuda)
    coords = torch.rand(n, 4, generator=g)
    coords[:50] = 0.0; coords[50:100] = 1.0                      # clamped taps at both ends
    coords[:, 3] = torch.randint(0, 6, (n,), generator=g).float() / 6   # few distinct time taps (atomic contention)
    coords = coords.to(cuda)
    dout = torch.randn(n, F, generator=g).half().to(cuda)
    # the stored sample: 1000 of the 5000 rows of every per-sample output, 8192 of the 262 144 vector gradients
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:1000].to(cuda)
    vec_idx = torch.randperm(4 * VR * F, generator=torch.Generator().manual_seed(2))[:8192].to(cuda)
    return feats, vec, coords, dout, rows, vec_idx


def _composition(mod, cuda):
    feats, vec, coords, dout, rows, vec_idx = _composition_inputs(cuda)
    fwd = mod.compose_tensors_forward(*feats, vec, coords)
    bwd = mod.compose_tensors_backward(*feats, vec, coords, dout)
    torch.cuda.synchronize()
    out = {"comp/fwd": fwd[rows], "comp/dvec": bwd[4].reshape(-1)[vec_idx], "comp/dvec_absmax": bwd[4].abs().max()}
    out.update({f"comp/dfeat{k}": bwd[k][rows] for k in range(4)})
    return {k: v.cpu().numpy() for k, v in out.items()}


def reference_composition(ref, cuda):
    return _composition(ref("tensor_composition_native"), cuda)


def test_tensor_composition_matches_reference_extension(cuda, gold):
    from humanrf_b200.scene_representation import tensor_composition_native as ours

    b = _composition(ours, cuda)
    a = {k: gold[k] for k in b}
    diff = np.abs(a["comp/fwd"].astype(np.float32) - b["comp/fwd"].astype(np.float32))
    print("compose fwd max abs diff", diff.max())
    assert (diff <= 2e-3 * np.abs(a["comp/fwd"].astype(np.float32)) + 1e-6).all()   # <= 1-2 fp16 ulp (reference: --use_fast_math)
    for k in range(4):
        x, y = a[f"comp/dfeat{k}"].astype(np.float32), b[f"comp/dfeat{k}"].astype(np.float32)
        assert (np.abs(x - y) <= 2e-3 * np.abs(x) + 1e-6).all()
    np.testing.assert_allclose(b["comp/dvec"], a["comp/dvec"], rtol=2e-3, atol=2e-3 * float(a["comp/dvec_absmax"]))


def _sampler(rs, og_cls, cuda):
    """One get_samples_occupancy_minmax call over 8192 random pixels of a 3-image scene; the outputs the test compares."""
    sc = make_scene(num_images=3, width=128, height=96, G=128)
    B = len(sc["grids"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    og = og_cls(sc["G"], B)
    grids_dev = [t(g) for g in sc["grids"]]
    handles = torch.tensor([og.add_grid(g) for g in grids_dev], dtype=torch.int64, device=cuda)
    rng = np.random.default_rng(1)
    idx = torch.from_numpy(rng.integers(0, B * 128 * 96, 8192).astype(np.int64)).to(cuda)
    rgba, lm = torch.from_numpy(sc["rgba_big"]) if "rgba_big" in sc else torch.from_numpy(
        rng.integers(0, 256, (B * 128 * 96, 4)).astype(np.uint8)), torch.zeros(B * 128 * 96, dtype=torch.bool)
    common = (t(sc["frame_numbers"]), t(sc["camera_numbers"]))
    tail = (t(sc["landscape"]), idx, t(sc["inverse_krs"]), t(sc["camera_origins"]), t(sc["aabb"]), sc["G"], 128, 96, 4e-4, False)
    a = rs.get_samples_occupancy_minmax(rgba, lm, *common, handles, *tail)
    torch.cuda.synchronize()
    mask = a[6].cpu().numpy()
    out = {"mask": mask, "dirs": a[1].cpu().numpy(), "rgba": a[2].cpu().numpy(), "frames": a[3].cpu().numpy(),
           "minmax": a[5].cpu().numpy(), "counts": np.bincount(a[8].cpu().numpy(), minlength=mask.sum()),
           "num_samples": np.array(a[7].numel()), "dtypes": np.array([str(a[k].dtype) for k in (6, 7, 8)])}
    del og
    return {f"sampler/{k}": v for k, v in out.items()}


def reference_sampler(ref, cuda):
    return _sampler(ref("ray_sampler_native"), ref("occupancy_grid_native").OccupanyGrid, cuda)


def test_sampler_against_reference_build(cuda, gold):
    """Measured mismatch of the canonical-IEEE sampler vs the reference's --use_fast_math + hardware-texture build."""
    from humanrf_b200.dataset import ray_sampler_native as rs
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    b = _sampler(rs, OccupanyGrid, cuda)
    a = {k: gold[k] for k in b}
    ma, mb = a["sampler/mask"], b["sampler/mask"]
    mask_mismatch = (ma != mb).mean()
    both = ma & mb
    # per-ray comparison on rays both keep
    ia, ib = np.cumsum(ma) - 1, np.cumsum(mb) - 1
    sel_a, sel_b = ia[both], ib[both]
    da, db = a["sampler/dirs"][sel_a], b["sampler/dirs"][sel_b]
    mma, mmb = a["sampler/minmax"][sel_a], b["sampler/minmax"][sel_b]
    ca, cb = a["sampler/counts"][sel_a], b["sampler/counts"][sel_b]
    na, nb = int(a["sampler/num_samples"]), int(b["sampler/num_samples"])
    print(f"ray-mask mismatch rate {mask_mismatch:.2e}; dir max|d| {np.abs(da - db).max():.2e}; "
          f"tmin/tmax max|d| {np.abs(mma - mmb).max():.2e}; rays with different sample count {(ca != cb).mean():.2e}; "
          f"total samples ref {na} ours {nb}")
    np.testing.assert_array_equal(a["sampler/rgba"][sel_a], b["sampler/rgba"][sel_b])       # rgba gather
    np.testing.assert_array_equal(a["sampler/frames"][sel_a], b["sampler/frames"][sel_b])   # frame numbers
    assert a["sampler/dtypes"].tolist() == b["sampler/dtypes"].tolist()
    assert mask_mismatch < 5e-3
    assert np.abs(da - db).max() < 1e-5
    assert np.abs(mma - mmb).max() < 5e-3            # one coarse march step is 0.5/G = 3.9e-3
    assert (ca != cb).mean() < 0.05
    assert abs(na - nb) < 0.01 * na
