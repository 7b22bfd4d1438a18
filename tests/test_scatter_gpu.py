"""The table / vector gradient scatter (hrf_field_backward_tables) in isolation, against float64 autograd through the
oracle's hash-grid encoding and tensor composition.  HRF_SCATTER picks the kernel: 6 = csrc/scatter_v6.cu, the one the
train step runs; 5 = csrc/scatter_v5.cu, the same lane-pair walk (csrc/scatter_pairs.cuh) over a different CTA shape,
kept as v6's second reference.  The kernels' only rounding is fp32 accumulation, so the bar is 1e-5 -- tight enough to
catch a single dropped or doubled corner contribution (the run-length accumulation and the shared-corner carry between
neighbouring cells are exactly where such a bug would sit).

The ragged-ray test runs both generations on two small temporal segments, with either feature source and several splits
of the 4 grids over launches.

v6 walks all grids of a launch inside one CTA, so its own test covers the cases that loop structure can get wrong: the
saved per-grid features read through a survivor index (egrid + feat_index, a column stride wider than the sample count)
and the re-gather path (egrid = NULL); one launch over the 4 grids and four one-grid launches (the overlapped exchange's
schedule); full-size tables with one and with three temporal segments; samples outside a dense level's grid (the cold
path); and a sample count that is not a multiple of the 1024 samples of a CTA."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import make_pair, positions_of, scatter_autograd_reference as _reference, scatter_workspace as _workspace
from helpers import segment_grads as _segment_grads, synthetic_rays
from humanrf_b200 import _lib as L
from oracle import field as OF

pytestmark = pytest.mark.gpu
CONFIGS = {"seg50": (50,), "seg100-100-50": (100, 100, 50)}


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _lerp_vectors(vectors, coords):
    """oracle.field.lerp_vectors with both taps clamped to the rows, as the kernels' make_tap does (coordinates outside
    [0, 1] reach the vectors here)."""
    vr = vectors.shape[1]
    out = []
    for i in range(4):
        c = coords[:, i] * vr - 0.5
        f = torch.floor(c)
        frac = (c - f).unsqueeze(1)
        i0 = torch.clamp(f, 0.0, vr - 1).long()
        i1 = torch.clamp(f + 1, 0.0, vr - 1).long()
        v0, v1 = vectors[i][i0], vectors[i][i1]
        out.append(v0 + frac * (v1 - v0))
    return torch.stack(out, 0)


def _bf16_bits(x):
    return (x.float().bfloat16().view(torch.int16).numpy().astype(np.int64) & 0xFFFF).astype(np.uint32)


def _bf16_model(segs, cuda):
    """An oracle / module pair with bf16-representable tables: the re-gather path reads the bf16 shadows."""
    om, m, frames = make_pair(segs, table_std=0.5, bf16=False, device=cuda)
    with torch.no_grad():
        for s, fg in enumerate(m.feature_grids):
            for k, g in enumerate(fg.grids()):
                q = g.detach().bfloat16().float()
                g.copy_(q)
                om.segments[s].grids[k] = q.cpu().reshape(-1, 2).clone()
    nat = m.native()
    nat.refresh()
    return om, m, nat, frames


def _saved_features(enc_all, g, cuda):
    """Saved per-(level, grid) features [16 * 4][stride] bf16x2, each sample at a shuffled column of a wider buffer."""
    n = enc_all.shape[0]
    stride = n + 37
    perm = torch.randperm(stride, generator=g)[:n]
    bits = _bf16_bits(enc_all)                                                 # [n, 4, 32]
    packed = bits[..., 0::2] | (bits[..., 1::2] << np.uint32(16))             # [n, 4 grids, 16 levels]
    egrid = np.zeros((64, stride), np.uint32)
    egrid[:, perm.numpy()] = packed.transpose(2, 1, 0).reshape(64, n)
    return stride, {"egrid": torch.from_numpy(egrid.view(np.int32)).to(cuda), "feat_index": perm.to(torch.int32).to(cuda)}


def _scatter(case, monkeypatch, gen, mode, schedule):
    """The kernel's gradients for one HRF_SCATTER generation, feature source and schedule of (grid_first, grid_count)."""
    monkeypatch.setenv("HRF_SCATTER", gen)
    nat = case["nat"]
    grads, sg_dev = _segment_grads(case["m"])
    eg, fi, stride = (case["dev"]["egrid"].data_ptr(), case["dev"]["feat_index"].data_ptr(), case["stride"]) if mode == "egrid" else (None, None, 0)
    for first, count in schedule:
        L.check(L.lib().hrf_field_backward_tables(C.byref(nat.field), C.byref(case["samples"]), sg_dev.data_ptr(), eg, fi, stride,
                                                  case["ws"].data_ptr(), first, count, L.stream()))
    torch.cuda.synchronize()
    return [g.cpu() for g in grads]


@pytest.fixture(scope="module")
def ragged(cuda):
    om, m, nat, frames = _bf16_model((6, 6), cuda)
    b = synthetic_rays(96, 48, frames, ragged=True, seed=21)   # consecutive samples of a ray: neighbouring cells at the fine levels
    pos, fr = positions_of(b), b["frames"][b["ri"]]
    n = pos.shape[0]
    seg = om.f2s[fr.numpy()]
    xyzt = torch.cat((pos + 0.5, torch.from_numpy(om.f2t[fr.numpy()]).unsqueeze(1)), dim=1).float()
    g = torch.Generator().manual_seed(2)
    d_out = torch.randn(n, 32, generator=g)
    d_out[::7] = 0                                            # zero upstream gradients are skipped, not scattered
    # fp32 tap arithmetic (exact: vec_res is a power of two), float64 blend
    ref_tables, ref_vec, enc_all = _reference(om, seg, xyzt, d_out, OF.lerp_vectors)
    stride, dev = _saved_features(enc_all, g, cuda)
    samples = nat.samples_query(pos.to(cuda).contiguous(), None, fr.to(cuda).to(torch.int32).contiguous())
    return dict(m=m, nat=nat, samples=samples, ws=_workspace(d_out, xyzt, seg, cuda), stride=stride, dev=dev,
                ref_tables=ref_tables, ref_vec=ref_vec)


SCHEDULES = {"split": ((0, 1), (1, 3)), "one": ((0, 4),), "four": ((0, 1), (1, 1), (2, 1), (3, 1)), "pairs": ((0, 2), (2, 2))}
RAGGED = [(gen, mode, sched) for gen in ("5", "6") for mode in ("gather", "egrid") for sched in SCHEDULES]


@pytest.mark.parametrize("gen,mode,sched", RAGGED, ids=[f"v{g_}-{'regather' if m_ == 'gather' else 'egrid+feat_index'}-{s_}" for g_, m_, s_ in RAGGED])
def test_table_scatter_matches_float64_autograd(ragged, monkeypatch, gen, mode, sched):
    """Ragged rays over two temporal segments of 6 frames, for both generations, both feature sources (the re-gather of
    the bf16 tables; the saved per-grid features read through a survivor index) and several splits of the 4 grids over
    launches (the per-table schedules)."""
    grads = _scatter(ragged, monkeypatch, gen, mode, SCHEDULES[sched])
    for s in range(len(ragged["ref_tables"])):
        for k in range(4):
            got, ref = grads[5 * s + k], ragged["ref_tables"][s][k]
            assert ((got != 0) & (ref == 0)).sum() == 0, "gradient written to an untouched table entry"
            e = _relnorm(got, ref)
            worst = float((got.double() - ref).abs().max() / ref.abs().max())
            print(f"v{gen} {mode} {sched} seg{s} grid{k}: relnorm {e:.2e} worst entry {worst:.2e} touched {(ref != 0).sum().item()}")
            assert e < 1e-5 and worst < 1e-5
        e = _relnorm(grads[5 * s + 4], ragged["ref_vec"][mode][s])
        print(f"v{gen} {mode} {sched} seg{s} vectors: relnorm {e:.2e}")
        assert e < 1e-5


@pytest.fixture(scope="module", params=list(CONFIGS), ids=list(CONFIGS))
def case(request, cuda):
    segs = CONFIGS[request.param]
    om, m, nat, frames = _bf16_model(segs, cuda)
    b = synthetic_rays(72, 96, frames, ragged=True, seed=31)
    pos, fr = positions_of(b), b["frames"][b["ri"]]
    # samples outside the dense levels' grids (x beyond 1 or below 0 after the +0.5): the kernels' cold path
    g = torch.Generator().manual_seed(4)
    pick = torch.randint(0, pos.shape[0], (96,), generator=g)
    out_pos = pos[pick].clone()
    out_pos[:48, 0] = 0.5 + 0.005 + 0.03 * torch.rand(48, generator=g)
    out_pos[48:, 0] = -0.5 - 0.02 - 0.03 * torch.rand(48, generator=g)
    pos, fr = torch.cat((pos, out_pos)), torch.cat((fr, fr[pick]))
    if pos.shape[0] % 1024 == 0:
        pos, fr = pos[:-1], fr[:-1]
    n = pos.shape[0]
    assert n > 2048 and n % 1024 != 0
    seg = om.f2s[fr.numpy()]
    if len(segs) > 1:
        assert len(np.unique(seg)) > 1
    xyzt = torch.cat((pos + 0.5, torch.from_numpy(om.f2t[fr.numpy()]).unsqueeze(1)), dim=1).float()
    d_out = torch.randn(n, 32, generator=g)
    d_out[::7] = 0                                            # zero upstream gradients are skipped, not scattered
    ref_tables, ref_vec, enc_all = _reference(om, seg, xyzt, d_out, _lerp_vectors)   # (coordinates outside [0, 1] here)
    stride, dev = _saved_features(enc_all, g, cuda)
    samples = nat.samples_query(pos.to(cuda).contiguous(), None, fr.to(cuda).to(torch.int32).contiguous())
    return dict(m=m, nat=nat, samples=samples, ws=_workspace(d_out, xyzt, seg, cuda), stride=stride, dev=dev,
                ref_tables=ref_tables, ref_vec=ref_vec)


@pytest.mark.parametrize("launches", ["one", "four"], ids=["grid_count4", "4x_grid_count1"])
@pytest.mark.parametrize("mode", ["egrid", "gather"], ids=["egrid+feat_index", "regather"])
def test_scatter_v6_matches_float64_autograd_and_v5(cuda, monkeypatch, case, mode, launches):
    got6 = _scatter(case, monkeypatch, "6", mode, SCHEDULES["one" if launches == "one" else "four"])
    got5 = _scatter(case, monkeypatch, "5", mode, SCHEDULES["one"])
    for s in range(len(case["ref_tables"])):
        for k in range(4):
            g6, g5, ref = got6[5 * s + k], got5[5 * s + k], case["ref_tables"][s][k]
            assert ((g6 != 0) & (ref == 0)).sum() == 0, "gradient written to an untouched table entry"
            e = _relnorm(g6, ref)
            worst = float((g6.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
            e5 = _relnorm(g6, g5)
            print(f"{mode} {launches} seg{s} grid{k}: relnorm {e:.2e} worst entry {worst:.2e} vs v5 {e5:.2e} touched {(ref != 0).sum().item()}")
            assert e < 1e-5 and worst < 1e-5 and e5 < 1e-5
        ev = _relnorm(got6[5 * s + 4], case["ref_vec"][mode][s])
        ev5 = _relnorm(got6[5 * s + 4], got5[5 * s + 4])
        print(f"{mode} {launches} seg{s} vectors: relnorm {ev:.2e} vs v5 {ev5:.2e}")
        assert ev < 1e-5 and ev5 < 1e-5
