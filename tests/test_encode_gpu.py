"""The hash-grid encode of every field-kernel instantiation that writes features, bit for bit against the
rounding-faithful reference tests/encode_oracle.py.

Bars:
* per-grid features (egrid, what the backward scatter reads): bit-identical for every sample whose frame has a segment,
  at every level, grid and feature, no tolerance;
* composed features: each output's bf16 bits must be produced by one of the contraction variants nvcc may pick for the
  lerp and the four-term sum (encode_oracle.VARIANTS).  The share of outputs whose variants disagree is printed with
  the variants that reproduce every output, and must stay below 1 %, so the bar cannot quietly become loose;
* rows whose frame has no segment (frames outside the LUT, negative, or mapped to no segment) have all-zero composed
  features.  Their egrid columns are left unwritten by contract: nothing is asserted about them.
Every output buffer is filled with a sentinel (0xFFFF per bf16, a NaN the encode cannot produce) before each launch, so a
value the kernel did not write cannot pass as an earlier allocation's leftovers.

Inputs: bench-like ragged rays plus an edge set (tests/encode_oracle.py: positions whose fused scale * x + 0.5 lands on
an integer at each level, their fp32 neighbours, x in {0, smallest reachable, nextafter(1, 0), 1}, coordinates beyond the
unit cube on both sides up to |x| = 4, row taps clamped at both ends) over every frame of every segment and frames with
no segment; query and ray-batch form; make_pair tables, and a wide-exponent variant (tables and vectors scaled by
2^U(-24, 8), mixed signs, exact zeros).  Counts are not multiples of 128.
"""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import encode_oracle as E
from helpers import field_without_vectors_t as _no_vectors_t, make_pair, synthetic_rays
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
MODELS = {"6": (6,), "6-12": (6, 12), "50": (50,), "100": (100,), "100-100-50": (100, 100, 50)}
_CACHE = {}


# ------------------------------------------------------------------------------------------------------ set-up
def _widen(x: np.ndarray, rng) -> np.ndarray:
    y = (np.abs(x) * 2.0 ** rng.uniform(-24, 8, x.shape) * np.where(rng.random(x.shape) < 0.5, -1, 1)).astype(np.float32)
    y[rng.random(x.shape) < 0.05] = 0
    return y


def _model(key, tables):
    """(module on the GPU, reference arrays from its fp32 masters, frames) for a model and a table variant."""
    ck = ("model", key, tables)
    if ck not in _CACHE:
        for k in [k for k in _CACHE if k[0] == "model"]:
            del _CACHE[k]                                    # one model resident at a time
        segs = MODELS[key]
        _, m, frames = make_pair(segs, table_std=6.0)
        if tables == "wide":
            rng = np.random.default_rng(17)
            with torch.no_grad():
                for fg in m.feature_grids:
                    for g in fg.grids() + [fg.vectors]:
                        g.copy_(torch.from_numpy(_widen(g.cpu().numpy(), rng)))
        m.invalidate_native()
        m.native()
        fa = _field_arrays(m, frames, segs)
        _CACHE[ck] = (m, fa, frames)
    return _CACHE[ck]


def _field_arrays(m, frames, segs):
    grids = [[g.detach().cpu().numpy() for g in fg.grids()] for fg in m.feature_grids]
    vecs = [fg.vectors.detach().cpu().numpy() for fg in m.feature_grids]
    return E.field_from_fp32(grids, vecs, frames, segs)


def _other_frames(frames):
    lut = frames[-1] + 1
    return [0, frames[0] - 1, -1, -1000, lut, lut + 5]      # no segment, negative, beyond the LUT


def _batch(fa, frames, seed, rays=48, per_ray=64, edges=3001):
    """Ray-batch arrays (numpy): bench-like ragged rays over every frame, then one-sample edge rays (origin = the edge
    position, t = 0, so the loaded position is the edge position) cycling through every frame and the frames with no
    segment."""
    b = synthetic_rays(rays, per_ray, frames, seed=seed, ragged=True, n_distinct_frames=len(frames))
    rng = np.random.default_rng(seed)
    p = E.edge_positions(fa.levels, edges, rng)
    d = rng.standard_normal((edges, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    pool = np.array(list(frames) + _other_frames(frames), np.int32)
    fr = pool[np.arange(edges) % pool.size]
    o = np.concatenate((b["o"].numpy(), p))
    dd = np.concatenate((b["d"].numpy(), d))
    rf = np.concatenate((b["frames"].numpy().astype(np.int32), fr))
    bfr = b["frames"].numpy().copy()
    bfr[::5] = pool[-6:][np.arange(bfr[::5].size) % 6]       # some bench rays in no segment too
    rf[:rays] = bfr
    t = np.concatenate((b["t"].numpy(), np.zeros(edges, np.float32)))
    ri = np.concatenate((b["ri"].numpy(), rays + np.arange(edges))).astype(np.int64)
    return dict(o=o, d=dd, frames=rf, t=t.astype(np.float32), ri=ri, num_rays=rays + edges)


def _samples(nat, bt, form, cuda):
    """(hrf_samples, reference positions x [N,3], reference frames [N]) of a batch in the given form."""
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in bt.items() if k != "num_rays"}
    if form == "rays":
        x, fr = E.load_rays(bt["o"], bt["d"], bt["frames"], bt["t"], bt["ri"])
        return nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"]), x, fr
    pos = E.fadd(bt["o"][bt["ri"]], E.fmul(bt["t"][:, None], bt["d"][bt["ri"]]))   # volume_rendering.py:66-69
    fr = bt["frames"][bt["ri"]]
    s = nat.samples_query(torch.from_numpy(pos).to(cuda), None, torch.from_numpy(fr).to(cuda))
    x, fr = E.load_query(pos, fr)
    return s, x, fr


def _forward(field, s, n, cuda, impl=0):
    """hrf_field_forward (density only) into sentinel-filled buffers -> (feat u16 [N,32], egrid u32 [64,N])."""
    feat = torch.full((n * 32,), -1, dtype=torch.int16, device=cuda)
    eg = torch.full((64 * n,), -1, dtype=torch.int32, device=cuda)
    sigma = torch.empty(n, dtype=torch.float32, device=cuda)
    L.check(L.lib().hrf_field_forward(C.byref(field), C.byref(s), 0, impl, sigma.data_ptr(), None, None, feat.data_ptr(),
                                      eg.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    return feat.cpu().numpy().view(np.uint16).reshape(n, 32), eg.cpu().numpy().view(np.uint32).reshape(64, n)


def _check(tag, fa, x, fr, feat, egrid, rows=None):
    """Both bars on the rows `rows` (default: all).  Returns the reference encoding."""
    if rows is not None:
        x, fr, feat, egrid = x[rows], fr[rows], feat[rows], egrid[:, rows]
    enc = E.encode(fa, x, fr, feat_gpu=feat)
    c = enc.check
    no_seg = enc.seg < 0
    assert (feat[no_seg] == 0).all(), f"{tag}: rows with no segment must be zero"
    em = E.egrid_mismatch(enc, egrid)
    share = c["ambiguous"] / max(c["outputs"], 1)
    everywhere = [k for k, v in c["matched"].items() if v == c["outputs"]]
    print(f"[{tag}] rows {x.shape[0]} (no segment {int(no_seg.sum())}); egrid words differing {em['words']} of "
          f"{em['checked']}; composed outside the candidate set {c['mismatch']} of {c['outputs']}; ambiguous {share:.3%}; "
          f"variants matching every output: "
          f"{everywhere if everywhere else sorted(c['matched'].items(), key=lambda kv: -kv[1])[:3]}")
    assert em["words"] == 0, (tag, em)
    assert c["mismatch"] == 0, (tag, sorted(c["mismatch_rows"])[:10])
    assert share < 0.01, (tag, share)
    assert (enc.seg >= 0).sum() > 0.3 * x.shape[0]
    return enc


# ------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("key,tables,form", [(k, t, f) for k in MODELS for t in ("pair", "wide") for f in ("query", "rays")])
def test_encode_bits(cuda, key, tables, form):
    """The training forward (per-grid features saved) on both vector layouts, and the simt debug path (mlp_impl=1),
    which saves them through its own instantiation."""
    m, fa, frames = _model(key, tables)
    nat = m.native()
    bt = _batch(fa, frames, seed=11 + len(key))
    s, x, fr = _samples(nat, bt, form, cuda)
    n = x.shape[0]
    assert n % 128 != 0
    feat, eg = _forward(nat.field, s, n, cuda)
    _check(f"{key} {tables} {form} fwd", fa, x, fr, feat, eg)
    _CACHE[("out", key, tables, form)] = (fa, x, fr, feat, eg)
    f2, keep = _no_vectors_t(nat)
    feat2, eg2 = _forward(f2, s, n, cuda)
    has = E.segment_and_time(fa, fr)[0] >= 0
    assert (feat2 == feat).all() and (eg2[:, has] == eg[:, has]).all(), "vectors_t = NULL must give the same bits"
    feat3, eg3 = _forward(nat.field, s, n, cuda, impl=1)
    _check(f"{key} {tables} {form} simt", fa, x, fr, feat3, eg3)


def test_encode_multi_tile(cuda):
    """Every forward CTA walks at least 3 tiles (3 x 5 CTAs per SM x SMs x 128 + 77 samples, the arithmetic of
    test_field_mlp_gpu._size): the persistent loop's sample index and the [64][N] stride of egrid over many tiles."""
    m, fa, frames = _model("6", "pair")
    nat = m.native()
    sms = (C.c_int * 3)()
    L.check(L.lib().hrf_device_info(sms))
    n = 3 * 5 * int(sms[0]) * 128 + 77
    tiles = (n + 127) // 128
    assert tiles // min(tiles, 5 * int(sms[0])) >= 3
    rng = np.random.default_rng(23)
    p = E.edge_positions(fa.levels, n, rng, outside=0.05)
    fr = np.array(list(frames) + _other_frames(frames), np.int32)[rng.integers(0, len(frames) + 6, n)]
    s = nat.samples_query(torch.from_numpy(p).cuda(), None, torch.from_numpy(fr).cuda())
    x, fr64 = E.load_query(p, fr)
    feat, eg = _forward(nat.field, s, n, cuda)
    _check("6 pair multi-tile", fa, x, fr64, feat, eg)


_KNOB_CASES = (("6-12", "pair", "query"), ("6-12", "wide", "rays"), ("50", "wide", "query"), ("100-100-50", "pair", "rays"))
_KNOB_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[2] + "/tests")
import test_encode_gpu as T
out = {}
for i, (key, tables, form) in enumerate(T._KNOB_CASES):
    m, fa, frames = T._model(key, tables)
    nat = m.native()
    s, x, fr = T._samples(nat, T._batch(fa, frames, seed=11 + len(key)), form, torch.device("cuda"))
    out[f"feat{i}"], out[f"egrid{i}"] = T._forward(nat.field, s, x.shape[0], torch.device("cuda"))
np.savez(sys.argv[1], **out)
"""


def test_level_unroll_instantiations(cuda, tmp_path):
    """HRF_FWD_UNROLL = 1 | 2 | 4 select the three training-forward instantiations (read once per process: one
    subprocess each).  Each must match the reference and each other bit for bit."""
    script = tmp_path / "knob.py"
    script.write_text(_KNOB_SCRIPT)
    res = {}
    for u in ("1", "2", "4"):
        env = {k: v for k, v in os.environ.items() if not k.startswith("HRF_")}
        env["HRF_FWD_UNROLL"] = u
        out = tmp_path / f"u{u}.npz"
        r = subprocess.run([sys.executable, str(script), str(out), str(ROOT)], env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, (u, r.stdout[-2000:], r.stderr[-2000:])
        res[u] = dict(np.load(out))
    for i, (key, tables, form) in enumerate(_KNOB_CASES):
        m, fa, frames = _model(key, tables)
        s, x, fr = _samples(m.native(), _batch(fa, frames, seed=11 + len(key)), form, cuda)
        for u in ("1", "2", "4"):
            _check(f"{key} {tables} {form} HRF_FWD_UNROLL={u}", fa, x, fr, res[u][f"feat{i}"], res[u][f"egrid{i}"])
            has = E.segment_and_time(fa, fr)[0] >= 0
            assert (res[u][f"feat{i}"] == res["1"][f"feat{i}"]).all()
            assert (res[u][f"egrid{i}"][:, has] == res["1"][f"egrid{i}"][:, has]).all()


@pytest.mark.parametrize("key,tables", [("6-12", "pair"), ("100-100-50", "wide")])
def test_early_stop_encode(cuda, key, tables):
    """hrf_field_density_early_stop with save="feat+grid": every sample it evaluates, bit for bit.  A chunk it skips (its
    ray already opaque) keeps the sentinel in every word; the rest are checked."""
    from humanrf_b200.volume_rendering import ray_offsets

    m, fa, frames = _model(key, tables)
    nat = m.native()
    bt = _batch(fa, frames, seed=5)
    s, x, fr = _samples(nat, bt, "rays", cuda)
    n = x.shape[0]
    ri = torch.from_numpy(bt["ri"]).to(cuda)
    off = ray_offsets(ri, bt["num_rays"])
    saved = torch.full((n * 160,), -1, dtype=torch.int16, device=cuda)
    nat.density_early_stop(s, off, bt["num_rays"], 4e-4, save="feat+grid", saved=saved)
    torch.cuda.synchronize()
    raw = saved.cpu().numpy().view(np.uint16)
    feat = raw[: 32 * n].reshape(n, 32)
    eg = raw[32 * n:].view(np.uint32).reshape(64, n)
    sentinel = (feat == 0xFFFF).all(axis=1)
    evaluated = ~sentinel
    assert ((feat == 0xFFFF).any(axis=1) == sentinel).all(), "a row is either written whole or skipped whole"
    print(f"[{key} {tables} early stop] evaluated {int(evaluated.sum())} of {n}")
    assert evaluated.sum() > 0.3 * n
    _check(f"{key} {tables} early stop", fa, x, fr, feat, eg, rows=np.nonzero(evaluated)[0])


def test_training_state_matches_masters(cuda):
    """After FusedTrainer steps (2 segments, pruning with reuse="feat+grid", segment 1 untouched in the second step) and
    without native() / refresh(): the bf16 shadows equal bf16(fp32 masters), the transposed vectors equal transpose(
    vectors) (adam_multi_kernel's vectorised vectors_t stores), the MLP blob equals its permuted bf16 copy; and an encode
    of that state matches the reference computed from the fp32 masters."""
    from humanrf_b200.scene_representation.grid_layout import MLP_BLOB_ELEMS, mlp_blob_permutation
    from humanrf_b200.training import FusedTrainer

    segs = (6, 12)
    _, m, frames = make_pair(segs, table_std=0.5)
    tr = FusedTrainer(m, prune=True, reuse="feat+grid", seed=3)
    for step, fr_pool in enumerate((frames, frames[:6], frames)):
        b = synthetic_rays(256, 64, fr_pool, seed=40 + step, ragged=True, n_distinct_frames=len(fr_pool))
        g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba")}
        before = [p.detach().clone() for p in m.hot_parameters()]
        tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], 256)
        torch.cuda.synchronize()
        if step == 1:
            moved = [not torch.equal(p, q) for p, q in zip(m.hot_parameters(), before)]
            assert not any(moved[5:10]) and all(moved[:5]), moved        # segment 1 untouched, segment 0 trained
    torch.cuda.synchronize()
    nat = tr.nat
    for s, fg in enumerate(m.feature_grids):
        for k, g in enumerate(fg.grids()):
            assert torch.equal(nat.shadows[s][k].view(torch.int16), g.detach().to(torch.bfloat16).view(torch.int16)), (s, k)
        vr = fg.vectors.shape[1]
        assert torch.equal(nat.vec_t[s].view(4, 16, vr, 2), fg.vectors.detach().view(4, vr, 16, 2).permute(0, 2, 1, 3)), s
    dst, src = mlp_blob_permutation(m.camera_embedding_dim)
    flat = torch.cat((m.sigma_net.params.detach(), m.color_net.params.detach()))
    want = torch.zeros(MLP_BLOB_ELEMS, dtype=torch.bfloat16, device=cuda)
    want[torch.from_numpy(dst).to(cuda)] = flat[torch.from_numpy(src).to(cuda)].to(torch.bfloat16)
    assert torch.equal(nat.blob.view(torch.int16), want.view(torch.int16))
    fa = _field_arrays(m, frames, segs)
    bt = _batch(fa, frames, seed=8)
    s, x, fr = _samples(nat, bt, "rays", cuda)
    feat, eg = _forward(nat.field, s, x.shape[0], cuda)
    _check("6-12 after training steps", fa, x, fr, feat, eg)


def test_bars_see_bugs(cuda):
    """Each deliberately wrong reference (encode_oracle.MUTANTS: to_cell unfused, corners accumulated in reverse, one
    level's scale one ulp up, t = (local + 0.5) / n, the lerp as (1 - f) v0 + f v1, bf16 truncation) run against the
    kernel's outputs reports at least one mismatch: the inputs reach the boundary each one moves."""
    cases = [("50", "pair", "query"), ("50", "wide", "query"), ("6-12", "wide", "rays")]
    outs = []
    for key, tables, form in cases:
        if ("out", key, tables, form) not in _CACHE:
            m, fa, frames = _model(key, tables)
            s, x, fr = _samples(m.native(), _batch(fa, frames, seed=11 + len(key)), form, cuda)
            _CACHE[("out", key, tables, form)] = (fa, x, fr) + _forward(m.native().field, s, x.shape[0], cuda)
        outs.append(_CACHE[("out", key, tables, form)])
    for mutant in E.MUTANTS:
        words = comp = 0
        for fa, x, fr, feat, eg in outs:
            enc = E.encode(fa, x, fr, feat_gpu=feat, mutant=mutant)
            words += E.egrid_mismatch(enc, eg)["words"]
            comp += enc.check["mismatch"]
        print(f"wrong reference '{mutant}': egrid words differing {words}, composed outputs outside the candidate set {comp}")
        assert words + comp > 0, mutant
