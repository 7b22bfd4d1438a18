"""The field kernels' MLPs, forward (field_fwd.cu, field_mlp.cuh) and backward (field_backward_kernel), against the
rounding-faithful float64 reference tests/mlp_oracle.py, through the C ABI.

Bars (derivations in tests/mlp_oracle.py):
* exact-class samples (every fp32 sum on the path provably exact, no ambiguous rounding): bf16 geometry features and
  d(features) bit-identical, on the wgmma path and on the fp32-FMA simt path alike.
* tight samples (no ambiguous rounding or relu mask): identical bf16 geometry features (their rounding is determined);
  d(features) within acc_delta(64) * sum|terms|; sigma within sigma * (exp_eps + bound of h0); rgb within
  r (1 - r) (exp_eps + bound of the pre-activation) + 2 fp32 ulps.
* ambiguous samples: entrywise within their propagated deviation bound (mlp_oracle.py, dev_relu_round and the
  D_* / *_dev arrays): how far a flipped rounding or relu mask can move each tile and output.  Their share is printed
  per case.  Under the worst-case accumulation bound nearly every realistic-input sample has an ambiguous decision
  somewhere on its ~400-decision path, so the realistic cases are checked almost entirely by deviation bounds; the exact
  and tight claims are carried by the dyadic cases.
* d_mlp: bit-identical on entries whose whole-batch sum is provably exact and untouched by ambiguous samples,
  acc_delta(chain) * S + 2 A elsewhere, with chain = 128 x (tiles per CTA) + CTAs (one register chain per CTA plus one
  atomic per CTA), where A bounds the ambiguous samples' deviation.  Colour W3 rows 3..15 (padded outputs) exactly 0.
* d_emb: rows no sample uses exactly 0; used rows within the sum of their samples' d(colour input) bounds, the atomic
  chain.
Sample counts derive from the SM count: every backward CTA owns >= 3 tiles at 3 * 2 * SMs * 128 + 77 samples, every
forward CTA >= 3 at 3 * 5 * SMs * 128 + 77 (3 * 4 * SMs * 128 + 77 with camera embeddings, which run 4 CTAs per SM); the
tests assert this from the launch arithmetic.
"""
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import mlp_oracle as M
from helpers import make_pair
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
_CACHE = {}


def _sms():
    out = (C.c_int * 3)()
    L.check(L.lib().hrf_device_info(out))
    return int(out[0])


def _size(tag, K=32, fwd=False):
    sms = _sms()
    if tag != "multi":
        return int(tag)
    if fwd:
        return 3 * _fwd_ctas_per_sm(K) * sms * 128 + 77
    return 3 * 2 * sms * 128 + 77


def _fwd_ctas_per_sm(K):
    return 4 if K == 48 else 5      # launch_field_forward: 5 CTAs per SM, 4 with the larger camera-embedding blob


def _launch(n, per_sm):
    tiles = (n + 127) // 128
    ctas = min(tiles, per_sm * _sms())
    return tiles, ctas, tiles // ctas, -(-tiles // ctas)


def _model(K):
    key = ("model", K)
    if key not in _CACHE:
        _CACHE[key] = make_pair((6,), seed=123, table_std=6.0, cam_emb=(2 if K == 48 else 0))
    return _CACHE[key]


def _set_weights(m, sp, cp):
    with torch.no_grad():
        m.sigma_net.params.copy_(torch.from_numpy(np.asarray(sp, np.float32)))
        m.color_net.params.copy_(torch.from_numpy(np.asarray(cp, np.float32)))
    nat = m.native()
    nat.refresh()
    return nat


def _ncam(m):
    """Rows of the embedding table: what the native field passes as num_cameras (0 without embeddings)."""
    return m.camera_embeddings.weight.shape[0] if m.camera_embedding_dim else 0


def _emb(m):
    return m.camera_embeddings.weight.detach().cpu().numpy() if m.camera_embedding_dim else None


class Batch:
    """One sample per ray (t = 0, origin = position): the ray-batch form every entry point accepts."""

    def __init__(self, rng, n, frames, K, ncam=0, cam_mix=True, no_seg=True, axis_dirs=True):
        self.n, self.ncam = n, ncam
        self.pos = rng.uniform(-0.45, 0.45, (n, 3)).astype(np.float32)
        self.dirs = M.axis_directions(rng, n) if axis_dirs else None
        if self.dirs is None:
            d = rng.standard_normal((n, 3))
            self.dirs = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
        fr = rng.choice(np.asarray(frames), n).astype(np.int32)
        if no_seg and n > 3:
            # frames outside the LUT and frames the LUT maps to no segment: both encode to a zero feature row
            k = rng.choice(n, max(1, n // 50), replace=False)
            fr[k] = rng.choice(np.array([-3, 5000, 0, 7, frames[0] - 1], np.int32), len(k))
        self.frames = fr
        self.cams = None
        if K == 48:
            c = rng.integers(0, 12, n).astype(np.int32)
            if cam_mix and n > 3:
                k = rng.choice(n, max(1, n // 20), replace=False)
                c[k] = rng.choice(np.array([-1, -7, ncam, ncam + 40], np.int32), len(k))
            self.cams = c
        self.seg_ok = (fr >= frames[0]) & (fr <= frames[-1])

    def ref_cams(self, use_cam=True):
        if self.cams is None or not use_cam:
            return np.full(self.n, -1, np.int64)
        c = self.cams.astype(np.int64)
        return np.where((c >= 0) & (c < self.ncam), c, -1)

    def samples(self, nat, cuda, use_cam=True, capacity=None, count_dev=None):
        cap = capacity or self.n
        pad = cap - self.n

        def dev(a, dtype):
            t = torch.from_numpy(np.concatenate([a, np.zeros((pad,) + a.shape[1:], a.dtype)]) if pad else a)
            return t.to(cuda, dtype).contiguous()

        o, d, fr = dev(self.pos, torch.float32), dev(self.dirs, torch.float32), dev(self.frames, torch.int32)
        t = torch.zeros(cap, device=cuda)
        ri = torch.arange(cap, device=cuda, dtype=torch.int64)
        cams = dev(self.cams, torch.int32) if (self.cams is not None and use_cam) else None
        return nat.samples_rays(o, d, fr, t, ri, ray_cameras=cams, count_dev=count_dev)


def _bf16_dev(a, cuda):
    return torch.from_numpy(np.asarray(a, np.float32)).to(cuda).to(torch.bfloat16).contiguous()


def _backward(nat, m, s, n, d_sigma, d_rgb, d_geo, feat, feat_index, cuda, cap=None, fill=0.0):
    cap = cap or n
    dev = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.float32)).to(cuda).contiguous()  # noqa: E731
    ups = [dev(d_sigma), dev(d_rgb), dev(d_geo)]
    if cap > n:
        ups = [None if u is None else torch.cat([u, torch.full((cap - n,) + tuple(u.shape[1:]), fill, device=cuda)]) for u in ups]
    d_mlp = torch.zeros(m.mlp_grad_elems, device=cuda)
    d_emb = torch.zeros((_ncam(m), m.camera_embedding_dim), device=cuda) if m.camera_embedding_dim else None
    ws = torch.full((cap * 40,), fill, device=cuda)
    L.check(L.lib().hrf_field_backward_mlp(C.byref(nat.field), C.byref(s), L.ptr(ups[0]), L.ptr(ups[1]), L.ptr(ups[2]),
                                           L.ptr(feat), L.ptr(feat_index), d_mlp.data_ptr(), L.ptr(d_emb), ws.data_ptr(),
                                           L.stream()))
    torch.cuda.synchronize()
    dfeat = ws[: 32 * cap].view(16, cap, 2).permute(1, 0, 2).reshape(cap, 32)[:n].double().cpu().numpy()
    return d_mlp.double().cpu().numpy(), dfeat, None if d_emb is None else d_emb.double().cpu().numpy(), ws


def _upstream(rng, n, which, dyadic):
    if dyadic:
        ds, dr, dg = M.dyadic_upstream(rng, n)
    else:
        ds = (rng.standard_normal(n) * 1e-2).astype(np.float32)
        dr = rng.standard_normal((n, 3)).astype(np.float32)
        dg = (rng.standard_normal((n, 15)) * 0.1).astype(np.float32)
    return (ds if which in ("sigma", "all") else None, dr if which in ("rgb", "all") else None,
            dg if which in ("geo", "all") else None)


def _demb_check(got, B, F, ncam):
    if got is None:
        return True, {}
    used = np.zeros(ncam, bool)
    ok_c = F.cams >= 0
    used[F.cams[ok_c]] = True
    E = F.E
    tol = np.zeros((ncam, E))
    cnt = np.zeros(ncam)
    np.add.at(cnt, F.cams[ok_c], 1)
    absd = np.abs(B.dcin[:, 31:31 + E])
    per = B.dcin_dev[:, 31:31 + E]     # accumulation bound, plus the deviation bound on ambiguous samples
    np.add.at(tol, F.cams[ok_c], per[ok_c])
    sabs = np.zeros((ncam, E))
    np.add.at(sabs, F.cams[ok_c], absd[ok_c])
    tol += cnt[:, None] * M.U23 * sabs
    d = np.abs(got - B.d_emb)
    ok = bool((got[~used] == 0).all() and (d <= tol).all())
    return ok, dict(used_rows=int(used.sum()), unused_nonzero=int((got[~used] != 0).sum()), bad=int((d > tol).sum()))


def _report(case, n, per_sm, parts):
    tiles, ctas, lo, hi = _launch(n, per_sm)
    print(f"[{case}] n={n} tiles={tiles} ctas={ctas} tiles/cta={lo}..{hi}")
    for name, rep in parts:
        print(f"    {name}: {json.dumps(rep)}")


def _check_backward(case, m, B, F, n, d_mlp, dfeat, d_emb):
    okf, rf = M.compare_rows(dfeat, B.dfeat, B.dfeat_e, B.exact_dfeat, B.amb, B.dfeat_dev)
    okm, rm = M.compare_dmlp(d_mlp, B)
    oke, re_ = _demb_check(d_emb, B, F, _ncam(m))
    K = F.K
    gcol3 = 3072 + 64 * K + 4096
    zeros = bool((d_mlp[gcol3 + 3 * 64: gcol3 + 16 * 64] == 0).all())
    _report(case, n, 2, [("dfeat", rf), ("d_mlp", rm), ("d_emb", re_)])
    assert zeros, "colour W3 rows 3..15 (padded outputs) must have zero gradient"
    assert okf and okm and oke, (rf, rm, re_)


def _dyadic_setup(K, seed):
    rng = np.random.default_rng(seed)
    om, m, frames = _model(K)
    sp, cp = M.dyadic_params(rng, K)
    return rng, m, frames, sp, cp


def _ref(key, build):
    if key not in _CACHE:
        _CACHE[key] = build()
    return _CACHE[key]


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", ["1", "127", "128", "129", "multi"])
@pytest.mark.parametrize("upstream", ["sigma", "rgb", "geo", "all"])
@pytest.mark.parametrize("K", [32, 48])
def test_backward_dyadic(cuda, K, upstream, size):
    """Identity feat_in with dyadic features and weights; frames in no segment; for K = 48 camera rows that are valid,
    at or above num_cameras and negative."""
    rng, m, frames, sp, cp = _dyadic_setup(K, 100 + K)
    nat = _set_weights(m, sp, cp)
    n = _size(size, K)
    b = Batch(rng, n, frames, K, _ncam(m))
    feat = M.dyadic_features(rng, n)
    ups = _upstream(rng, n, upstream, True)
    s = b.samples(nat, cuda)
    d_mlp, dfeat, d_emb, _ = _backward(nat, m, s, n, *ups, _bf16_dev(feat, cuda), None, cuda)

    def build():
        fref = np.where(b.seg_ok[:, None], feat, 0.0)        # field_bwd.cu:524: no segment -> zero feature row
        F = M.Forward(fref, b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K), m.density_scale, K)
        return F, M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=M.wgrad_chain(n, min((n + 127) // 128, 2 * _sms())))
    F, B = _ref(("bwd-dyadic", K, upstream, size), build)
    print("classes (exact, tight, ambiguous):", B.classes())
    _check_backward(f"bwd dyadic K={K} {upstream} {size}", m, B, F, n, d_mlp, dfeat, d_emb)
    if upstream == "geo":
        assert B.exact.all()      # the dyadic d_geo path is exact end to end: every sample was compared bit for bit


@pytest.mark.parametrize("source", ["identity", "permuted", "reencode"])
def test_backward_feature_sources(cuda, source):
    """Where d(features) come from: saved rows, rows picked through feat_index from a wider buffer (the survivor path),
    or the backward's own re-encode, checked against the forward's saved features."""
    K = 32
    rng, m, frames, sp, cp = _dyadic_setup(K, 7)
    nat = _set_weights(m, sp, cp)
    n = _size("multi", K)
    b = Batch(rng, n, frames, K, _ncam(m))
    s = b.samples(nat, cuda)
    ups = _upstream(rng, n, "all", True)
    _, _, _, saved = nat.forward(s, 1, want_geo=False, want_feat=True)
    torch.cuda.synchronize()
    enc = nat.saved_features(saved, n).float().cpu().numpy().astype(np.float64)
    if source == "identity":
        feat_ref, feat_dev, idx = enc, nat.saved_features(saved, n).contiguous(), None
    elif source == "permuted":
        wide = M.dyadic_features(rng, 2 * n)
        perm = rng.permutation(2 * n)[:n].astype(np.int32)
        wide[perm] = enc
        feat_ref, feat_dev, idx = enc, _bf16_dev(wide, cuda), torch.from_numpy(perm).to(cuda)
    else:
        feat_ref, feat_dev, idx = enc, None, None
    assert (enc[~b.seg_ok] == 0).all()        # the encode writes a zero row for frames in no segment
    d_mlp, dfeat, d_emb, _ = _backward(nat, m, s, n, *ups, feat_dev, idx, cuda)

    def build():   # the same seeded batch and saved features for every source: one reference
        F = M.Forward(feat_ref, b.dirs, b.ref_cams(), None, M.split_params(sp, cp, K), m.density_scale, K)
        return F, M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=M.wgrad_chain(n, 2 * _sms()))
    F, B = _ref(("bwd-sources",), build)
    assert (F.feat == feat_ref).all()
    print("classes (exact, tight, ambiguous):", B.classes())
    _check_backward(f"bwd source={source}", m, B, F, n, d_mlp, dfeat, d_emb)


@pytest.mark.parametrize("size", ["129", "multi"])
@pytest.mark.parametrize("K", [32, 48])
def test_backward_realistic(cuda, K, size):
    """Features a real encode writes, Xavier weights, random upstream gradients, random view directions."""
    om, m, frames = _model(K)
    rng = np.random.default_rng(31 + K)
    sp = torch.cat([w.reshape(-1) for w in om.w_sigma]).numpy()
    cp = torch.cat([w.reshape(-1) for w in om.w_color]).numpy()
    nat = _set_weights(m, sp, cp)
    n = _size(size, K)
    b = Batch(rng, n, frames, K, _ncam(m), axis_dirs=False)
    s = b.samples(nat, cuda)
    _, _, _, saved = nat.forward(s, 1, want_geo=False, want_feat=True)
    torch.cuda.synchronize()
    enc = nat.saved_features(saved, n).float().cpu().numpy().astype(np.float64)
    ups = _upstream(rng, n, "all", False)
    d_mlp, dfeat, d_emb, _ = _backward(nat, m, s, n, *ups, nat.saved_features(saved, n).contiguous(), None, cuda)
    F = M.Forward(enc, b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K), m.density_scale, K)
    B = M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=M.wgrad_chain(n, min((n + 127) // 128, 2 * _sms())))
    print("classes (exact, tight, ambiguous):", B.classes())
    # Under the worst-case accumulation bound nearly every realistic sample has some ambiguous decision among the ~400
    # roundings and masks of its backward path (the share is printed): these cases rest on the norm-wise bars, d_mlp's
    # included, and the few tight samples; the exact and tight claims are carried by the dyadic cases.
    _check_backward(f"bwd realistic K={K} {size}", m, B, F, n, d_mlp, dfeat, d_emb)


@pytest.mark.parametrize("size", ["1", "127", "128", "129", "multi"])
@pytest.mark.parametrize("impl", ["wgmma", "simt"])
@pytest.mark.parametrize("K", [32, 48])
def test_forward_encode(cuda, K, impl, size):
    """hrf_field_forward (mlp_impl 0 = wgmma, 1 = the fp32-FMA simt debug path): the reference is fed the features the
    kernel saved.  Dyadic weights and axis-aligned directions keep most sums exact, so geometry bits are compared bit for
    bit on exact samples on both paths."""
    rng, m, frames, sp, cp = _dyadic_setup(K, 300 + K)
    nat = _set_weights(m, sp, cp)
    n = _size(size, K, fwd=True)
    b = Batch(rng, n, frames, K, _ncam(m))
    s = b.samples(nat, cuda)
    sig, geo, rgb, saved = nat.forward(s, 1, want_geo=True, want_feat=True, mlp_impl=(1 if impl == "simt" else 0))
    torch.cuda.synchronize()
    enc = nat.saved_features(saved, n).float().cpu().numpy().astype(np.float64)
    F = M.Forward(enc, b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K), m.density_scale, K)
    none = np.zeros(n, bool)
    okg, rg = M.compare_rows(geo.double().cpu().numpy(), F.geo, 0.0, F.exact_geo, F.amb_geo, F.D_geo)
    oks, rs = M.compare_rows(sig.double().cpu().numpy(), F.sigma, F.sigma_tol, none, F.amb_geo, F.sigma_dev)
    okr, rr = M.compare_rows(rgb.double().cpu().numpy(), F.rgb, F.rgb_tol, none, F.amb, F.rgb_dev)
    _report(f"fwd {impl} K={K} {size}", n, 4 if K == 48 else 5, [("geo", rg), ("sigma", rs), ("rgb", rr)])
    assert okg and oks and okr
    if size == "multi":
        assert _launch(n, _fwd_ctas_per_sm(K))[2] >= 3      # every forward CTA owns at least 3 tiles
    if n >= 128:
        assert rg["exact"] > 0.5 * n       # the bit-exact claim covers most of the batch


@pytest.mark.parametrize("size", ["1", "129", "multi"])
@pytest.mark.parametrize("K", [32, 48])
def test_forward_from_features(cuda, K, size):
    """hrf_field_forward_from_features with dyadic features, identity and through feat_index.  Frames in no segment: this
    kernel takes the feature row as given (field_fwd.cu:108), while the backward zeroes it (field_bwd.cu:524) -- both
    encodes write a zero row there, so the two agree whenever feat_in comes from an encode.  Pinned here."""
    rng, m, frames, sp, cp = _dyadic_setup(K, 500 + K)
    nat = _set_weights(m, sp, cp)
    n = _size(size, K, fwd=True)
    b = Batch(rng, n, frames, K, _ncam(m))
    s = b.samples(nat, cuda)
    feat = M.dyadic_features(rng, n)
    F = M.Forward(feat, b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K), m.density_scale, K)
    none = np.zeros(n, bool)
    perm = rng.permutation(3 * n)[:n].astype(np.int32)
    wide = M.dyadic_features(rng, 3 * n)
    wide[perm] = feat
    for name, fd, idx in (("identity", _bf16_dev(feat, cuda), None),
                          ("feat_index", _bf16_dev(wide, cuda), torch.from_numpy(perm).to(cuda))):
        sig, rgb = nat.forward_from_features(s, fd, idx)
        torch.cuda.synchronize()
        oks, rs = M.compare_rows(sig.double().cpu().numpy(), F.sigma, F.sigma_tol, none, F.amb_geo, F.sigma_dev)
        okr, rr = M.compare_rows(rgb.double().cpu().numpy(), F.rgb, F.rgb_tol, none, F.amb, F.rgb_dev)
        _report(f"fwd-from-features {name} K={K} {size}", n, 4 if K == 48 else 5, [("sigma", rs), ("rgb", rr)])
        assert oks and okr
    if size == "multi":
        assert _launch(n, _fwd_ctas_per_sm(K))[2] >= 3
    if (~b.seg_ok).any():
        assert np.abs(feat[~b.seg_ok]).sum() > 0          # the rows really were non-zero and were used as given


def test_live_count_below_capacity(cuda):
    """num_samples_dev below the capacity: outputs and workspace past the live count keep their sentinel."""
    K = 48
    rng, m, frames, sp, cp = _dyadic_setup(K, 9)
    nat = _set_weights(m, sp, cp)
    cap = _size("multi", K)
    n = cap - 3 * 128 - 50
    b = Batch(rng, n, frames, K, _ncam(m))
    count = torch.tensor([n], dtype=torch.int64, device=cuda)
    s = b.samples(nat, cuda, capacity=cap, count_dev=count)
    feat = M.dyadic_features(rng, n)
    fd = _bf16_dev(np.concatenate([feat, M.dyadic_features(rng, cap - n)]), cuda)
    sent = float("nan")
    sig = torch.full((cap,), sent, device=cuda)
    rgb = torch.full((cap, 3), sent, device=cuda)
    nat.forward_from_features(s, fd, None, sigma=sig, rgb=rgb)
    ups = _upstream(rng, n, "all", True)
    d_mlp, dfeat, d_emb, ws = _backward(nat, m, s, n, *ups, fd, None, cuda, cap=cap, fill=sent)
    torch.cuda.synchronize()
    assert torch.isnan(sig[n:]).all() and torch.isnan(rgb[n:]).all()
    wsv = ws.view(torch.int32).cpu().numpy()
    nan_bits = np.float32(np.nan).view(np.int32)
    dfr = wsv[: 32 * cap].reshape(16, cap, 2)
    assert (dfr[:, n:] == nan_bits).all(), "d(features) written past the live count"
    assert (wsv[32 * cap: 36 * cap].reshape(cap, 4)[n:] == nan_bits).all(), "positions written past the live count"
    seg8 = ws.view(torch.uint8)[144 * cap: 145 * cap].cpu().numpy()
    assert (seg8[n:] == np.frombuffer(np.float32(np.nan).tobytes(), np.uint8)[np.arange(n, cap) % 4]).all()
    F = M.Forward(np.where(b.seg_ok[:, None], feat, 0.0), b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K),
                  m.density_scale, K)
    B = M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=M.wgrad_chain(cap, 2 * _sms()))
    _check_backward("live count below capacity", m, B, F, n, d_mlp, dfeat, d_emb)
    Ff = M.Forward(feat, b.dirs, b.ref_cams(), _emb(m), M.split_params(sp, cp, K), m.density_scale, K)
    okr, rr = M.compare_rows(rgb[:n].double().cpu().numpy(), Ff.rgb, Ff.rgb_tol, np.zeros(n, bool), Ff.amb, Ff.rgb_dev)
    assert okr, rr


def test_camera_embeddings_off(cuda):
    """K = 48 with use_camera_embeddings off: the embedding columns are 0 and the embedding gradient stays 0."""
    K = 48
    rng, m, frames, sp, cp = _dyadic_setup(K, 13)
    nat = _set_weights(m, sp, cp)
    n = 129 * 7
    b = Batch(rng, n, frames, K, _ncam(m))
    s = b.samples(nat, cuda, use_cam=False)
    feat = M.dyadic_features(rng, n)
    ups = _upstream(rng, n, "all", True)
    d_mlp, dfeat, d_emb, _ = _backward(nat, m, s, n, *ups, _bf16_dev(feat, cuda), None, cuda)
    assert (d_emb == 0).all()
    F = M.Forward(np.where(b.seg_ok[:, None], feat, 0.0), b.dirs, b.ref_cams(use_cam=False), _emb(m),
                  M.split_params(sp, cp, K), m.density_scale, K)
    B = M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=M.wgrad_chain(n, 2 * _sms()))
    _check_backward("camera embeddings off", m, B, F, n, d_mlp, dfeat, d_emb)


def test_bars_see_bugs(cuda):
    """The comparators reject deliberately wrong references: a dropped tile that some CTA owns as its second or later
    tile, row 127 of every tile dropped, one hidden unit's relu mask inverted, d_emb shifted by one camera row."""
    K = 48
    rng, m, frames, sp, cp = _dyadic_setup(K, 17)
    nat = _set_weights(m, sp, cp)
    n = _size("multi", K)
    b = Batch(rng, n, frames, K, _ncam(m), cam_mix=False)
    feat = M.dyadic_features(rng, n)
    ups = _upstream(rng, n, "all", True)
    s = b.samples(nat, cuda)
    d_mlp, dfeat, d_emb, _ = _backward(nat, m, s, n, *ups, _bf16_dev(feat, cuda), None, cuda)
    fref = np.where(b.seg_ok[:, None], feat, 0.0)
    P = M.split_params(sp, cp, K)
    F = M.Forward(fref, b.dirs, b.ref_cams(), _emb(m), P, m.density_scale, K)
    tiles, ctas, _, _ = _launch(n, 2)
    chain = M.wgrad_chain(n, ctas)
    B = M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=chain)

    def verdict(Bx, demb=None):
        okf, rf = M.compare_rows(dfeat, Bx.dfeat, Bx.dfeat_e, Bx.exact_dfeat, Bx.amb, Bx.dfeat_dev)
        okm, rm = M.compare_dmlp(d_mlp, Bx)
        if demb is not None:
            Bx.d_emb = demb
        oke, re_ = _demb_check(d_emb, Bx, F, _ncam(m))
        return okf, okm, oke, (rf, rm, re_)

    assert all(verdict(B)[:3])

    def dropped(mask):
        z = [None if u is None else np.where(mask.reshape((-1,) + (1,) * (u.ndim - 1)), 0, u) for u in ups]
        return M.Backward(F, *z, m.density_scale, _ncam(m), wgrad_chain=chain)

    tile = ctas + 5                 # CTA 5's second tile
    assert tile < tiles
    drop = np.zeros(n, bool)
    drop[tile * 128:(tile + 1) * 128] = True
    row127 = (np.arange(n) % 128) == 127
    variants = {"dropped tile": dropped(drop), "row 127 of every tile": dropped(row127),
                "inverted relu mask (colour hidden 1, unit 5)": M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=chain,
                                                                           invert_mask=("h1", 5))}
    for name, Bx in variants.items():
        okf, okm, oke, reps = verdict(Bx)
        print(f"wrong reference '{name}': dfeat ok={okf} d_mlp ok={okm} d_emb ok={oke}; d_mlp {json.dumps(reps[1])}")
        assert not (okf and okm and oke), name
        assert not okm, f"the d_mlp bar alone must see '{name}'"
    shifted = np.roll(B.d_emb, 1, axis=0)
    okf, okm, oke, reps = verdict(M.Backward(F, *ups, m.density_scale, _ncam(m), wgrad_chain=chain), demb=shifted)
    print(f"wrong reference 'd_emb shifted by one row': d_emb ok={oke} {json.dumps(reps[2])}")
    assert not oke


_KNOB_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[2] + "/tests")
from helpers import make_pair
om, m, frames = make_pair((6,), seed=123, table_std=6.0)
rng = np.random.default_rng(1)
sms = int(sys.argv[3])
n = 3 * 2 * sms * 128 + 77
with torch.no_grad():
    m.sigma_net.params.copy_(torch.cat([w.reshape(-1) for w in om.w_sigma]).cuda())
    m.color_net.params.copy_(torch.cat([w.reshape(-1) for w in om.w_color]).cuda())
nat = m.native(); nat.refresh()
pos = torch.from_numpy(rng.uniform(-0.45, 0.45, (n, 3)).astype(np.float32)).cuda()
d = rng.standard_normal((n, 3)); d = torch.from_numpy((d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)).cuda()
fr = torch.from_numpy(rng.choice(np.asarray(frames), n).astype(np.int32)).cuda()
s = nat.samples_rays(pos, d, fr, torch.zeros(n, device="cuda"), torch.arange(n, device="cuda"))
sig, geo, rgb, saved = nat.forward(s, 1, want_geo=True, want_feat=True)
sig2, geo2, rgb2, _ = nat.forward(s, 1, want_geo=True, want_feat=False)
ds = torch.from_numpy((rng.standard_normal(n) * 1e-2).astype(np.float32)).cuda()
dr = torch.from_numpy(rng.standard_normal((n, 3)).astype(np.float32)).cuda()
from humanrf_b200 import _lib as L
import ctypes as C
out = {}
for name, feat in (("saved", nat.saved_features(saved, n).contiguous()), ("reencode", None)):
    d_mlp = torch.zeros(m.mlp_grad_elems, device="cuda"); ws = torch.zeros(n * 40, device="cuda")
    L.check(L.lib().hrf_field_backward_mlp(C.byref(nat.field), C.byref(s), ds.data_ptr(), dr.data_ptr(), None, L.ptr(feat), None,
                                           d_mlp.data_ptr(), None, ws.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    out["d_mlp_" + name] = d_mlp.cpu().numpy(); out["dfeat_" + name] = ws[:32 * n].cpu().numpy()
out.update(sigma=sig.cpu().numpy(), geo=geo.view(torch.int16).cpu().numpy(), rgb=rgb.cpu().numpy(),
           feat=saved.view(torch.int16).cpu().numpy(), sigma_nofeat=sig2.cpu().numpy(),
           geo_nofeat=geo2.view(torch.int16).cpu().numpy(), rgb_nofeat=rgb2.cpu().numpy())
np.savez(sys.argv[1], **out)
"""


def test_tuning_knob_instantiations(cuda, tmp_path):
    """HRF_FWD_UNROLL = 2 | 4, HRF_FWD_CTAS = 4 | 6 and HRF_BWD_UNROLL = 1 select kernel instantiations nothing else runs.
    They are read once per process, so each runs in its own subprocess on the same seeded multi-tile batch.  Each run
    does one forward that saves features (the training instantiations, where HRF_FWD_CTAS changes only the grid size) and
    one that does not (where HRF_FWD_CTAS selects the instantiation: 4, 6 with 1-level unroll, 6 with 4-level unroll).  The
    arithmetic per level and per layer is the same in every instantiation, so every per-sample output is expected to be
    bit-identical to the default's; d_mlp differs only by the order of its fp32 atomic adds across CTAs, so it gets the
    atomic-order bound instead (relative norm 1e-6: 264 CTA partials, 2^-23 each)."""
    script = tmp_path / "knob.py"
    script.write_text(_KNOB_SCRIPT)
    sms = _sms()
    res = {}
    for tag, env in (("default", {}), ("fwd_unroll2", {"HRF_FWD_UNROLL": "2"}), ("fwd_unroll4", {"HRF_FWD_UNROLL": "4"}),
                     ("fwd_ctas4", {"HRF_FWD_CTAS": "4"}), ("fwd_ctas6", {"HRF_FWD_CTAS": "6"}),
                     ("fwd_ctas6_unroll4", {"HRF_FWD_CTAS": "6", "HRF_FWD_UNROLL": "4"}), ("bwd_unroll1", {"HRF_BWD_UNROLL": "1"})):
        e = {k: v for k, v in os.environ.items() if not k.startswith("HRF_")}
        e.update(env)
        out = tmp_path / f"{tag}.npz"
        r = subprocess.run([sys.executable, str(script), str(out), str(ROOT), str(sms)], env=e, capture_output=True, text=True,
                           timeout=300)
        assert r.returncode == 0, (tag, r.stdout[-2000:], r.stderr[-2000:])
        res[tag] = dict(np.load(out))
    base = res.pop("default")
    for tag, got in res.items():
        for k, v in got.items():
            if k.startswith("d_mlp"):
                rel = np.linalg.norm(v.astype(np.float64) - base[k]) / np.linalg.norm(base[k])
                print(f"{tag} {k}: relnorm vs default {rel:.2e}")
                assert rel <= 1e-6, (tag, k, rel)
            else:
                diff = int((v != base[k]).sum())
                print(f"{tag} {k}: {diff} of {v.size} differ from the default")
                assert diff == 0, (tag, k)
