"""The volume-rendering kernels on the H100 against the float64 reference of tests/composite_oracle.py, per element and
within its error bound: hrf_ray_offsets, hrf_prune, hrf_composite_forward / _backward, the compositing epilogue of the
fused render (hrf_render_fused, hrf_render_fused_depth) with its fix-up, and the exactness of the early-stop density
pass at chunk borders.  Every output buffer is filled with a sentinel first, and entries no kernel should write must
keep it.  Each test prints the largest error / bound it saw per kernel and case."""
import ctypes as C

import numpy as np
import pytest
import torch

import composite_oracle as O
from helpers import make_pair
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu

STEP = O.STEP
SENT = {torch.float32: -12345.5, torch.uint8: 0xAB, torch.int32: -77, torch.int64: -77}
PAD = 5     # sentinel entries past the end of every output


def _sent(shape, dtype, cuda):
    return torch.full(shape if isinstance(shape, tuple) else (shape,), SENT[dtype], dtype=dtype, device=cuda)


def _untouched(x, name):
    assert (x == SENT[x.dtype]).all(), f"{name}: an entry past the end was written"


def _dev(x, cuda, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(cuda)


def _check(kernel, case, got, ref, bound):
    r = O.ratio(got, ref, bound)
    print(f"{kernel} [{case}]: largest error / bound {r:.3g}")
    assert r <= 1.0, (kernel, case, r)


@pytest.fixture(scope="module")
def batch():
    return O.ray_batch()


# ---------------------------------------------------------------------------------------------------------------------
def test_ray_offsets_gaps_trailing_rays_and_empty_batch(cuda):
    rng = np.random.default_rng(1)
    cases = [("gaps + trailing empty rays", np.sort(rng.integers(0, 3000, 5000)), 3100),
             ("one ray", np.zeros(7, np.int64), 1),
             ("n = 0", np.zeros(0, np.int64), 5)]
    for name, ri, R in cases:
        assert name != "gaps + trailing empty rays" or len(np.setdiff1d(np.arange(3000), ri)) > 0
        ri_d = _dev(ri.astype(np.int64), cuda)
        off = _sent(R + 1 + PAD, torch.int32, cuda)
        L.check(L.lib().hrf_ray_offsets(ri_d.data_ptr(), ri.shape[0], R, off.data_ptr(), L.stream()))
        np.testing.assert_array_equal(off[:R + 1].cpu().numpy(), O.ray_offsets(ri, R), err_msg=name)
        _untouched(off[R + 1:], name)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["thresholds 1e-4", "thresholds hit exactly", "no source index"])
def test_prune_against_reference(cuda, batch, case):
    B = batch
    eps, thre = (1.0, 0.0) if case == "thresholds hit exactly" else (1e-4, 1e-4)
    n, R = B["t"].shape[0], B["num_rays"]
    sig, t, ri = _dev(B["sigma"], cuda), _dev(B["t"], cuda), _dev(B["ri"], cuda, torch.int64)
    off = _dev(B["off"], cuda, torch.int32)
    keep = _sent(n + PAD, torch.uint8, cuda)
    kept = _sent(R + 1 + PAD, torch.int32, cuda)
    out_t, out_ri = _sent(n + PAD, torch.float32, cuda), _sent(n + PAD, torch.int64, cuda)
    src = None if case == "no source index" else _sent(n + PAD, torch.int32, cuda)
    cnt = _sent(1, torch.int64, cuda)
    L.check(L.lib().hrf_prune(sig.data_ptr(), t.data_ptr(), ri.data_ptr(), off.data_ptr(), R, STEP, eps, thre,
                              keep.data_ptr(), kept.data_ptr(), out_t.data_ptr(), out_ri.data_ptr(), L.ptr(src),
                              cnt.data_ptr(), L.stream()))
    got = keep[:n].cpu().numpy()
    _untouched(keep[n:], "keep")
    assert set(np.unique(got)) <= {0, 1}
    got = got.astype(bool)
    ref, amb, _ = O.visibility(B["sigma"], B["off"], STEP, eps, thre)
    bad = (got != ref) & ~amb
    print(f"hrf_prune [{case}]: {int(ref.sum())} kept by the reference, {int(amb.sum())} ambiguous, "
          f"{int((got != ref).sum())} decided the other way there, {int(bad.sum())} elsewhere")
    assert bad.sum() == 0, np.nonzero(bad)[0][:10]
    # counts, the in-place scan (2600 rays: three 1024-ray blocks) and the compaction are exact given the kernel's mask
    exp_off = O.kept_offsets(got, B["off"])
    np.testing.assert_array_equal(kept[:R + 1].cpu().numpy(), exp_off)
    _untouched(kept[R + 1:], "kept_offsets")
    k = int(cnt.item())
    assert k == got.sum() == exp_off[-1]
    et, eri, esrc = O.compact(got, B["t"], B["off"])
    np.testing.assert_array_equal(out_t[:k].cpu().numpy(), et)
    np.testing.assert_array_equal(out_ri[:k].cpu().numpy(), eri)
    _untouched(out_t[k:], "out_distances"), _untouched(out_ri[k:], "out_ray_indices")
    if src is not None:
        np.testing.assert_array_equal(src[:k].cpu().numpy(), esrc)
        _untouched(src[k:], "out_source_index")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_bg,with_weights", [(False, True), (True, True), (True, False)])
def test_composite_forward_against_reference(cuda, batch, with_bg, with_weights):
    B = batch
    n, R = B["t"].shape[0], B["num_rays"]
    case = f"bg={with_bg} weights={'buffer' if with_weights else 'NULL'}"
    bg = B["bg"] if with_bg else None
    F = O.Forward(B["sigma"], B["rgb"], B["t"], B["off"], STEP, bg)
    sig, rgb, t = _dev(B["sigma"], cuda), _dev(B["rgb"], cuda), _dev(B["t"], cuda)
    off = _dev(B["off"], cuda, torch.int32)
    bg_d = _dev(bg, cuda) if with_bg else None
    color, wsum = _sent((R + PAD, 3), torch.float32, cuda), _sent(R + PAD, torch.float32, cuda)
    w = _sent(n + PAD, torch.float32, cuda) if with_weights else None
    L.check(L.lib().hrf_composite_forward(sig.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(), R, STEP,
                                          L.ptr(bg_d), color.data_ptr(), wsum.data_ptr(), L.ptr(w), L.stream()))
    _untouched(color[R:], "color"), _untouched(wsum[R:], "weights_sum")
    _check("hrf_composite_forward color", case, color[:R].cpu().numpy(), F.color, F.color_err)
    _check("hrf_composite_forward weights_sum", case, wsum[:R].cpu().numpy(), F.wsum, F.wsum_err)
    if with_weights:
        _untouched(w[n:], "weights")
        _check("hrf_composite_forward weights", case, w[:n].cpu().numpy(), F.weights, F.weights_err)


@pytest.mark.parametrize("with_bg,with_dwsum,with_drgb", [(False, True, True), (True, True, True), (True, False, True),
                                                          (True, True, False)])
def test_composite_backward_against_reference(cuda, batch, with_bg, with_dwsum, with_drgb):
    B = batch
    n, R = B["t"].shape[0], B["num_rays"]
    case = f"bg={with_bg} d_weights_sum={'buffer' if with_dwsum else 'NULL'} d_rgb={'buffer' if with_drgb else 'NULL'}"
    bg = B["bg"] if with_bg else None
    dws = B["dwsum"] if with_dwsum else None
    F = O.Forward(B["sigma"], B["rgb"], B["t"], B["off"], STEP, bg)
    G = O.Backward(F, B["rgb"], bg, B["dcolor"], dws)
    sig, rgb, t = _dev(B["sigma"], cuda), _dev(B["rgb"], cuda), _dev(B["t"], cuda)
    off = _dev(B["off"], cuda, torch.int32)
    bg_d = _dev(bg, cuda) if with_bg else None
    dc = _dev(B["dcolor"], cuda)
    dw = _dev(dws, cuda) if with_dwsum else None
    ds = _sent(n + PAD, torch.float32, cuda)
    dr = _sent((n + PAD, 3), torch.float32, cuda) if with_drgb else None
    L.check(L.lib().hrf_composite_backward(sig.data_ptr(), rgb.data_ptr(), t.data_ptr(), off.data_ptr(), R, STEP,
                                           L.ptr(bg_d), dc.data_ptr(), L.ptr(dw), ds.data_ptr(), L.ptr(dr), L.stream()))
    _untouched(ds[n:], "d_sigma")
    _check("hrf_composite_backward d_sigma", case, ds[:n].cpu().numpy(), G.d_sigma, G.d_sigma_err)
    if with_drgb:
        _untouched(dr[n:], "d_rgb")
        _check("hrf_composite_backward d_rgb", case, dr[:n].cpu().numpy(), G.d_rgb, G.d_rgb_err)


# ---------------------------------------------------------------------------------------------------------------------
# fused render
# ---------------------------------------------------------------------------------------------------------------------
def _layout_counts(n_target, rng):
    """Ray lengths laid out on purpose against the 128-sample tiles, then random rays up to n_target samples:
    [0,128) one ray starting and ending on tile borders; 128: a one-sample ray at a tile start; rays ending on the warp
    borders 160/192/224 (32/64/96 into tile 1); one-sample rays at 255 and 256, on both sides of a border, with an empty
    ray between; a ray over 11 tiles (257..1669); tile 13 (1664..1791) then starts inside that ray and ends inside
    the ray at 1770..1809.  Random rays of 0..600 samples follow (every 7th empty), then 5 empty rays."""
    counts = [128, 1, 31, 32, 32, 31, 1, 0, 1, 128 * 11 + 5, 100, 40]
    total = sum(counts)
    i = 0
    while total < n_target:
        c = 0 if i % 7 == 0 else int(rng.integers(1, 601))
        counts.append(c)
        total += c
        i += 1
    return np.array(counts + [0] * 5, np.int64)


def _fused_rays(counts, frames, cuda, seed=0, cam=False):
    """Rays through the unit cube; origins pulled back 6 units along the ray so t runs from about 6 to 8."""
    g = torch.Generator().manual_seed(seed)
    R = counts.shape[0]
    o = torch.randn(R, 3, generator=g)
    o = 2.0 * o / o.norm(dim=1, keepdim=True)
    d = (torch.rand(R, 3, generator=g) - 0.5) * 0.7 - o
    d = d / d.norm(dim=1, keepdim=True)
    o = o - 6.0 * d
    ri = torch.repeat_interleave(torch.arange(R), torch.as_tensor(counts))
    first = torch.cumsum(torch.as_tensor(counts), 0) - torch.as_tensor(counts)
    k = torch.arange(ri.numel()) - first[ri]
    t0 = 6.0 + 1.2 + torch.rand(R, generator=g) * 0.4
    t = (t0[ri] + k.float() * STEP).float()
    fr = torch.tensor(frames, dtype=torch.int32)[torch.randint(0, len(frames), (R,), generator=g)]
    out = dict(o=o.float(), d=d.float(), frames=fr, t=t, ri=ri.long())
    if cam:
        out["cams"] = torch.randint(0, 100, (R,), generator=g, dtype=torch.int32)
    return {k: v.to(cuda).contiguous() for k, v in out.items()}


def _run_fused(nat, samples, off, R, bg, feat, src, want_depth, n_cap, cuda):
    lib = L.lib()
    color, wsum = _sent((R + PAD, 3), torch.float32, cuda), _sent(R + PAD, torch.float32, cuda)
    depth = _sent(R + PAD, torch.float32, cuda) if want_depth else None
    ws = torch.empty(int(lib.hrf_render_fused_workspace_bytes(n_cap)), dtype=torch.uint8, device=cuda)
    if want_depth:
        L.check(lib.hrf_render_fused_depth(C.byref(nat.field), C.byref(samples), off.data_ptr(), R, STEP, L.ptr(bg),
                                           L.ptr(feat), L.ptr(src), color.data_ptr(), wsum.data_ptr(), depth.data_ptr(),
                                           ws.data_ptr(), L.stream()))
    else:
        L.check(lib.hrf_render_fused(C.byref(nat.field), C.byref(samples), off.data_ptr(), R, STEP, L.ptr(bg), L.ptr(feat),
                                     L.ptr(src), color.data_ptr(), wsum.data_ptr(), ws.data_ptr(), L.stream()))
    _untouched(color[R:], "color"), _untouched(wsum[R:], "weights_sum")
    if want_depth:
        _untouched(depth[R:], "depth")
        depth = depth[:R]
    return color[:R], wsum[:R], depth


def _check_fused(name, F, color, wsum, depth):
    _check("fused color", name, color.cpu().numpy(), F.color, F.color_err)
    _check("fused weights_sum", name, wsum.cpu().numpy(), F.wsum, F.wsum_err)
    if depth is not None:
        _check("fused depth", name, depth.cpu().numpy(), F.depth, F.depth_err)


@pytest.mark.parametrize("cam_emb", [0, 2])
def test_fused_render_against_reference(cuda, cam_emb):
    """All four fused variants (encode / from features, with / without depth) on a batch of at least 3 tiles per
    resident CTA, with tile layouts built on purpose, then with a live count below the capacity."""
    from humanrf_b200.volume_rendering import ray_offsets

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas_per_sm = 4 if cam_emb else 5               # launch_field_forward: 5 CTAs per SM, 4 with the 48-wide colour net
    n_target = 3 * sms * ctas_per_sm * O.TILE + 1000
    _, m, frames = make_pair((6,), table_std=2.0, cam_emb=cam_emb)
    rng = np.random.default_rng(11 + cam_emb)
    counts = _layout_counts(n_target, rng)
    g = _fused_rays(counts, frames, cuda, seed=3 + cam_emb, cam=bool(cam_emb))
    R, n = counts.shape[0], int(counts.sum())
    tiles = (n + O.TILE - 1) // O.TILE
    print(f"cam_emb={cam_emb}: {n} samples, {R} rays, {tiles} tiles over {sms * ctas_per_sm} CTAs "
          f"({tiles / (sms * ctas_per_sm):.2f} tiles per CTA)")
    assert tiles >= 3 * sms * ctas_per_sm
    nat = m.native()
    cams = g.get("cams")
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"], cams)
    off = ray_offsets(g["ri"], R)
    sigma, _, rgb, saved = nat.forward(samples, 1, want_geo=False, want_feat=True)
    feat = nat.saved_features(saved, n)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(5)).to(cuda)     # rows read through an index
    shuffled = torch.empty_like(feat)
    shuffled[perm] = feat
    src = perm.to(torch.int32)
    sig_np, rgb_np, t_np, off_np = sigma.cpu().numpy(), rgb.cpu().numpy(), g["t"].cpu().numpy(), off.cpu().numpy().astype(np.int64)
    assert (O.dt32(t_np, STEP) != np.float32(STEP)).any()
    bg = torch.rand(R, 3, generator=torch.Generator().manual_seed(1)).to(cuda)
    Fs = {wb: O.Forward(sig_np, rgb_np, t_np, off_np, STEP, bg.cpu().numpy() if wb else None, kernel="fused")
          for wb in (False, True)}
    for variant, (fe, fs) in (("encode", (None, None)), ("from features", (shuffled, src))):
        for want_depth in (False, True):
            for wb in (False, True):
                name = f"cam_emb={cam_emb} {variant} depth={want_depth} bg={wb}"
                col, ws, dep = _run_fused(nat, samples, off, R, bg if wb else None, fe, fs, want_depth, n, cuda)
                _check_fused(name, Fs[wb], col, ws, dep)
                if want_depth:      # colour and weights sum of the depth variant are the plain kernel's, bit for bit
                    col0, ws0, _ = _run_fused(nat, samples, off, R, bg if wb else None, fe, fs, False, n, cuda)
                    assert torch.equal(col, col0) and torch.equal(ws, ws0), name
    # a live count on the device below the capacity: the samples past it are not seen
    cut_ray = R // 2
    cut = int(off_np[cut_ray])
    off_cut = off.clone()
    off_cut[cut_ray + 1:] = cut
    count = torch.tensor([cut], dtype=torch.int64, device=cuda)
    samples_cut = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"], cams, count_dev=count)
    Fc = O.Forward(sig_np, rgb_np, t_np, off_cut.cpu().numpy().astype(np.int64), STEP, bg.cpu().numpy(), kernel="fused")
    col, ws, dep = _run_fused(nat, samples_cut, off_cut, R, bg, None, None, True, n, cuda)
    _check_fused(f"cam_emb={cam_emb} live count {cut} of {n}", Fc, col, ws, dep)


def test_fused_render_of_infinite_densities(cuda):
    """Zero sigma-net weights and density_scale = inf make the field itself produce sigma = +inf on every sample: each
    ray's first sample is opaque, so colour = its rgb and weights sum = 1, through the tile borders too."""
    from humanrf_b200.volume_rendering import ray_offsets

    _, m, frames = make_pair((6,), table_std=2.0)
    with torch.no_grad():
        m.sigma_net.params.zero_()
    m.density_scale = float("inf")
    m._native = None
    counts = _layout_counts(20000, np.random.default_rng(2))
    g = _fused_rays(counts, frames, cuda, seed=9)
    R, n = counts.shape[0], int(counts.sum())
    nat = m.native()
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"])
    off = ray_offsets(g["ri"], R)
    sigma, _, rgb, _ = nat.forward(samples, 1, want_geo=False, want_feat=False)
    assert torch.isinf(sigma).all()
    bg = torch.rand(R, 3, generator=torch.Generator().manual_seed(4)).to(cuda)
    sig_np, rgb_np, t_np, off_np = sigma.cpu().numpy(), rgb.cpu().numpy(), g["t"].cpu().numpy(), off.cpu().numpy().astype(np.int64)
    F = O.Forward(sig_np, rgb_np, t_np, off_np, STEP, bg.cpu().numpy(), kernel="fused")
    nonempty = counts > 0
    assert (F.wsum[nonempty] == 1).all()
    for want_depth in (False, True):
        col, ws, dep = _run_fused(nat, samples, off, R, bg, None, None, want_depth, n, cuda)
        _check_fused(f"sigma=+inf depth={want_depth}", F, col, ws, dep)
    # the unfused kernels on the same densities
    col = _sent((R, 3), torch.float32, cuda)
    ws = _sent(R, torch.float32, cuda)
    L.check(L.lib().hrf_composite_forward(sigma.data_ptr(), rgb.data_ptr(), g["t"].data_ptr(), off.data_ptr(), R, STEP,
                                          bg.data_ptr(), col.data_ptr(), ws.data_ptr(), None, L.stream()))
    Fu = O.Forward(sig_np, rgb_np, t_np, off_np, STEP, bg.cpu().numpy())
    _check("hrf_composite_forward color", "sigma=+inf", col.cpu().numpy(), Fu.color, Fu.color_err)
    dc = torch.randn(R, 3, generator=torch.Generator().manual_seed(6)).to(cuda)
    ds = _sent(n, torch.float32, cuda)
    L.check(L.lib().hrf_composite_backward(sigma.data_ptr(), rgb.data_ptr(), g["t"].data_ptr(), off.data_ptr(), R, STEP,
                                           bg.data_ptr(), dc.data_ptr(), None, ds.data_ptr(), None, L.stream()))
    G = O.Backward(Fu, rgb_np, bg.cpu().numpy(), dc.cpu().numpy(), None)
    _check("hrf_composite_backward d_sigma", "sigma=+inf", ds.cpu().numpy(), G.d_sigma, G.d_sigma_err)


# ---------------------------------------------------------------------------------------------------------------------
# early stop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_rays", [48, 3000])
def test_early_stop_exact_at_chunk_borders(cuda, num_rays):
    """With the sigma net zeroed (the field MLPs have no bias terms, tests/mlp_oracle.py) every sample's density is
    __expf(0) * density_scale = density_scale, so each ray's optical depth is known exactly.  step = 2^-11 and
    stop_depth = 9.25 make sigma * step and its partial sums exact in fp32; density_scale puts the depth at stop_depth
    one sample before, exactly on, or one sample after the end of chunk K.  Few rays: later chunks of a ray are pulled
    while its earlier ones are still running; many rays: the schedule's usual order."""
    from humanrf_b200.volume_rendering import ray_offsets

    _, m, frames = make_pair((6,), table_std=2.0)
    with torch.no_grad():
        m.sigma_net.params.zero_()
    step, stop = 2.0 ** -11, 9.25
    rng = np.random.default_rng(num_rays)
    lib = L.lib()
    for K in (1, 2, 4):
        for where, samples_to_stop in (("before", 128 * K - 1), ("on", 128 * K), ("after", 128 * K + 1)):
            d = np.float32(stop / samples_to_stop)
            m.density_scale = float(d) * 2048.0          # sigma * step = d exactly
            m._native = None
            nat = m.native()
            counts = rng.integers(128 * K - 3, 128 * (K + 2) + 6, num_rays)
            counts[: min(num_rays, 6)] = [128 * K - 1, 128 * K, 128 * K + 1, 128 * (K + 1), 128 * (K + 2), 128 * (K + 3)][: min(num_rays, 6)]
            g = _fused_rays(counts, frames, cuda, seed=K)
            n = int(counts.sum())
            samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"])
            off = ray_offsets(g["ri"], num_rays)
            full, _, _, _ = nat.forward(samples, 0, want_geo=False, want_feat=False)
            es = _sent(n, torch.float32, cuda)
            nat.density_early_stop(samples, off, num_rays, step, stop_depth=stop, sigma=es)
            assert (full == float(np.float32(m.density_scale))).all()
            skipped = es == 0
            assert not (es == SENT[torch.float32]).any(), "the early-stop pass left a density unwritten"
            torch.testing.assert_close(es[~skipped], full[~skipped], rtol=0, atol=0)
            masks = []
            for sig in (full, es):
                keep = _sent(n, torch.uint8, cuda)
                kept = _sent(num_rays + 1, torch.int32, cuda)
                ot, ori = torch.empty(n, device=cuda), torch.empty(n, dtype=torch.int64, device=cuda)
                cnt = torch.zeros(1, dtype=torch.int64, device=cuda)
                L.check(lib.hrf_prune(sig.data_ptr(), g["t"].data_ptr(), g["ri"].data_ptr(), off.data_ptr(), num_rays, step,
                                      1e-4, 1e-4, keep.data_ptr(), kept.data_ptr(), ot.data_ptr(), ori.data_ptr(), None,
                                      cnt.data_ptr(), L.stream()))
                masks.append(keep.cpu().numpy().astype(bool))
            ref, amb, _ = O.visibility(full.cpu().numpy(), off.cpu().numpy().astype(np.int64), step)
            # every sample of chunk K + 1 and later lies behind depth >= stop_depth
            pos = np.arange(n) - np.repeat(off.cpu().numpy()[:-1].astype(np.int64), counts)
            beyond = pos >= 128 * (K + (where == "after"))
            print(f"early stop K={K} {where} rays={num_rays}: {int(skipped.sum())} of {n} skipped "
                  f"({int(skipped.cpu().numpy()[beyond].sum())} of {int(beyond.sum())} past the crossing chunk), "
                  f"kept {int(masks[0].sum())}, ambiguous {int(amb.sum())}")
            assert not skipped.cpu().numpy()[~beyond].any(), "a chunk before the crossing was skipped"
            assert (masks[0] == masks[1]).all(), (K, where)
            assert not (masks[0] & beyond).any()
            assert ((masks[0] != ref) & ~amb).sum() == 0, (K, where)
