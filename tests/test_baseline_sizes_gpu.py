"""CUDA vs oracle parity on BASELINE's own table sizes (VERDICT r1, item 1).

segment_sizes (50,) -> log2T 18 (dense levels 0-2: 32768 / 79512 / 175616 entries, 3 is hashed), (100,) -> log2T 19
(dense levels 0-3, 405224 entries at level 3), (100,100,50) = the 250-frame model of configs[3]
(humanrf/run.py:44-56, table sizes humanrf/scene_representation/humanrf.py:104-109).  The small-model suites
(test_field_gpu / test_backward_gpu, log2T 15/16) only ever see ONE dense level of exactly 32^3 entries, so the
non-power-of-two dense index path (csrc/field_common.cuh corner_indices), level offsets beyond 2^16 entries and
multi-segment routing at full size are covered here: forward, backward in all three saved-feature modes, the table
scatter alone at float64 precision, prune + render end to end, and an image-level PSNR against the fp32 oracle.

The samples are a 2048-sample slice of the bench batch itself (synthetic_rays(4096, 512, seed=123)).
Tolerances are those of test_field_gpu / test_backward_gpu / test_scatter_gpu (stated there).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import input_batch_of, make_pair, synthetic_rays
from humanrf_b200 import _lib as L
from oracle import field as OF
from oracle import hashgrid
from oracle import rendering as R

pytestmark = pytest.mark.gpu
CONFIGS = {"seg50": (50,), "seg100": (100,), "seg100-100-50": (100, 100, 50)}
GRID_AXES = ([0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3])
VECTOR_OF_GRID = (3, 2, 0, 1)


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module", params=list(CONFIGS), ids=list(CONFIGS))
def pair(request, cuda):
    segs = CONFIGS[request.param]
    om, m, frames = make_pair(segs, table_std=6.0, device=cuda)
    return segs, om, m, frames


def bench_slice(frames, segs, rays=16, per_ray=128):
    """`rays` x `per_ray` consecutive samples of the 4096 x 512 bench batch (seed 123), in query form.  For
    multi-segment models the frames of the chosen rays are re-drawn so that every segment AND both sides of every
    segment boundary are hit (the bench batch's 8 random frames of 250 may miss a segment)."""
    b = synthetic_rays(4096, 512, frames, seed=123)
    pick = torch.arange(rays) * (4096 // rays) + 3
    fr = b["frames"].clone()
    if len(segs) > 1:
        edges = np.cumsum(segs)
        special = [frames[0], frames[-1]] + [frames[e - 1] for e in edges[:-1]] + [frames[e] for e in edges[:-1]]
        for j, r in enumerate(pick.tolist()):
            fr[r] = special[j % len(special)]
    sel = torch.cat([torch.arange(per_ray) + 512 * r + 97 for r in pick.tolist()])
    ri = b["ri"][sel]
    pos = b["o"][ri] + b["t"][sel].unsqueeze(1) * b["d"][ri]          # volume_rendering.py:66-69 (fp32 mul, then add)
    return pos.contiguous(), b["d"][ri].contiguous(), fr[ri].contiguous()


def test_level_tables_have_the_dense_non_pow2_levels(pair):
    """What this file is for: the dense levels beyond 32^3 exist at these sizes (SURVEY 8 level table)."""
    segs, om, m, _ = pair
    for s, ss in enumerate(segs):
        lay = m.feature_grids[s].layout
        dense = [l for l in range(16) if not (lay.hashed_mask >> l) & 1]
        sizes = [int(lay.size[l]) for l in dense]
        assert sizes[:3] == [32768, 79512, 175616]
        assert (ss == 100) == (len(dense) == 4 and sizes[3] == 405224)
        assert int(lay.offset[15]) + int(lay.size[15]) == lay.n_entries > (1 << 16)


@pytest.mark.parametrize("impl", [0, 1], ids=["tcgen05", "simt-debug"])
def test_forward_matches_oracle(cuda, pair, impl):
    segs, om, m, frames = pair
    pos, dirs, fr = bench_slice(frames, segs)
    with torch.no_grad():
        osig, ogeo, orgb = om.forward(pos, dirs, fr)
        ofeat = om.features(pos, fr).numpy()
    nat = m.native()
    s = nat.samples_query(pos.to(cuda), dirs.to(cuda), fr.to(cuda))
    sig, geo, rgb, saved = nat.forward(s, 1, want_geo=True, want_feat=True, mlp_impl=impl)
    torch.cuda.synchronize()
    n = pos.shape[0]
    # composed features, level by level: a wrong corner index at any level moves that level's pair by O(1)
    feat = nat.saved_features(saved, n).float().cpu().numpy()
    ferr = np.abs(feat - ofeat).reshape(n, 16, 2).max(axis=(0, 2))
    scale = np.abs(ofeat).reshape(n, 16, 2).max(axis=(0, 2))
    print("per-level feature err / scale:", np.round(ferr / scale, 4))
    assert (ferr <= 2.0 ** -7 * scale + 1e-6).all(), (ferr, scale)
    # per-(level, grid) interpolated features saved for the backward scatter: egrid[(4 l + k) * n + i].  Checked from a
    # second run of the same path into a sentinel-filled buffer, so that nothing the kernel was asked to write can pass
    # as the leftovers of an earlier allocation (`saved` is torch.empty); both runs must write the same bytes.
    seg_of = om.f2s[fr.numpy()]
    sent = torch.full((n * 160,), -1, dtype=torch.int16, device=cuda)
    L.check(L.lib().hrf_field_forward(C.byref(nat.field), C.byref(s), 1, impl, torch.empty_like(sig).data_ptr(), None, None,
                                      sent.data_ptr(), sent.data_ptr() + 64 * n, L.stream()))
    torch.cuda.synchronize()
    assert torch.equal(sent, saved.view(torch.int16))
    eg = sent[n * 32:].view(torch.int32).view(64, n)
    lo = (eg << 16).view(torch.float32).cpu().numpy()
    hi = (eg & -65536).view(torch.float32).cpu().numpy()
    xyzt = torch.cat((pos + 0.5, torch.from_numpy(om.f2t[fr.numpy()]).unsqueeze(1)), dim=1).float()
    for si, sd in enumerate(om.segments):
        sel = np.nonzero(seg_of == si)[0]
        if sel.size == 0:
            continue
        for k in range(4):
            e = hashgrid.encode(OF.rbf(sd.grids[k]), xyzt[sel][:, GRID_AXES[k]], sd.log2T).numpy().reshape(-1, 16, 2)
            got = np.stack((lo[k::4][:, sel].T, hi[k::4][:, sel].T), axis=2)       # [n_sel, 16, 2]
            tol = 2.0 ** -8 * np.abs(e).max(axis=(0, 2), keepdims=True) + 1e-6
            assert (np.abs(got - e) <= tol).all(), (si, k, np.abs(got - e).max(axis=(0, 2)))
    h0 = geo[:, 0].float().cpu().numpy()
    oh0 = np.log(osig.numpy() / 100.0)
    assert np.abs(h0 - oh0).max() < 3e-2
    rel = np.abs(sig.cpu().numpy() - osig.numpy()) / np.maximum(osig.numpy(), 1e-3)
    err = np.abs(rgb.cpu().numpy() - orgb.numpy())
    print(f"[{segs} impl={impl}] density rel max {rel.max():.3e} mean {rel.mean():.3e}; radiance abs max {err.max():.3e}")
    assert rel.max() < 4e-2 and rel.mean() < 6e-3
    assert err.max() < 6e-3 and err.mean() < 1e-3
    assert len(set(seg_of.tolist())) == len(segs), "every segment must be exercised"


@pytest.mark.parametrize("use_saved_features", [True, False, "composed-only"], ids=["saved", "re-encode", "re-gather"])
def test_backward_matches_autograd(cuda, pair, use_saved_features):
    segs, om, m, frames = pair
    for p in om.parameters():
        p.requires_grad_(True)
        p.grad = None
    pos, dirs, fr = bench_slice(frames, segs, rays=8, per_ray=128)
    n = pos.shape[0]
    g = torch.Generator().manual_seed(5)
    d_sigma = torch.randn(n, generator=g) * 1e-2
    d_rgb = torch.randn(n, 3, generator=g)
    osig, _, orgb = om.forward(pos, dirs, fr)
    ((osig * d_sigma).sum() + (orgb * d_rgb).sum()).backward()
    nat = m.native()
    s = nat.samples_query(pos.to(cuda), dirs.to(cuda), fr.to(cuda))
    _, _, _, feat = nat.forward(s, 1, want_geo=False, want_feat=True)
    grads = [torch.zeros_like(p) for p in m.hot_parameters()]
    saved = {True: feat, False: None, "composed-only": feat[: n * 32].clone()}[use_saved_features]
    nat.backward(s, d_sigma.to(cuda), d_rgb.to(cuda).contiguous(), saved, grads)
    torch.cuda.synchronize()
    i = 0
    for si, seg in enumerate(om.segments):
        lay = m.feature_grids[si].layout
        for k in range(4):
            ref, got = seg.grids[k].grad.reshape(-1), grads[i].cpu()
            assert ((got != 0) & (ref == 0)).sum() == 0, "gradient written to an untouched table entry"
            e = _relnorm(got, ref)
            # the dense non-power-of-two levels on their own (they carry a small share of the norm)
            worst_dense = 0.0
            for l in range(1, 4):
                if (lay.hashed_mask >> l) & 1:
                    continue
                a, b = 2 * int(lay.offset[l]), 2 * (int(lay.offset[l]) + int(lay.size[l]))
                worst_dense = max(worst_dense, _relnorm(got[a:b], ref[a:b]))
            print(f"seg{si} grid{k} relnorm {e:.3e} dense levels 1-3 {worst_dense:.3e} touched {(ref != 0).sum().item()}")
            assert e < 3e-2 and worst_dense < 3e-2
            i += 1
        e = _relnorm(grads[i].cpu(), seg.vectors.grad)
        assert e < 3e-2, (si, e)
        i += 1
    ref_sigma = torch.cat([w.grad.reshape(-1) for w in om.w_sigma])
    ref_color = torch.cat([w.grad.reshape(-1) for w in om.w_color])
    es, ec = _relnorm(grads[i].cpu(), ref_sigma), _relnorm(grads[i + 1].cpu(), ref_color)
    print(f"sigma-net relnorm {es:.3e}  colour-net relnorm {ec:.3e}")
    assert es < 3e-2 and ec < 3e-2
    for p in om.parameters():
        p.requires_grad_(False)
        p.grad = None


def test_table_scatter_matches_float64_autograd(cuda, pair):
    """The default table / vector gradient scatter (scatter_v6.cu) alone at 1e-5 against float64 autograd, on the dense and hashed levels
    of the full-size tables."""
    segs, om, m, frames = pair
    pos, _, fr = bench_slice(frames, segs, rays=8, per_ray=128)
    n = pos.shape[0]
    seg = om.f2s[fr.numpy()]
    xyzt = torch.cat((pos + 0.5, torch.from_numpy(om.f2t[fr.numpy()]).unsqueeze(1)), dim=1).float()
    g = torch.Generator().manual_seed(2)
    d_out = torch.randn(n, 32, generator=g)
    d_out[::7] = 0
    nat = m.native()
    ref_tables, ref_vectors = [], []
    for s, sd in enumerate(om.segments):
        sel = torch.from_numpy(np.nonzero(seg == s)[0])
        # the kernel re-gathers the bf16 shadows: reference tables = the bf16-rounded values in float64
        tabs = [t.detach().bfloat16().double().requires_grad_(True) for t in sd.grids]
        vec = sd.vectors.detach().double().requires_grad_(True)
        c = xyzt[sel]
        sv = OF.lerp_vectors(vec, c)
        out = sum(hashgrid.encode(tabs[k], c[:, GRID_AXES[k]], sd.log2T) * sv[VECTOR_OF_GRID[k]] for k in range(4))
        (out * d_out[sel].double()).sum().backward()
        ref_tables.append([t.grad.reshape(-1) if t.grad is not None else torch.zeros(t.numel(), dtype=torch.float64) for t in tabs])
        ref_vectors.append(vec.grad if vec.grad is not None else torch.zeros_like(vec))
    ws = torch.zeros(n * 40, dtype=torch.float32, device=cuda)
    ws[: 32 * n] = d_out.reshape(n, 16, 2).permute(1, 0, 2).reshape(-1).to(cuda)
    ws[32 * n: 36 * n] = xyzt.reshape(-1).to(cuda)
    ws.view(torch.uint8)[144 * n: 145 * n] = torch.from_numpy(seg.astype(np.uint8)).to(cuda)
    grads = [torch.zeros_like(p) for p in m.hot_parameters()]
    sg = (L.SegmentGrads * m.num_segments)()
    for s in range(m.num_segments):
        for k in range(4):
            sg[s].grid[k] = grads[5 * s + k].data_ptr()
        sg[s].vectors = grads[5 * s + 4].data_ptr()
    sg_dev = torch.from_numpy(np.frombuffer(bytes(sg), dtype=np.uint8).copy()).to(cuda)
    samples = nat.samples_query(pos.to(cuda), None, fr.to(cuda).to(torch.int32))
    L.check(L.lib().hrf_field_backward_tables(C.byref(nat.field), C.byref(samples), sg_dev.data_ptr(), None, None, 0, ws.data_ptr(),
                                              0, 4, L.stream()))
    torch.cuda.synchronize()
    for s in range(m.num_segments):
        for k in range(4):
            got, ref = grads[5 * s + k].cpu(), ref_tables[s][k]
            assert ((got != 0) & (ref == 0)).sum() == 0
            e = _relnorm(got, ref)
            worst = float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
            print(f"seg{s} grid{k}: relnorm {e:.2e} worst entry {worst:.2e} touched {(ref != 0).sum().item()}")
            assert e < 1e-5 and worst < 1e-5
        assert _relnorm(grads[5 * s + 4].cpu(), ref_vectors[s]) < 1e-5


def test_prune_and_render_match_oracle(cuda, pair):
    """prune_samples + render (the public API, ray-batch form) vs the oracle pipeline on rays of the bench batch."""
    from humanrf_b200.volume_rendering import prune_samples, render

    segs, om, m, frames = pair
    full = synthetic_rays(4096, 512, frames, seed=123)
    nr, per = 24, 96
    pick = torch.arange(nr) * 170 + 1
    sel = torch.cat([torch.arange(per) + 512 * r + 40 for r in pick.tolist()])
    b = dict(o=full["o"][pick], d=full["d"][pick], frames=full["frames"][pick], cams=full["cams"][pick], rgba=full["rgba"][pick],
             t=full["t"][sel], ri=torch.arange(nr).repeat_interleave(per))
    ib = input_batch_of(b, cuda)
    pos = b["o"][b["ri"]] + b["t"].unsqueeze(1) * b["d"][b["ri"]]
    with torch.no_grad():
        osig, _ = om.density(pos, b["frames"][b["ri"]])
    prune_samples(ib, m, is_training=False)
    keep_o = R.prune_mask(osig, b["ri"]).numpy()
    got_t, exp_t = ib.sample_distances.view(-1).cpu().numpy(), b["t"].numpy()[keep_o]
    common = np.intersect1d(got_t, exp_t).size
    print("pruned:", got_t.size, "oracle:", exp_t.size, "common:", common)
    assert abs(got_t.size - exp_t.size) <= 0.02 * exp_t.size + 2 and common >= 0.97 * min(got_t.size, exp_t.size)
    t_k, ri_k = ib.sample_distances.view(-1).cpu(), ib.ray_indices.cpu()
    bg = torch.rand(nr, 3, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        out = render(ib, m, bg.to(cuda), is_training=False)
        p2 = b["o"][ri_k] + t_k.unsqueeze(1) * b["d"][ri_k]
        s_o, _, c_o = om.forward(p2, b["d"][ri_k], b["frames"][ri_k])
        col_o, ws_o = R.render(t_k, s_o, c_o, ri_k, nr, bg)
    np.testing.assert_allclose(out.color.cpu().numpy(), col_o.numpy(), atol=6e-3)
    np.testing.assert_allclose(out.weights_sum.cpu().numpy(), ws_o.numpy(), atol=6e-3)


def _psnr(a, b):
    """humanrf/trainer.py:216-222 : -10 log10(mean((a-b)^2)) on [0,1] images."""
    mse = float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))
    return float("inf") if mse == 0 else -10.0 * np.log10(mse)


@pytest.mark.parametrize("segs", [(50,)], ids=["seg50"])
def test_image_psnr_vs_fp32_oracle(cuda, segs):
    """A 64x48 image through sampler -> prune -> render on the CUDA path (bf16 tables / activations) against the SAME
    pipeline evaluated by the un-rounded fp32 oracle (oracle sampler, oracle pruning, oracle field, oracle compositing).
    SURVEY 8c: image PSNR(new vs reference render) >= 45 dB."""
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.parallel import TileShardedRenderer
    from humanrf_b200.synthetic_scene import make_scene
    from oracle import sampler as OS

    om, m, frames = make_pair(segs, table_std=6.0, device=cuda, bf16=False)
    W, H, G = 64, 48, 64
    sc = make_scene(num_images=1, width=W, height=H, G=G, portrait_every=0)
    og = OccupanyGrid(G, 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    cam = dict(frame_numbers=t(sc["frame_numbers"]), camera_numbers=t(sc["camera_numbers"]),
               grid_handles=torch.tensor([og.add_grid(t(sc["grids"][0]))], dtype=torch.int64, device=cuda),
               landscape=t(sc["landscape"]), inverse_krs=t(sc["inverse_krs"]), camera_origins=t(sc["camera_origins"]),
               aabb=t(sc["aabb"]), G=G, width=W, height=H)
    img = TileShardedRenderer(m, og, rays_per_batch=W * H).render_range(cam, 0, W * H).cpu().numpy()
    # ---- oracle pipeline on the CPU
    o, d, _, fr, _, _, ray_mask, tt, ri = OS.get_data(
        sc["rgba"], sc["light_mask"], sc["frame_numbers"], sc["camera_numbers"], sc["grids"], sc["landscape"],
        np.arange(W * H, dtype=np.int64), sc["inverse_krs"], sc["camera_origins"], sc["aabb"], G, W, H, 4e-4, False,
        occupancy=True, samples=True)
    o, d, tt = torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(tt)
    fr, ri = torch.from_numpy(fr).to(torch.int32), torch.from_numpy(ri).long()
    with torch.no_grad():
        pos = o[ri] + tt.unsqueeze(1) * d[ri]
        sig, _ = om.density(pos, fr[ri])
        keep = R.prune_mask(sig, ri)
        tk, rk = tt[keep], ri[keep]
        pk = o[rk] + tk.unsqueeze(1) * d[rk]
        s2, _, c2 = om.forward(pk, d[rk], fr[rk])
        col, _ = R.render(tk, s2, c2, rk, o.shape[0], torch.zeros(o.shape[0], 3))
    ref = np.zeros((W * H, 3), np.float32)
    ref[np.nonzero(np.asarray(ray_mask))[0]] = col.numpy()
    psnr = _psnr(img, ref)
    print(f"image PSNR CUDA(bf16) vs fp32 oracle: {psnr:.2f} dB; object pixels {(ref.sum(1) > 0).mean():.2%}; "
          f"max abs pixel err {np.abs(img - ref).max():.3e}")
    assert (ref.sum(1) > 0).mean() > 0.05
    assert psnr >= 45.0
