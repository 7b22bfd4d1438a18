"""The compact model (int8 hash tables, toolbox/compact_model.py, DESIGN.md §3.19) on the H100.

* The quantiser against tests/quant_oracle.py: codes, scales and folded vectors bit for bit; the chosen clip ratio
  wherever the float64 errors decide it; non-finite masters refused with their segment, grid and level.
* The int8 encode against encode_oracle.encode over the codes (quant_oracle.int8_field), with encode_oracle's bar:
  every composed feature produced by one of the contraction variants, ambiguous outputs under 1 %, rows with no
  segment all zero.  Query and ray-batch form, the edge positions, frames without a segment.
* Every int8 instantiation agrees with the int8 query: early-stop densities, the fused render (colour, weights sum,
  depth) against composite_oracle applied to the query outputs, the occupancy bake and the density lattice bit for
  bit against densities of the query, at colour-net widths 32 and 48.
* Refusals by every backward C entry, the position gradient, a forward asking for per-grid features, the SIMT path,
  and the Python paths that need gradients.
* save -> load renders bit-identically; malformed files raise ValueError; sizes on a (50,) model.
* Quality on the synthetic training example: int8 against bf16 renders of the held-out views.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import encode_oracle as E
import quant_oracle as Q
from helpers import make_pair
from humanrf_b200 import _lib as L
from test_encode_gpu import _batch, _samples, _widen

pytestmark = pytest.mark.gpu


def _quantize(m):
    from humanrf_b200.toolbox.compact_model import quantize_model

    cm = quantize_model(m)
    torch.cuda.synchronize()
    return cm


def _pair(segs, tables="pair", cam_emb=0):
    _, m, frames = make_pair(segs, table_std=6.0, cam_emb=cam_emb)
    rng = np.random.default_rng(17)
    with torch.no_grad():
        if tables == "wide":
            for fg in m.feature_grids:
                for g in fg.grids() + [fg.vectors]:
                    g.copy_(torch.from_numpy(_widen(g.cpu().numpy(), rng)))
        elif tables == "zero+outlier":      # one all-zero slice, one slice that is zero but for one value
            lay = m.feature_grids[0].layout
            g1 = m.feature_grids[0].grids()[1].view(-1, 2)
            g1[int(lay.offset[3]):int(lay.offset[3] + lay.size[3]), 0] = 0
            g2 = m.feature_grids[0].grids()[2].view(-1, 2)
            a, b = int(lay.offset[9]), int(lay.offset[9] + lay.size[9])
            g2[a:b, 1] = 0
            g2[a + 17, 1] = 3.0
    m.invalidate_native()
    return m, frames


QUANT_CASES = [((6,), "pair"), ((6, 12), "pair"), ((50,), "pair"), ((6, 12), "wide"), ((6,), "zero+outlier")]


@pytest.mark.parametrize("segs,tables", QUANT_CASES, ids=["6", "6-12", "50", "6-12-wide", "6-zero-outlier"])
def test_quantiser_matches_oracle(cuda, segs, tables):
    m, _ = _pair(segs, tables)
    cm = _quantize(m)
    undecided = 0
    for s, fg in enumerate(m.feature_grids):
        lt = E.level_table(fg.layout.log2_hashmap_size)
        grids = [g.detach().cpu().numpy() for g in fg.grids()]
        scales, clip, errs, codes, folded = Q.quantize_segment(grids, fg.vectors.detach().cpu().numpy(), lt)
        assert np.array_equal(cm.scales[s].cpu().numpy().view(np.uint32), scales.view(np.uint32)), f"scales of segment {s}"
        for k in range(4):
            got = cm.codes[s][k].cpu().numpy()
            assert np.array_equal(got, codes[k]), f"codes of segment {s} grid {k}: {int((got != codes[k]).sum())} differ"
        assert np.array_equal(cm.vectors[s].cpu().numpy().view(np.uint32), folded.view(np.uint32)), f"vectors of {s}"
        got_clip = cm.clip[s].cpu().numpy()
        for k in range(4):
            for l in range(16):
                for f in range(2):
                    if Q.decided(errs[k, l, f]):
                        assert got_clip[k, l, f] == clip[k, l, f], (s, k, l, f)
                    else:
                        undecided += 1
    if tables == "zero+outlier":
        assert float(cm.scales[0, 1, 3, 0]) == 0.0 and int(cm.clip[0, 1, 3, 0]) == 0
        assert not cm.codes[0][1][int(m.feature_grids[0].layout.offset[3]):, 0][:8].any()
    chosen = np.bincount(cm.clip.cpu().numpy().ravel(), minlength=8)
    print(f"segs={segs} {tables}: clip ratios chosen {dict(zip(Q.CLIP_RATIOS.tolist(), chosen.tolist()))}; "
          f"{undecided} slices whose two best candidates tie within 1e-9")


def test_non_finite_masters_refused(cuda):
    m, _ = _pair((6, 12))
    lay = m.feature_grids[1].layout
    with torch.no_grad():
        m.feature_grids[1].grids()[2][2 * int(lay.offset[7]) + 11] = float("nan")
    with pytest.raises(RuntimeError, match=r"segment 1, grid 2 \(yzt\), level 7"):
        _quantize(m)


# ------------------------------------------------------------------------------------------------ int8 encode
def _int8_arrays(cm, frames, segs):
    codes = [[c.cpu().numpy() for c in cs] for cs in cm.codes]
    return Q.int8_field(codes, [v.cpu().numpy() for v in cm.vectors], frames, segs)


def _feat(field, s, n, cuda):
    feat = torch.full((n * 32,), -1, dtype=torch.int16, device=cuda)
    sigma = torch.empty(n, dtype=torch.float32, device=cuda)
    L.check(L.lib().hrf_field_forward(C.byref(field), C.byref(s), 0, 0, sigma.data_ptr(), None, None, feat.data_ptr(), None,
                                      L.stream()))
    torch.cuda.synchronize()
    return feat.cpu().numpy().view(np.uint16).reshape(n, 32), sigma


@pytest.mark.parametrize("segs,tables,form", [((6, 12), "pair", "query"), ((6, 12), "wide", "rays"), ((50,), "pair", "rays"),
                                              ((50,), "wide", "query")])
def test_int8_encode_against_oracle(cuda, segs, tables, form):
    m, frames = _pair(segs, tables)
    cm = _quantize(m)
    fa = _int8_arrays(cm, frames, segs)
    bt = _batch(fa, frames, seed=7)
    nat = cm.native()
    s, x, fr = _samples(nat, bt, form, cuda)
    n = x.shape[0]
    feat, _ = _feat(nat.field, s, n, cuda)
    enc = E.encode(fa, x, fr, feat_gpu=feat)
    c = enc.check
    share = c["ambiguous"] / max(c["outputs"], 1)
    print(f"segs={segs} {tables} {form}: {n} rows (no segment {int((enc.seg < 0).sum())}); outside the candidate set "
          f"{c['mismatch']} of {c['outputs']}; ambiguous {share:.3%}")
    assert (feat[enc.seg < 0] == 0).all()
    assert c["mismatch"] == 0, sorted(c["mismatch_rows"])[:10]
    assert share < 0.01
    assert (enc.seg < 0).sum() > 0 and (enc.seg >= 0).sum() > 0.3 * n


# ------------------------------------------------------------------------------------------------ the int8 kernels
@pytest.mark.parametrize("cam_emb", [0, 2])
def test_int8_early_stop_and_fused_render(cuda, cam_emb):
    """Early-stop densities equal the int8 query's where evaluated; the fused render (all four variants of the int8
    encode: with / without depth and background) matches composite_oracle over the int8 query outputs."""
    import composite_oracle as O
    from test_volume_rendering_gpu import STEP, _check_fused, _fused_rays, _layout_counts, _run_fused

    from humanrf_b200.volume_rendering import ray_offsets

    _, m, frames = make_pair((6,), table_std=2.0, cam_emb=cam_emb)
    cm = _quantize(m)
    nat = cm.native()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    counts = _layout_counts(3 * sms * 5 * O.TILE + 1000, np.random.default_rng(11 + cam_emb))
    g = _fused_rays(counts, frames, cuda, seed=3 + cam_emb)
    R, n = counts.shape[0], int(counts.sum())
    samples = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"])
    off = ray_offsets(g["ri"], R)
    sigma, _, rgb, _ = nat.forward(samples, 1, want_geo=False, want_feat=False)
    es = nat.density_early_stop(samples, off, R, STEP)
    torch.cuda.synchronize()
    evaluated = es != 0
    assert torch.equal(es[evaluated], sigma[evaluated]) and int(evaluated.sum()) > 0.3 * n
    sig_np, rgb_np, t_np = sigma.cpu().numpy(), rgb.cpu().numpy(), g["t"].cpu().numpy()
    off_np = off.cpu().numpy().astype(np.int64)
    bg = torch.rand(R, 3, generator=torch.Generator().manual_seed(1)).to(cuda)
    for wb in (False, True):
        F = O.Forward(sig_np, rgb_np, t_np, off_np, STEP, bg.cpu().numpy() if wb else None, kernel="fused")
        for want_depth in (False, True):
            col, ws, dep = _run_fused(nat, samples, off, R, bg if wb else None, None, None, want_depth, n, cuda)
            _check_fused(f"int8 cam_emb={cam_emb} depth={want_depth} bg={wb}", F, col, ws, dep)
    print(f"cam_emb={cam_emb}: {n} samples, {R} rays, early stop evaluated {int(evaluated.sum())}")


@pytest.mark.parametrize("segs,cam_emb", [((50,), 0), ((100, 100, 50), 0), ((50,), 2)])
def test_int8_bake_and_lattice_equal_query(cuda, segs, cam_emb):
    import torch.nn.functional as Fn
    from test_learned_occupancy_gpu import STEP, unfused_bake

    from humanrf_b200.scene_representation.query_io import QueryInput
    from humanrf_b200.synthetic_scene import ellipsoid_grid
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid
    from humanrf_b200.toolbox.mesh_extraction import density_lattice

    _, m, frames = make_pair(segs, table_std=2.0, cam_emb=cam_emb)
    cm = _quantize(m)
    G = 64
    hull = torch.from_numpy(ellipsoid_grid(G)).to(cuda)
    for frame in (frames[0], frames[-1]):
        out, ms = bake_occupancy_grid(cm, frame, hull, STEP, return_max_sigma=True)
        ref_out, ref_ms, _ = unfused_bake(cm, frame, hull, STEP)
        assert torch.equal(ms.view(torch.int32), ref_ms.view(torch.int32)) and torch.equal(out, ref_out)
        lat = density_lattice(cm, frame, hull)
        occ = Fn.pad((hull != 0).float()[None, None], (1, 1, 1, 1, 1, 1))
        z, y, x = torch.nonzero(Fn.max_pool3d(occ, 2, stride=1)[0, 0] > 0, as_tuple=True)
        Gt = torch.tensor(float(G), dtype=torch.float32, device=cuda)
        pos = torch.stack([i.to(torch.float32) / Gt - 0.5 for i in (x, y, z)], -1).contiguous()
        ref = torch.zeros((G + 1,) * 3, dtype=torch.float32, device=cuda)
        with torch.no_grad():
            ref[z, y, x] = cm.density(QueryInput(is_training=False, positions=pos, frame_numbers=torch.full(
                (pos.shape[0],), frame, dtype=torch.int32, device=cuda))).density
        assert torch.equal(lat.view(torch.int32), ref.view(torch.int32))
        print(f"segs={segs} cam_emb={cam_emb} frame={frame}: live {int((out != 0).sum())}, lattice {int((lat != 0).sum())}")


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(cuda):
    from humanrf_b200.scene_representation.query_io import QueryInput
    from humanrf_b200.toolbox.camera_refinement import refine_camera
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.toolbox.normal_maps import export_normal_sequence, render_normal_map
    from humanrf_b200.training import FusedTrainer

    _, m, frames = make_pair((6,))
    cm = _quantize(m)
    nat = cm.native()
    lib = L.lib()
    n = 256
    pos = (torch.rand(n, 3, device=cuda) - 0.5) * 0.5
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, device=cuda), dim=1)
    fr = torch.full((n,), frames[0], dtype=torch.int32, device=cuda)
    s = nat.samples_query(pos, dirs, fr)
    f32 = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=cuda)     # noqa: E731
    sig, rgb, ws = f32(n), f32(n, 3), f32(n * 40)
    feat = torch.zeros(n * 160, dtype=torch.bfloat16, device=cuda)
    d_mlp, sg = f32(m.mlp_grad_elems), torch.zeros(256, dtype=torch.uint8, device=cuda)
    F, S = C.byref(nat.field), C.byref(s)
    calls = {
        "hrf_field_forward egrid": lambda: lib.hrf_field_forward(F, S, 1, 0, sig.data_ptr(), None, rgb.data_ptr(),
                                                                  feat.data_ptr(), feat.data_ptr() + 64 * n, L.stream()),
        "hrf_field_forward simt": lambda: lib.hrf_field_forward(F, S, 1, 1, sig.data_ptr(), None, rgb.data_ptr(), None, None,
                                                                 L.stream()),
        "hrf_field_backward": lambda: lib.hrf_field_backward(F, S, sg.data_ptr(), sig.data_ptr(), rgb.data_ptr(), None, None,
                                                             None, None, 0, d_mlp.data_ptr(), None, ws.data_ptr(), L.stream()),
        "hrf_field_backward_mlp": lambda: lib.hrf_field_backward_mlp(F, S, sig.data_ptr(), rgb.data_ptr(), None, None, None,
                                                                     d_mlp.data_ptr(), None, ws.data_ptr(), L.stream()),
        "hrf_field_backward_mlp_dirs": lambda: lib.hrf_field_backward_mlp_dirs(
            F, S, sig.data_ptr(), rgb.data_ptr(), None, None, None, d_mlp.data_ptr(), None, rgb.data_ptr(), ws.data_ptr(),
            L.stream()),
        "hrf_field_backward_tables": lambda: lib.hrf_field_backward_tables(F, S, sg.data_ptr(), None, None, 0, ws.data_ptr(),
                                                                           0, 4, L.stream()),
        "hrf_field_position_grad": lambda: lib.hrf_field_position_grad(F, S, ws.data_ptr(), rgb.data_ptr(), L.stream()),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="int8 field"):
            L.check(call())
        print("refused:", name)
    R = 8
    es = nat.samples_rays(pos[:R].contiguous(), dirs[:R].contiguous(), fr[:R].contiguous(), torch.zeros(n, device=cuda),
                          torch.arange(R, device=cuda).repeat_interleave(n // R))
    wse = torch.empty(int(lib.hrf_density_early_stop_workspace_bytes(R)), dtype=torch.uint8, device=cuda)
    off = torch.arange(0, n + 1, n // R, dtype=torch.int32, device=cuda)
    with pytest.raises(RuntimeError, match="int8 field"):
        L.check(lib.hrf_field_density_early_stop(F, C.byref(es), off.data_ptr(), R, 4e-4, 9.4, sig.data_ptr(),
                                                 feat.data_ptr(), feat.data_ptr() + 64 * n, wse.data_ptr(), L.stream()))
    # Python paths that need a gradient
    with pytest.raises(RuntimeError, match="CompactHumanRF"):
        cm.density(QueryInput(is_training=False, positions=pos.clone().requires_grad_(True), frame_numbers=fr))
    with pytest.raises(RuntimeError, match="CompactHumanRF"):
        cm.forward(QueryInput(is_training=False, positions=pos, directions=dirs.clone().requires_grad_(True),
                              frame_numbers=fr))
    from helpers import input_batch_of, synthetic_rays
    from humanrf_b200.volume_rendering import render

    ib = input_batch_of(synthetic_rays(16, 8, frames, seed=2), cuda)
    ib.ray_origins.requires_grad_(True)
    with pytest.raises(RuntimeError, match="CompactHumanRF"):
        render(ib, cm, torch.zeros(3, device=cuda), is_training=False)
    for name, call in (("FusedTrainer", lambda: FusedTrainer(cm)),
                       ("refine_camera", lambda: refine_camera(cm, None, 0, [frames[0]])),
                       ("fit_held_out", lambda: CameraResponses.__new__(CameraResponses).fit_held_out(cm, None, [(0, frames[0])])),
                       ("normal maps", lambda: render_normal_map(cm, None, 0, frames[0])),
                       ("normal maps", lambda: export_normal_sequence(cm, None, [(0, frames[0])], "/nonexistent"))):
        with pytest.raises(RuntimeError, match="CompactHumanRF"):
            call()
        print("refused:", name)


# ------------------------------------------------------------------------------------------------ file
def _render(model, frames, cuda):
    from helpers import input_batch_of, synthetic_rays
    from humanrf_b200.volume_rendering import prune_samples, render, render_with_depth

    ib = input_batch_of(synthetic_rays(512, 64, frames, seed=4), cuda)
    prune_samples(ib, model, is_training=False)
    out = render(ib, model, torch.ones(3, device=cuda), is_training=False)
    ib2 = input_batch_of(synthetic_rays(512, 64, frames, seed=4), cuda)
    out2, depth = render_with_depth(ib2, model, torch.ones(3, device=cuda))
    return out.color, out.weights_sum, out2.color, depth


def test_save_load_round_trip_and_sizes(cuda, tmp_path):
    import io

    from humanrf_b200.toolbox.compact_model import CompactHumanRF

    _, m, frames = make_pair((50,), table_std=2.0)
    cm = _quantize(m)
    a = _render(cm, frames, cuda)
    path = tmp_path / "compact.pt"
    cm.save(path)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    cl = CompactHumanRF.load(path, cuda)
    b = _render(cl, frames, cuda)
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - before
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    buf = io.BytesIO()
    torch.save(m.state_dict(), buf)
    sd_bytes, file_bytes = buf.tell(), path.stat().st_size
    fmt = sum(cl.parts().values())
    print(f"(50,): file {file_bytes} B = {file_bytes / sd_bytes:.4f} x state_dict {sd_bytes} B; format {fmt} B; "
          f"device bytes held after load and a render {held} B ({held / fmt:.4f} x); report total "
          f"{cl.report()['total_bytes']} B")
    assert file_bytes <= 0.27 * sd_bytes
    assert cl.device_bytes() <= 1.05 * fmt
    assert held <= 1.05 * fmt + (2 << 20)     # + the allocator's rounding of the small tensors
    for how in ("version", "table_length", "dtype", "truncated"):
        d = torch.load(path, weights_only=True)
        if how == "version":
            d["version"] = 2
        elif how == "table_length":
            d["codes"][0][3] = d["codes"][0][3][1:]
        elif how == "dtype":
            d["vectors"][0] = d["vectors"][0].double()
        bad = tmp_path / f"{how}.pt"
        torch.save(d, bad)
        if how == "truncated":
            bad.write_bytes(path.read_bytes()[:-4096])
        with pytest.raises(ValueError):
            CompactHumanRF.load(bad, cuda)


# ------------------------------------------------------------------------------------------------ quality
def test_quality_on_synthetic_training(cuda):
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "examples"))
    import train_synthetic as T

    from humanrf_b200.parallel import TileShardedRenderer

    _, st = T.main(steps=300, quiet=True, return_state=True)
    student, ds, og, tables, frames, held = (st[k] for k in ("student", "dataset", "occupancy_grid", "tables", "frames",
                                                              "held_out"))
    cm = _quantize(student)
    r16, r8 = TileShardedRenderer(student, og, rays_per_batch=8192), TileShardedRenderer(cm, og, rays_per_batch=8192)
    vs_bf16, gt16, gt8 = [], [], []
    for f in frames:
        cam = tables(held, f)
        n = cam["width"] * cam["height"]
        a = r16.render_range(cam, 0, n).clamp(0, 1)
        b = r8.render_range(cam, 0, n).clamp(0, 1)
        gt = torch.from_numpy(ds._images[(held, f)].reshape(-1, 3).copy()).to(cuda)
        vs_bf16.append(T.psnr(b, a))
        gt16.append(T.psnr(a, gt))
        gt8.append(T.psnr(b, gt))
    print(f"held-out camera {held}, frames {frames}: PSNR int8 vs bf16 per view {np.round(vs_bf16, 2).tolist()} dB; "
          f"mean PSNR vs ground truth bf16 {np.mean(gt16):.3f} dB, int8 {np.mean(gt8):.3f} dB; "
          f"clip ratios chosen {np.bincount(cm.clip.cpu().numpy().ravel(), minlength=8).tolist()}")
    assert min(vs_bf16) >= 40.0
    assert abs(np.mean(gt8) - np.mean(gt16)) <= 0.1
