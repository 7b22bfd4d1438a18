"""Training occupancy on the H100 (humanrf_b200/csrc/training_occupancy.cu, toolbox/training_occupancy.py): the three
kernels against tests/training_occupancy_oracle.py bit for bit, the densities against HumanRF.density, the loader hook,
the schedule, the state round trip, the refusals, the trainer through warm-up, and end to end on a loose-hull scene."""
import ctypes as C

import numpy as np
import pytest
import torch

import training_occupancy_oracle as O
from helpers import make_pair

pytestmark = pytest.mark.gpu


class _Raw:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": "<i4", "data": (ptr, False), "version": 2}


def _slot(handle, G):
    """The words of the ring slot at device address `handle`, as uint32 numpy."""
    words = (G ** 3 + 31) // 32
    return torch.as_tensor(_Raw(int(handle), 4 * words), device="cuda").clone().cpu().numpy().view(np.uint32)


def _sharp_pair(segs, cuda, cam_emb=0):
    """make_pair's model with the density row of the sigma net scaled by 16 (exact in bf16): densities span many
    decades, so live and dead voxels both occur."""
    om, m, frames = make_pair(segs, table_std=6.0, device=cuda, cam_emb=cam_emb)
    with torch.no_grad():
        m.sigma_net.params[32 * 64:32 * 64 + 64] *= 16.0
    m._native = None
    return m, frames


def _density(m, frame, pts):
    from humanrf_b200.scene_representation.query_io import QueryInput

    p = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    with torch.no_grad():
        return m.density(QueryInput(is_training=False, positions=p, frame_numbers=torch.full(
            (p.shape[0],), int(frame), dtype=torch.int32, device=p.device))).density.reshape(-1).cpu().numpy()


def _hull(G, seed):
    from humanrf_b200.synthetic_scene import ellipsoid_grid

    if G == 1:
        return np.full((1, 1, 1), 255, np.uint8)
    if G == 33:
        return np.where(np.random.default_rng(seed).random((G, G, G)) < 0.3, 255, 0).astype(np.uint8)
    return ellipsoid_grid(G, seed)


def _step_between(bound):
    """A step that puts the alpha threshold in the widest gap of the sorted bounds near their 60th percentile, so no
    bound sits within rounding of it."""
    b = np.sort(bound[np.isfinite(bound)].astype(np.float64))
    if b.size < 2:
        return 4e-4
    lo, hi = int(0.5 * b.size), max(int(0.7 * b.size), int(0.5 * b.size) + 1)
    k = lo + int(np.argmax(b[lo + 1:hi + 1] / np.maximum(b[lo:hi], 1e-30)))
    thr = np.sqrt(max(b[k], 1e-30) * b[k + 1])
    return float(-np.log1p(-1e-4) / thr)


CASES = [((6,), 1, (15,), 0), ((6,), 33, (15, 20), 0), ((50,), 64, (15, 64), 0), ((50, 50), 64, (64, 65), 0),
         ((50,), 256, (40,), 0), ((6,), 64, (17,), 2)]


@pytest.mark.parametrize("segs,G,frames,cam_emb", CASES, ids=["seg6-G1", "seg6-G33", "seg50-G64", "border-G64",
                                                              "seg50-G256", "seg6-G64-camemb2"])
def test_kernels_match_oracle(cuda, segs, G, frames, cam_emb):
    from humanrf_b200 import _lib as L
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    m, _ = _sharp_pair(segs, cuda, cam_emb)
    lib = L.lib()
    hull_np = _hull(G, 3)
    hull = torch.from_numpy(hull_np).to(cuda)
    ws = torch.empty(int(lib.hrf_training_occupancy_workspace_bytes(G)), dtype=torch.uint8, device=cuda)
    count = torch.zeros(1, dtype=torch.int32, device=cuda)
    L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), G, None, count.data_ptr(), ws.data_ptr(), L.stream()))
    n = int(count.item())
    ids = torch.empty(n, dtype=torch.int32, device=cuda)
    L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), G, ids.data_ptr(), count.data_ptr(), ws.data_ptr(),
                                               L.stream()))
    ids_o = O.compact(hull_np)
    assert n == ids_o.size and np.array_equal(ids.cpu().numpy(), ids_o)
    seed, decay = 0xC0FFEE + G, 0.9
    for frame in frames:
        bound = torch.full((n,), float("inf"), dtype=torch.float32, device=cuda)
        expect = np.full(n, np.inf, np.float32)
        for counter in (0, 1, 2):
            pts = torch.empty((n, 3), dtype=torch.float32, device=cuda)
            L.check(lib.hrf_training_occupancy_update(C.byref(m.native().field), frame, G, ids.data_ptr(),
                                                      count.data_ptr(), n, seed, counter, decay, bound.data_ptr(),
                                                      pts.data_ptr(), L.stream()))
            pts_o = O.points(ids_o, G, seed, frame, counter)
            assert np.array_equal(pts.cpu().numpy(), pts_o), (frame, counter)
            sigma = _density(m, frame, pts_o)             # HumanRF.density at the oracle's points
            expect = O.update(expect, sigma, decay)
            got = bound.cpu().numpy()
            assert np.array_equal(got.view(np.uint32), expect.view(np.uint32)), (frame, counter)
        # CUDA's expf and numpy's exp may round a bound within ~0.1 % of the threshold to opposite sides: the packed
        # bounds are the evaluated ones moved 2 % away from it, so the pack is checked bit for bit on every voxel
        step = _step_between(expect)
        thr = np.float32(-np.log1p(-1e-4) / step)
        near = np.isfinite(expect) & (np.abs(expect / thr - 1) < 0.02)
        expect = np.where(near, np.where(expect < thr, thr * np.float32(0.98), thr * np.float32(1.02)), expect).astype(
            np.float32)
        bound = torch.from_numpy(expect).to(cuda)
        og = OccupanyGrid(G, 3)
        slot = og.add_grid(hull)
        other = og.add_grid(torch.zeros_like(hull))
        other_before = _slot(other, G)
        counts = torch.zeros(2, dtype=torch.int64, device=cuda)
        L.check(lib.hrf_training_occupancy_pack(ids.data_ptr(), bound.data_ptr(), n, G, step, 1e-4, slot, counts.data_ptr(),
                                                ws.data_ptr(), L.stream()))
        grid_o = O.grid(ids_o, expect, G, step)
        ref = OccupanyGrid(G, 1)
        ref_slot = ref.add_grid(torch.from_numpy(grid_o).to(cuda))
        words = _slot(slot, G)
        assert np.array_equal(words, _slot(ref_slot, G)) and np.array_equal(words, O.pack_bits(grid_o))
        assert np.array_equal(_slot(other, G), other_before)
        live = int(O.live(expect, step).sum())
        assert counts.cpu().tolist() == [live, int((grid_o != 0).sum())]
        if G >= 33:
            assert 0 < live < n, (live, n)


def test_compaction_of_an_empty_and_a_full_hull(cuda):
    from humanrf_b200 import _lib as L

    lib = L.lib()
    for G, fill in ((20, 0), (20, 255), (40, 255)):
        hull = torch.full((G, G, G), fill, dtype=torch.uint8, device=cuda)
        ws = torch.empty(int(lib.hrf_training_occupancy_workspace_bytes(G)), dtype=torch.uint8, device=cuda)
        count = torch.zeros(1, dtype=torch.int32, device=cuda)
        ids = torch.empty(G ** 3, dtype=torch.int32, device=cuda)
        L.check(lib.hrf_training_occupancy_compact(hull.data_ptr(), G, ids.data_ptr(), count.data_ptr(), ws.data_ptr(),
                                                   L.stream()))
        n = int(count.item())
        assert n == (G ** 3 if fill else 0)
        assert np.array_equal(ids[:n].cpu().numpy(), np.arange(n, dtype=np.int32))


# ------------------------------------------------------------------------------------------------ on a loader
def _loader(cuda, mode=None, space=None, frames=range(15, 21), G=64, **kw):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(num_cameras=5, frames=frames, G=G)
    mode = DL.Mode.TRAINING if mode is None else mode
    args = dict(max_num_frames_per_batch=2, use_mask=False, filter_light_bloom=False) if mode == DL.Mode.TRAINING \
        else dict(use_mask=False, filter_light_bloom=False, render_sequence=[(0, frames[0])])
    args.update(kw)
    space = DL.SpacePruningMode.OCCUPANCY_GRID if space is None else space
    return DL(dataset=ds, device="cuda", mode=mode, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
              space_pruning_mode=space, batch_size=4096, camera_numbers=tuple(range(5)),
              frame_numbers=tuple(ds.frames), max_buffer_size=8, **args)


def _batch_arrays(b):
    return [t.detach().cpu().numpy().copy() for t in (b.ray_masks, b.minmaxes, b.ray_origins, b.ray_directions,
                                                       b.sample_distances, b.ray_indices, b.rgba)]


def test_warmup_batches_are_those_without_a_source(cuda):
    from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy

    m, _ = _sharp_pair((6,), cuda)

    def run(with_source):
        np.random.seed(3)
        dl = _loader(cuda)
        occ = TrainingOccupancy(dl, m, interval=2, warmup=8) if with_source else None
        out = []
        it = iter(dl)
        for t in range(1, 8):
            torch.manual_seed(100 + t)
            out.append(_batch_arrays(next(it)))
            if occ is not None:
                assert occ.update(t) == 0
        if occ is not None:
            assert dl.occupancy_source is occ and not occ.active
            assert all(st.evaluations == 0 for st in occ.frames.values()) and len(occ.frames) >= 2
        return out

    a, b = run(False), run(True)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)


def test_refresh_writes_resident_slots_and_a_returning_frame_gets_its_learned_grid(cuda):
    from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy

    m, _ = _sharp_pair((6,), cuda)
    np.random.seed(5)
    dl = _loader(cuda, replace_per_next=1)
    G = dl.occupancy_grid_resolution
    occ = TrainingOccupancy(dl, m, interval=1000, warmup=4)
    for t in range(1, 4):
        occ.update(t)
    assert not occ.active
    assert occ.update(4) > 0 and occ.active and occ.refreshes == 1
    for f, h in dl.frame_to_grid_texture.items():
        st = occ.frames[f]
        assert st.evaluations == 1
        grid = occ.grid(f).cpu().numpy()          # the pack of the current bounds (checked against the oracle above)
        assert np.array_equal(_slot(h, G), O.pack_bits(grid))
        hull = dl.dataset.get_occupancy_grid(f)
        assert not np.any((grid != 0) & (hull == 0))
        live, ngrid, nhull = occ.stats()[f].cpu().tolist()
        assert nhull == st.n and ngrid == int((grid != 0).sum()) and 0 < live <= ngrid <= nhull
    added, seen, returned = [], set(dl.frame_to_grid_texture), []
    real = occ.grid_added

    def spy(frame, hull, handle):
        added.append((int(frame), int(handle)))
        return real(frame, hull, handle)

    occ.grid_added = spy
    handles = set(dl.frame_to_grid_texture.values())
    it = iter(dl)
    for _ in range(60):
        before = {h: _slot(h, G) for h in handles}
        added.clear()
        next(it)
        for f, h in added:
            handles.add(h)
            st = occ.frames[f]
            assert np.array_equal(_slot(h, G), O.pack_bits(occ.grid(f).cpu().numpy()))   # evaluated and packed at entry
            if f in seen:
                returned.append(f)
            seen.add(f)
        for h, w in before.items():
            if h not in [h2 for _, h2 in added]:
                assert np.array_equal(_slot(h, G), w)                     # no other slot was written
        if len(returned) >= 2:
            break
    assert returned, "no frame left the ring and came back"
    assert all(occ.frames[f].evaluations >= 2 for f in returned)


def test_state_round_trip(cuda):
    from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy

    m, _ = _sharp_pair((6,), cuda)
    np.random.seed(6)
    occ = TrainingOccupancy(_loader(cuda), m, interval=1, warmup=0, seed=9)
    occ.update(0)
    occ.update(1)
    sd = occ.state_dict()
    np.random.seed(6)
    dl2 = _loader(cuda)
    occ2 = TrainingOccupancy(dl2, m, interval=1, warmup=0, seed=1)
    occ2.load_state_dict(sd)
    assert occ2.seed == 9 and occ2.t == 1 and occ2.refreshes == 2
    G = dl2.occupancy_grid_resolution
    for f, st in occ.frames.items():
        st2 = occ2.frames[f]
        assert torch.equal(st.bound, st2.bound) and torch.equal(st.ids, st2.ids) and st.evaluations == st2.evaluations
        assert torch.equal(occ.grid(f), occ2.grid(f))
    for f, h in dl2.frame_to_grid_texture.items():
        assert np.array_equal(_slot(h, G), O.pack_bits(occ2.grid(f).cpu().numpy()))
    occ.update(2)
    occ2.update(2)
    for f in dl2.frame_to_grid_texture:
        assert torch.equal(occ.frames[f].bound, occ2.frames[f].bound)
    bad = [dict(sd, G=32), {k: v for k, v in sd.items() if k != "frames"}, dict(sd, t=-1),
           dict(sd, frames={99: next(iter(sd["frames"].values()))})]
    f0, s0 = next(iter(sd["frames"].items()))
    bad.append(dict(sd, frames={f0: dict(s0, ids=s0["ids"].long())}))
    bad.append(dict(sd, frames={f0: dict(s0, bound=s0["bound"][:-1])}))
    bad.append(dict(sd, frames={f0: dict(s0, ids=s0["ids"].flip(0))}))
    bad.append(dict(sd, frames={f0: dict(s0, bound=torch.full_like(s0["bound"], float("nan")))}))
    for b in bad:
        with pytest.raises(ValueError):
            occ2.load_state_dict(b)


def test_refusals(cuda):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.toolbox.compact_model import quantize_model
    from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy
    from humanrf_b200.training import FusedTrainer

    m, _ = _sharp_pair((6,), cuda)
    np.random.seed(7)
    dl = _loader(cuda)
    with pytest.raises(ValueError, match="loader"):
        TrainingOccupancy(_loader(cuda, mode=DL.Mode.VALIDATION), m)
    with pytest.raises(ValueError, match="loader"):
        TrainingOccupancy(_loader(cuda, space=DL.SpacePruningMode.AABB), m)
    small, _ = _sharp_pair((3,), cuda)
    with pytest.raises(ValueError, match="loader"):
        TrainingOccupancy(dl, small)
    with pytest.raises(ValueError, match="model"):
        TrainingOccupancy(dl, quantize_model(m))
    for kw, name in ((dict(interval=0), "interval"), (dict(interval=1.5), "interval"), (dict(warmup=-1), "warmup"),
                     (dict(decay=0.0), "decay"), (dict(decay=1.5), "decay"), (dict(render_step_size=0.0), "render_step"),
                     (dict(render_step_size=float("nan")), "render_step"), (dict(rank=-1), "rank")):
        with pytest.raises(ValueError, match=name):
            TrainingOccupancy(dl, m, **kw)
    dl.occupancy_grid_resolution = 2048
    with pytest.raises(ValueError, match="loader"):
        TrainingOccupancy(dl, m)
    dl.occupancy_grid_resolution = 64
    assert dl.occupancy_source is None                  # nothing was installed by a refused construction
    occ = TrainingOccupancy(dl, m, rank=1)
    with pytest.raises(ValueError, match="training_occupancy"):
        FusedTrainer(m, training_occupancy=occ)


def test_trainer_through_warmup_is_the_one_without_a_source(cuda):
    """For a fixed batch, loss, sample count and parameters with a source in warm-up differ from a run without one no
    more than two runs without one differ from each other (the order of the float atomics)."""
    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy
    from humanrf_b200.training import FusedTrainer

    b = synthetic_rays(4096, 32, list(range(15, 21)), seed=4)
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri", "rgba")}
    np.random.seed(8)
    dl = _loader(cuda)

    def run(occ_on):
        m, _ = make_model((6,), seed=1, device=cuda)
        occ = TrainingOccupancy(dl, m, warmup=100) if occ_on else None
        tr = FusedTrainer(m, training_occupancy=occ)
        out = []
        for _ in range(3):
            loss = tr.step(g["o"], g["d"], g["frames"], g["t"], g["ri"], g["rgba"], 4096, return_loss=True)
            out.append((loss, int(tr.last["samples"])))
        if occ is not None:
            assert occ.t == 3 and not occ.active and all(st.evaluations == 0 for st in occ.frames.values())
        return out, torch.cat([p.detach().reshape(-1) for p in m.hot_parameters()])

    (a, pa), (b_, pb), (c, pc) = run(False), run(False), run(True)
    assert a[0][1] == c[0][1]
    for (la, na), (lb, nb), (lc, nc) in zip(a, b_, c):
        assert abs(lc - la) <= 4 * abs(lb - la) + 1e-5 * abs(la)
        assert abs(nc - na) <= 4 * abs(nb - na) + 2
    noise = float((pb - pa).norm())
    assert float((pc - pa).norm()) <= 4 * noise + 1e-6 * float(pa.norm())


# ------------------------------------------------------------------------------------------------ end to end
def compare_on_pool(state, num_rays=1 << 16, seed=0):
    """The trained student on the same un-jittered ray batches of the training pool, sampled through the hulls and
    through the learned grids: candidates, rays kept, survivors of pruning and the rendered colours."""
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid
    from humanrf_b200.volume_rendering import prune_samples, render

    dl, occ, m, ds = state["loader"], state["training_occupancy"], state["student"], state["dataset"]
    G = dl.occupancy_grid_resolution
    slot_frames = [int(f) for f in dl.frame_numbers_cuda.cpu().tolist()]
    for f in set(slot_frames):
        occ.evaluate(f)                        # every pooled frame's grid from the trained model
    ring = OccupanyGrid(G, 2 * dl.buffer_size)
    hull_handles = torch.tensor([ring.add_grid(torch.from_numpy(ds.get_occupancy_grid(f)).cuda().contiguous())
                                 for f in slot_frames], dtype=torch.int64, device="cuda")
    learned_handles = torch.tensor([ring.add_grid(occ.grid(f)) for f in slot_frames], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, dl.buffer_size * dl.num_pixels_per_camera, (num_rays,), device="cuda", generator=gen)
    W, H = dl.resolution
    out = {}
    for kind, handles in (("hull", hull_handles), ("learned", learned_handles)):
        r = dl.ray_sampler_func(dl.pixel_colors.view(-1, 4), dl.light_mask.view(-1), dl.frame_numbers_cuda,
                                dl.camera_numbers_cuda, handles, dl.landscape_mode_cuda, idx, dl.inverse_krs_cuda,
                                dl.camera_origins_cuda, dl.aabb, G, W, H, 4e-4, False)
        (ro, rd, rgba, fr, cams, mm, mask, dist, rel) = r
        ib = InputBatch(ray_origins=ro.view(-1, 3), ray_directions=rd.view(-1, 3), minmaxes=mm.view(-1, 2),
                        rgba=rgba.view(-1, 4), ray_masks=mask.view(-1, 1), frame_numbers=fr.view(-1, 1),
                        camera_numbers=cams.view(-1, 1), unique_frame_numbers=torch.unique(fr).view(-1, 1),
                        sample_distances=dist.view(-1, 1), ray_indices=rel.view(-1).long(), width=W, height=H)
        cand = int(ib.sample_distances.numel())
        color = torch.zeros((num_rays, 3), device="cuda")
        surv = 0
        if ib.num_rays > 0 and cand > 0:
            prune_samples(ib, m, is_training=False)
            surv = int(ib.sample_distances.numel())
            with torch.no_grad():
                color[mask.view(-1)] = render(ib, m, torch.zeros(3, device="cuda"), is_training=False).color
        out[kind] = dict(candidates=cand, rays=int(mask.sum()), survivors=surv, color=color)
    mse = float(((out["hull"]["color"] - out["learned"]["color"]) ** 2).mean())
    psnr = float("inf") if mse == 0 else -10 * np.log10(mse)
    return dict(candidate_ratio=out["learned"]["candidates"] / out["hull"]["candidates"],
                survivor_ratio=out["learned"]["survivors"] / max(out["hull"]["survivors"], 1),
                rays_left=1 - out["learned"]["rays"] / max(out["hull"]["rays"], 1), psnr=psnr,
                hull=out["hull"]["candidates"], learned=out["learned"]["candidates"])


def test_loose_hull_scene_end_to_end(cuda):
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "examples"))
    import train_synthetic

    hist, state = train_synthetic.main(steps=600, log_every=600, quiet=True, return_state=True, loose_hull=True,
                                       training_occupancy=dict(warmup=256, interval=16))
    r = compare_on_pool(state)
    print(f"loose hull, 600 steps: held-out PSNR {hist[-1][1]:.2f} dB; candidates {r['learned']} / {r['hull']} = "
          f"{r['candidate_ratio']:.3f} of the hull's (bar <= 0.6), survivors {r['survivor_ratio']:.4f} (bar >= 0.995), "
          f"rays leaving the batch {r['rays_left']:.4f}, images hull vs learned {r['psnr']:.2f} dB (bar >= 50)")
    # measured on an H100 80GB HBM3 at 700 W: 0.521 of the candidates (first estimated at <= 0.5), 0.9992 of the
    # survivors, 83.2 dB, 34 % of the rays leave the batch
    assert state["training_occupancy"].refreshes >= 2
    assert r["candidate_ratio"] <= 0.6
    assert r["survivor_ratio"] >= 0.995
    assert r["psnr"] >= 50.0
