"""Data-parallel camera refinement without a GPU: the float64 reference of the ranked pose step (tests/pose_dp_oracle.py)
against the single-rank references and the union batch, the wrong steps it tells apart, and the construction checks
(world size, and every rank's cameras and settings in a 2-process gloo group)."""
import os

import numpy as np
import pytest
import torch

import intrinsics_oracle as IO
import pose_dp_oracle as DO
import pose_oracle as PO


def _state(C, K, rng=None):
    p = np.zeros((C, K)) if rng is None else rng.standard_normal((C, K)) * 1e-2
    return dict(params=p, m=np.zeros((C, K)), v=np.zeros((C, K)), steps=np.zeros(C, np.int64))


def _copy(st):
    return {k: v.copy() for k, v in st.items()}


def _equal(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("K", [6, 10])
def test_one_rank_is_the_single_rank_step_bit_for_bit(K):
    rng = np.random.default_rng(K)
    C = 9
    fixed = np.zeros(C, bool)
    fixed[0] = True
    a, b = _state(C, K, rng), None
    b = _copy(a)
    for _ in range(5):
        g = (rng.standard_normal((C, K)) * 10.0 ** rng.uniform(-6, 1, (C, 1))).astype(np.float32)
        n = rng.integers(0, 3, C).astype(np.int32)
        if K == 6:
            DO.ranked_step(a, [g], [n], [0], fixed, 3e-3)
            PO.adam(b, g, n, fixed, 3e-3)
        else:
            DO.ranked_step(a, [g], [n], [0], fixed, 3e-3, 1e-3)
            IO.adam(b, g, n, fixed, 3e-3, 1e-3)
    assert _equal(a, b) and a["steps"].sum() > 0


@pytest.mark.parametrize("W", [2, 3, 8])
def test_reduced_gradient_is_the_union_batch_gradient(W):
    """Per-ray loss gradients split over W ranks at unequal shares (one rank empty); rank r's loss is its mean times
    W R_r / R_total, so its per-camera record is W / R_total times its rays' sum."""
    rng = np.random.default_rng(W)
    R, C, K = 3000, 7, 10
    cams = rng.integers(0, C, R)
    terms = rng.standard_normal((R, K)) * rng.uniform(0.01, 10.0, (R, 1))
    cuts = np.sort(rng.choice(np.arange(1, R), W - 2, replace=False))
    bounds = np.concatenate(([0, 0], cuts, [R]))            # rank 0 empty, the others unequal
    union = np.zeros((C, K))
    np.add.at(union, cams, terms / R)
    grads, counts = [], []
    for r in range(W):
        lo, hi = bounds[r], bounds[r + 1]
        g = np.zeros((C, K))
        np.add.at(g, cams[lo:hi], terms[lo:hi] * (W * (hi - lo) / R) / max(hi - lo, 1))
        grads.append(g)
        counts.append(np.bincount(cams[lo:hi], minlength=C))
    assert counts[0].sum() == 0
    g, touched = DO.reduce_records(grads, counts)
    np.testing.assert_allclose(g, union, rtol=1e-12, atol=1e-12 * np.abs(union).max())
    assert np.array_equal(touched, np.bincount(cams, minlength=C) > 0)


# ------------------------------------------------------------------------------------------------ wrong steps
def _reversed(grads, counts):
    s = np.asarray(grads[-1]).astype(np.float64)
    for r in range(len(grads) - 2, -1, -1):
        s = s + np.asarray(grads[r]).astype(np.float64)
    return s / len(grads), DO.reduce_records(grads, counts)[1]


def _no_division(grads, counts):
    g, t = DO.reduce_records(grads, counts)
    return g * len(grads), t


def _intersection(grads, counts):
    g, _ = DO.reduce_records(grads, counts)
    return g, np.logical_and.reduce([np.asarray(c) != 0 for c in counts])


def _wrong_step(reduce, state, grads, counts, errors, fixed, lr, ignore_peer_errors=False, rank=0):
    if (errors[rank] if ignore_peer_errors else any(errors)):
        return
    g, touched = reduce(grads, counts)
    PO.adam(state, g, touched.astype(np.int64), fixed, lr)


def _records_w8(rng):
    """Eight ranks' records with each of the distinguishing features: camera 1's gradients round differently summed
    from rank 7 down (2^-30 + 2^30 - 2^30 is 0 in rank order, 2^-30 from the top); camera 2 is seen by rank 7 only;
    rank 3 is empty; camera 0 is fixed."""
    W, C = 8, 4
    grads = [(rng.standard_normal((C, 6)) * 1e-3).astype(np.float32) for _ in range(W)]
    counts = [rng.integers(1, 50, C).astype(np.int32) for _ in range(W)]
    for r in range(W):
        grads[r][1] = 0.0
        grads[r][2], counts[r][2] = 0.0, 0
    grads[0][1], grads[1][1], grads[2][1] = 2.0 ** -30, 2.0 ** 30, -(2.0 ** 30)
    grads[7][2], counts[7][2] = 0.5, 3
    grads[3][:], counts[3][:] = 0.0, 0
    return grads, counts


@pytest.mark.parametrize("wrong", ["reversed", "no_division", "intersection", "peer_error_ignored"])
def test_wrong_steps_are_told_apart(wrong):
    rng = np.random.default_rng(11)
    grads, counts = _records_w8(rng)
    fixed = np.array([True, False, False, False])
    errors = [0] * 8
    if wrong == "peer_error_ignored":
        errors[5] = 1
    ref = _state(4, 6)
    DO.ranked_step(ref, grads, counts, errors, fixed, 1e-3)
    got = _state(4, 6)
    reduce = {"reversed": _reversed, "no_division": _no_division, "intersection": _intersection,
              "peer_error_ignored": DO.reduce_records}[wrong]
    _wrong_step(reduce, got, grads, counts, errors, fixed, 1e-3, ignore_peer_errors=wrong == "peer_error_ignored")
    assert not _equal(got, ref)
    if wrong == "reversed":
        assert ref["params"][1].tolist() == [0.0] * 6 and got["params"][1, 1] != 0.0
    if wrong == "intersection":
        assert ref["steps"][2] == 1 and got["steps"][2] == 0
    if wrong == "peer_error_ignored":
        assert ref["steps"].sum() == 0 and got["steps"].sum() > 0
        assert DO.error_words(errors)[1] == [2, 2, 2, 2, 2, 1, 2, 2]


# ------------------------------------------------------------------------------------------------ construction
def _cpu_loader():
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(num_cameras=6, width=64, height=48)
    return DL(dataset=ds, device="cpu", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS,
              space_pruning_mode=DL.SpacePruningMode.AABB, batch_size=64, camera_numbers=tuple(range(6)),
              frame_numbers=tuple(ds.frames), max_buffer_size=2, render_sequence=[(2, 15), (4, 16)])


def test_world_size_mismatch_raises():
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.training import FusedTrainer

    poses = CameraPoses(_cpu_loader())
    assert poses.world_size == 1
    with pytest.raises(ValueError, match="world_size"):
        FusedTrainer(None, world_size=2, camera_poses=poses)
    with pytest.raises(ValueError, match="world_size"):
        CameraPoses(_cpu_loader(), world_size=9)


def _build_on_rank(rank, port, settings, q):
    import torch.distributed as dist

    from humanrf_b200.toolbox.camera_refinement import CameraPoses

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        poses = CameraPoses(_cpu_loader(), world_size=2, **settings[rank])
    except ValueError as e:
        q.put((rank, str(e)))
    else:
        # the trainer must exchange over the group the poses were checked in
        from humanrf_b200.training import FusedTrainer

        other = dist.new_group([0, 1])
        try:
            FusedTrainer(None, world_size=2, process_group=other, camera_poses=poses)
            q.put((rank, "FusedTrainer took camera_poses built over another process group"))
        except ValueError as e:
            q.put((rank, None if "process_group" in str(e) else str(e)))
    finally:
        dist.destroy_process_group()


def _run_two_ranks(settings, port_offset):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29100 + os.getpid() % 1000 + port_offset
    procs = [ctx.Process(target=_build_on_rank, args=(r, port, settings, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


@pytest.mark.parametrize("field,settings", [
    (None, [{}, {}]),
    ("lr", [{"lr": 2e-3}, {"lr": 1e-3}]),
    ("fixed_cameras", [{"fixed_cameras": (0,)}, {"fixed_cameras": (1,)}]),
    ("intrinsics", [{"intrinsics": True}, {}]),
])
def test_configuration_mismatch_raises_on_every_rank(field, settings):
    out = _run_two_ranks(settings, ["lr", "fixed_cameras", "intrinsics", None].index(field))
    if field is None:
        assert out == {0: None, 1: None}
    else:
        assert out[0] is not None and out[1] is not None, out
        assert field in out[0] and field in out[1], out
