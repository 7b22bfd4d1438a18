"""Camera colour responses in data-parallel training, simulated on one GPU: hrf_camera_response_step_ranks at world sizes
1-8 with every rank's gradient record in device memory, against tests/response_oracle.py's ranked step (float64 sum in
rank order / W, the union of the touched cameras, the error words).  The replicas must stay bit-identical, W = 1 must
equal hrf_camera_response_step bit for bit, the rank order must matter, and a bad camera number on one rank must stop
every rank.  FusedTrainer with camera_responses at world 2 runs on two GPUs (NCCL, skipped with fewer), and on one GPU
as two processes sharing it over a gloo group, so the trainer's exchange of the response record runs either way.
Parameters and moments are held to 1e-12 relative of the oracle (the kernel's float64 Adam rounds in another
order than numpy's; where steps or moments cancel, to 1e-12 of one step or of the largest gradient), the tables within 1 fp32 ulp of the oracle's (CUDA's and numpy's expm1 may differ in the last
float64 bit)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import response_oracle as RO

pytestmark = pytest.mark.gpu


def _world(cuda, C_, W, fixed=(0,)):
    from humanrf_b200.toolbox.camera_response import CameraResponses

    out = []
    for r in range(W):
        ld = SimpleNamespace(all_inverse_krs=torch.zeros((C_, 3, 3), device=cuda), camera_numbers=tuple(range(C_)))
        p = CameraResponses(ld, lr=4e-3, final_lr_ratio=1.0, fixed_cameras=fixed)
        p.world_size, p.rank = W, r           # a simulated rank of a W-rank group on this device
        out.append(p)
    return out


def _fill(world, rng):
    C_ = world[0].num_cameras
    grads, counts = [], []
    for p in world:
        g = (rng.standard_normal((C_, 6)) * 10.0 ** rng.uniform(-6, -1, (C_, 1))).astype(np.float32)
        n = np.where(rng.uniform(0, 1, C_) < 0.4, 0, rng.integers(1, 500, C_)).astype(np.int32)
        g[n == 0] = 0.0
        p.response_grad.copy_(torch.from_numpy(g))
        p.ray_count.copy_(torch.from_numpy(n))
        grads.append(g)
        counts.append(n)
    return grads, counts


def _snapshot(p):
    return {n: getattr(p, n).clone() for n in ("params", "exp_avg", "exp_avg_sq", "steps", "table", "error")}


def _same(a, b):
    return [n for n in a if not torch.equal(a[n], b[n])]


@pytest.mark.parametrize("C_", [1, 160, 1024])
@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_step_ranks_against_oracle(cuda, W, C_):
    rng = np.random.default_rng(W * 1000 + C_)
    world = _world(cuda, C_, W)
    st = {"params": np.zeros((C_, 6)), "m": np.zeros((C_, 6)), "v": np.zeros((C_, 6)), "steps": np.zeros(C_, np.int64)}
    fixed = np.zeros(C_, bool)
    fixed[0] = True
    for k in range(4):
        grads, counts = _fill(world, rng)
        addrs = [p.record.data_ptr() for p in world]
        for p in world:
            p.step(k, addrs)
        torch.cuda.synchronize()
        RO.ranked_step(st, grads, counts, [0] * W, fixed, 4e-3)
    p0 = _snapshot(world[0])
    for p in world[1:]:
        assert _same(p0, _snapshot(p)) == []                                 # replicas bit-identical
    got = world[0].params.cpu().numpy()
    assert np.allclose(got, st["params"], rtol=1e-12, atol=1e-12 * 4e-3)     # 1e-12 of one step where steps cancel
    # the moments where they cancel: 1e-12 of the largest gradient (0.1 here) and of its square
    assert np.allclose(world[0].exp_avg.cpu().numpy(), st["m"], rtol=1e-12, atol=1e-13)
    assert np.allclose(world[0].exp_avg_sq.cpu().numpy(), st["v"], rtol=1e-12, atol=1e-14)
    assert np.array_equal(world[0].steps.cpu().numpy(), st["steps"])
    want = RO.table_of(got)
    assert (np.abs(world[0].table.cpu().numpy().astype(np.float64) - want) <= np.spacing(np.abs(want))).all()
    assert (world[0].table[0] == 0).all() and int(world[0].steps[0]) == 0
    if C_ > 1:
        assert int(world[0].steps.max()) > 0


@pytest.mark.parametrize("C_", [8, 1024])
def test_one_rank_equals_single_rank_step_bit_for_bit(cuda, C_):
    rng = np.random.default_rng(C_)
    (a,), (b,) = _world(cuda, C_, 1), _world(cuda, C_, 1)
    for k in range(3):
        grads, counts = _fill([a], rng)
        b.response_grad.copy_(a.response_grad)
        b.ray_count.copy_(a.ray_count)
        a.step(k, [a.record.data_ptr()])
        b.step(k)
    torch.cuda.synchronize()
    assert _same(_snapshot(a), _snapshot(b)) == []
    assert int(a.steps.sum()) > 0


def test_reversed_rank_order_changes_the_step(cuda):
    """Records (1e20, -1e20, 3) sum to 3 in rank order and to 0 with rank 2 first (3 is lost in 1e20 in float64)."""
    world = _world(cuda, 4, 3)
    for p, v in zip(world, (1e20, -1e20, 3.0)):
        p.ray_count.fill_(1)
        p.response_grad.zero_()
        p.response_grad[1, 3] = v
    addrs = [p.record.data_ptr() for p in world]
    world[0].step(0, addrs)
    world[1].step(0, [addrs[2], addrs[0], addrs[1]])
    torch.cuda.synchronize()
    assert float(world[0].exp_avg[1, 3]) > 0 and float(world[1].exp_avg[1, 3]) == 0
    assert float(world[0].params[1, 3]) < 0 and float(world[1].params[1, 3]) == 0


def test_bad_camera_on_one_rank_stops_every_rank(cuda):
    W, C_, R = 3, 6, 500
    world = _world(cuda, C_, W)
    rng = np.random.default_rng(0)
    _fill(world, rng)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)   # noqa: E731
    cams = rng.integers(0, C_, R).astype(np.int32)
    cams[17] = C_                                                  # rank 1's batch holds a bad camera number
    f = lambda *s: dev(rng.uniform(0, 1, s).astype(np.float32))   # noqa: E731
    dc, dw, loss = torch.empty((R, 3), device=cuda), torch.empty(R, device=cuda), torch.zeros(1, device=cuda)
    world[1].loss(f(R, 3), f(R), f(R, 4), f(R, 3), dev(cams), R, 0.01, 1e-3, None, dc, dw, loss)
    before = [_snapshot(p) for p in world]
    addrs = [p.record.data_ptr() for p in world]
    for p in world:
        p.step(0, addrs)
    torch.cuda.synchronize()
    assert [int(p.error[0]) for p in world] == [2, 1, 2]
    for r, p in enumerate(world):
        changed = _same(before[r], _snapshot(p))
        assert changed == (["error"] if r != 1 else []), (r, changed)
        with pytest.raises(RuntimeError, match="outside"):
            p.check()


# ------------------------------------------------------------------------------------------------ FusedTrainer, 2 ranks
def _train_rank(rank, world, port, spans, q, exchange, with_poses, plan_bad, shared, steps=3):
    """One rank of FusedTrainer(camera_responses=...) on its share of a 512-ray batch.  `shared`: both ranks on
    cuda:0 over a gloo group (the peer buffers are then CUDA IPC mappings on the same device); otherwise rank r on
    cuda:r over NCCL."""
    import torch.distributed as dist

    from humanrf_b200.synthetic import make_model, synthetic_rays
    from humanrf_b200.toolbox.camera_refinement import CameraPoses
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.training import FusedTrainer
    from test_camera_poses_dp_gpu import _world_loaders
    from test_dp_gpu import _subset

    dev = torch.device("cuda", 0 if shared else rank)
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        if shared:
            dist.init_process_group("gloo", rank=rank, world_size=world)
        else:
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    model, frames = make_model((6,), table_std=0.5, device=dev)
    b = synthetic_rays(512, 48, frames, seed=4, ragged=True)
    bg_all = torch.rand(512, 3, generator=torch.Generator().manual_seed(9))
    cams_all = (torch.arange(512, dtype=torch.int32) * 7) % 5
    (ld,) = _world_loaders(dev, 5, 1, 6)
    poses = CameraPoses(ld, lr=1e-3, final_lr_ratio=1.0, world_size=world) if with_poses else None
    resp = CameraResponses(ld, lr=1e-2, final_lr_ratio=1.0, world_size=world)
    tr = FusedTrainer(model, lr=1e-2, prune=False, world_size=world, exchange=exchange, camera_poses=poses,
                      camera_responses=resp)
    lo, hi = spans[rank]
    first = None
    for step in range(steps):
        sb = {k: v.to(dev).contiguous() for k, v in _subset(b, lo, hi).items()}
        cams = cams_all[lo:hi].clone()
        if plan_bad and rank == 1:
            cams[3] = 99
        tr.step(sb["o"], sb["d"], sb["frames"], sb["t"], sb["ri"], sb["rgba"], hi - lo, background=bg_all[lo:hi].to(dev),
                cameras=cams.to(dev))
        if step == 0:
            torch.cuda.synchronize()
            first = resp.params.cpu().numpy().copy()
    tr.gather_master_parameters()
    torch.cuda.synchronize()
    err = None
    try:
        state = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in resp.state_dict().items()}
        state["table"] = resp.table.cpu().numpy()
        if with_poses:
            state["omega"], state["tau"] = poses.omega.cpu().numpy(), poses.tau.cpu().numpy()
    except RuntimeError as e:
        state, err = None, str(e)
    q.put((rank, [p.detach().cpu().numpy() for p in model.hot_parameters()], state, first, err))
    if world > 1:
        dist.barrier()
        tr.close()
        dist.destroy_process_group()


def _spawn(world, spans, exchange, with_poses, plan_bad, shared, port_offset):
    import torch.multiprocessing as mp
    from test_dp_gpu import _collect

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + os.getpid() % 50 + 2 * port_offset
    procs = [ctx.Process(target=_train_rank, args=(r, world, port, spans, q, exchange, with_poses, plan_bad, shared))
             for r in range(world)]
    for p in procs:
        p.start()
    got = {r: rest for r, *rest in _collect(q, procs, world)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return got


_RESPONSE_STATE = ("params", "exp_avg", "exp_avg_sq", "steps", "table")


def _check_two_ranks(ref, got, with_poses):
    """Replicas bit-identical (field, responses, poses); field and responses against the one-rank union batch: the field
    within test_dp_gpu's bar, the responses within 1e-3 of the distance they moved (the share's loss_scale 2 R_r / R
    rounds the field's bf16 backward differently from the union batch, and the responses see that field)."""
    (f0, s0, first0, e0), (f1, s1, first1, e1) = got[0], got[1]
    assert e0 is None and e1 is None, (e0, e1)
    for k in _RESPONSE_STATE + (("omega", "tau") if with_poses else ()):
        assert np.array_equal(np.asarray(s0[k]), np.asarray(s1[k])), k
    assert np.array_equal(first0, first1)
    assert all(np.array_equal(a, b) for a, b in zip(f0, f1))
    for a, b in zip(f0, ref[0]):
        assert np.linalg.norm(a - b) <= 1e-4 * max(np.linalg.norm(b), 1e-12) + 1e-6
    moved = np.linalg.norm(ref[1]["params"])
    assert moved > 0 and np.linalg.norm(s0["params"] - ref[1]["params"]) <= 1e-3 * moved
    assert np.array_equal(np.asarray(s0["steps"]), np.asarray(ref[1]["steps"]))
    return first0


SPANS = [(0, 200), (200, 512)]


@pytest.mark.parametrize("with_poses", [False, True], ids=["responses", "responses+poses"])
def test_two_rank_training_with_camera_responses(cuda, with_poses):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ref = _spawn(1, [(0, 512)], "nccl", with_poses, False, False, 0)[0]
    firsts = {ex: _check_two_ranks(ref, _spawn(2, SPANS, ex, with_poses, False, False, 1 + i + 2 * with_poses), with_poses)
              for i, ex in enumerate(("nccl", "p2p"))}
    assert np.array_equal(firsts["nccl"], firsts["p2p"])


@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_two_rank_bad_camera_stops_both_ranks(cuda, exchange):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = _spawn(2, SPANS, exchange, False, True, False, 6 + ["nccl", "p2p"].index(exchange))
    assert got[0][3] is not None and "another rank" in got[0][3]
    assert got[1][3] is not None and "outside" in got[1][3]


@pytest.mark.parametrize("with_poses", [False, True], ids=["responses", "responses+poses"])
@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_two_ranks_sharing_one_gpu(cuda, exchange, with_poses):
    """The same two-rank run with both ranks on one GPU over a gloo group: the exchange of the response (and pose)
    record, the ranked steps, the replica checks and close() run on a one-GPU machine too."""
    ref = _spawn(1, [(0, 512)], exchange, with_poses, False, True, 8)[0]
    _check_two_ranks(ref, _spawn(2, SPANS, exchange, with_poses, False, True, 9 + 2 * (exchange == "p2p") + with_poses),
                     with_poses)


def test_two_ranks_sharing_one_gpu_bad_camera(cuda):
    got = _spawn(2, SPANS, "p2p", False, True, True, 14)
    assert got[0][3] is not None and "another rank" in got[0][3]
    assert got[1][3] is not None and "outside" in got[1][3]
