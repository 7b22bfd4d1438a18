"""CameraResponses in data-parallel training, without a GPU: the construction's collective check in a 2-process gloo group
(every rank must have the same cameras, fixed cameras and settings, or every rank raises ValueError naming the field),
and FusedTrainer's checks of the responses' world size and process group."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _cpu_loader(seed=0):
    rng = np.random.default_rng(seed)
    return SimpleNamespace(all_inverse_krs=torch.from_numpy(rng.standard_normal((6, 3, 3)).astype(np.float32)),
                           camera_numbers=tuple(range(6)))


def test_world_size_mismatch_raises():
    from humanrf_b200.toolbox.camera_response import CameraResponses
    from humanrf_b200.training import FusedTrainer

    resp = CameraResponses(_cpu_loader())
    assert resp.world_size == 1
    with pytest.raises(ValueError, match="world_size"):
        FusedTrainer(None, world_size=2, camera_responses=resp)
    with pytest.raises(ValueError, match="world_size"):
        CameraResponses(_cpu_loader(), world_size=9)


def _build_on_rank(rank, port, settings, q):
    import torch.distributed as dist

    from humanrf_b200.toolbox.camera_response import CameraResponses

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    s = dict(settings[rank])
    seed = s.pop("loader_seed", 0)
    try:
        resp = CameraResponses(_cpu_loader(seed), world_size=2, **s)
    except ValueError as e:
        q.put((rank, str(e)))
    else:
        from humanrf_b200.training import FusedTrainer

        other = dist.new_group([0, 1])
        try:
            FusedTrainer(None, world_size=2, process_group=other, camera_responses=resp)
            q.put((rank, "FusedTrainer took camera_responses built over another process group"))
        except ValueError as e:
            q.put((rank, None if "process_group" in str(e) else str(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("field,settings", [
    (None, [{}, {}]),
    ("lr", [{"lr": 2e-3}, {"lr": 1e-3}]),
    ("fixed_cameras", [{"fixed_cameras": (0,)}, {"fixed_cameras": (1,)}]),
    ("cameras", [{}, {"loader_seed": 1}]),
])
def test_configuration_mismatch_raises_on_every_rank(field, settings):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29300 + os.getpid() % 500 + ["lr", "fixed_cameras", "cameras", None].index(field)
    procs = [ctx.Process(target=_build_on_rank, args=(r, port, settings, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    if field is None:
        assert out == {0: None, 1: None}
    else:
        assert out[0] is not None and out[1] is not None, out
        assert f"in {field}:" in out[0] and f"in {field}:" in out[1], out
