"""Differential tests against the reference's first-party pure-Python pieces of the path, on randomized inputs.  What the
reference computes on these inputs is stored in tests/golden/reference_live.npz: tests/golden/make_reference_live_golden.py
imports a checkout of the reference and runs every `reference_*` function below (the only code here that touches the
reference); each test recomputes our side on the same inputs and compares.  They complement tests/golden/reference_host.npz
with many more cases."""
import dataclasses
import json
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch

GOLD = Path(__file__).resolve().parent / "golden" / "reference_live.npz"


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _json(gold, key):
    return json.loads(str(gold[key]))


def _surface(cls):
    fields = [[f.name, "MISSING" if f.default is dataclasses.MISSING else repr(f.default)] for f in dataclasses.fields(cls)]
    return [fields, sorted(m for m in dir(cls) if not m.startswith("_"))]


def reference_surfaces(ref):
    return {"surfaces": json.dumps({"InputBatch": _surface(ref.ib.InputBatch), "QueryInput": _surface(ref.qio.QueryInput),
                                    "QueryOutput": _surface(ref.qio.QueryOutput)})}


def test_dataclass_surfaces_match(gold):
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.scene_representation.query_io import QueryInput, QueryOutput

    theirs = _json(gold, "surfaces")
    assert _surface(InputBatch) == theirs["InputBatch"]
    assert _surface(QueryInput) == theirs["QueryInput"]
    assert _surface(QueryOutput) == theirs["QueryOutput"]


FIELDS = ["ray_origins", "ray_directions", "minmaxes", "rgba", "ray_masks", "frame_numbers", "unique_frame_numbers",
          "camera_numbers", "sample_distances", "ray_indices"]


def _batch(cls, rng, num_rays, masked):
    counts = rng.integers(0, 9, num_rays)
    ri = np.repeat(np.arange(num_rays), counts)
    mask = np.ones((num_rays + masked, 1), bool)
    mask[rng.permutation(num_rays + masked)[:masked]] = False
    fr = rng.integers(15, 40, (num_rays, 1)).astype(np.int32)
    t = torch.from_numpy
    return cls(ray_origins=t(rng.normal(size=(num_rays, 3)).astype(np.float32)),
               ray_directions=t(rng.normal(size=(num_rays, 3)).astype(np.float32)),
               minmaxes=t(rng.random((num_rays, 2)).astype(np.float32)), rgba=t(rng.random((num_rays, 4)).astype(np.float32)),
               ray_masks=t(mask), frame_numbers=t(fr), unique_frame_numbers=torch.unique(t(fr)).view(-1, 1),
               camera_numbers=t(rng.integers(0, 160, (num_rays, 1)).astype(np.int32)),
               sample_distances=t(rng.random((int(counts.sum()), 1)).astype(np.float32)), ray_indices=t(ri.astype(np.int64)),
               width=64, height=48)


def _merge_cases():
    """60 random configurations of merge_input_batches: (case, batch specs, seed)."""
    rng = np.random.default_rng(7)
    for case in range(60):
        nb = int(rng.integers(1, 5))
        specs = [(int(rng.integers(1, 30)), int(rng.integers(0, 5))) for _ in range(nb)]
        yield case, specs, int(rng.integers(0, 2 ** 31))


def _merged(cls, fn, case, specs, seed):
    r2 = np.random.default_rng(seed)
    batches = [_batch(cls, r2, *s) for s in specs]
    total = sum(b.sample_distances.shape[0] for b in batches)
    budget = [None, max(1, total // 2), max(1, total - 1), total, total + 5, 1][case % 6]
    return fn(batches, budget), budget, total


def reference_merge(ref):
    out = {}
    for case, specs, seed in _merge_cases():
        a, _, _ = _merged(ref.ib.InputBatch, ref.inp.merge_input_batches, case, specs, seed)
        for f in FIELDS:
            out[f"merge/{case}/{f}"] = getattr(a, f).numpy()
        out[f"merge/{case}/wh"] = np.array([a.width, a.height])
    return out


def test_merge_input_batches_randomized(gold):
    """input.py:10-55 incl. the sample-budget cut-off and its `cumsum < cutoff` behaviour, 60 random configurations."""
    from humanrf_b200.dataset.input_batch import InputBatch
    from humanrf_b200.input import merge_input_batches

    checked_cut = 0
    for case, specs, seed in _merge_cases():
        b, budget, total = _merged(InputBatch, merge_input_batches, case, specs, seed)
        if budget is not None and budget < total:
            checked_cut += 1
        for f in FIELDS:
            x, y = torch.from_numpy(gold[f"merge/{case}/{f}"]), getattr(b, f)
            if f == "unique_frame_numbers":
                x, y = torch.sort(x.reshape(-1))[0], torch.sort(y.reshape(-1))[0]
            assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y), (case, f)
        assert gold[f"merge/{case}/wh"].tolist() == [b.width, b.height]
    assert checked_cut >= 15


def _activation_inputs():
    g = torch.Generator().manual_seed(3)
    xs = [(torch.randn(513, generator=g) * scale, torch.randn(513, generator=g)) for scale in (1.0, 9.0, 30.0)]
    pred = torch.rand(777, 1, generator=g) * 1.6 - 0.3
    target = (torch.rand(777, 1, generator=g) > 0.4).float()
    return xs, pred, target


def _exp_and_grad(fn, x, dy):
    xi = x.clone().requires_grad_(True)
    y = fn(xi)
    y.backward(dy)
    return y.detach(), xi.grad


def reference_activation(ref):
    xs, pred, target = _activation_inputs()
    out = {"bce": ref.loss.bce_loss(pred, target).numpy()}
    for k, (x, dy) in enumerate(xs):
        y, gx = _exp_and_grad(ref.act.truncated_exp, x, dy)
        out[f"texp/{k}/y"], out[f"texp/{k}/grad"] = y.numpy(), gx.numpy()
    return out


def test_truncated_exp_and_bce_randomized(gold):
    from humanrf_b200.utils.activation import truncated_exp
    from humanrf_b200.utils.loss import bce_loss

    xs, pred, target = _activation_inputs()
    for k, (x, dy) in enumerate(xs):
        y, gx = _exp_and_grad(truncated_exp, x, dy)
        assert torch.equal(torch.from_numpy(gold[f"texp/{k}/y"]), y) and torch.equal(torch.from_numpy(gold[f"texp/{k}/grad"]), gx)
    assert torch.equal(torch.from_numpy(gold["bce"]), bce_loss(pred, target))


class _DS:
    def __init__(self, grids):
        self.grids = grids

    def get_occupancy_grid(self, frame_number):
        return self.grids[frame_number].copy()       # the reference ORs into the first grid of a cluster in place


def _partitioning_cases():
    rng = np.random.default_rng(11)
    for case in range(12):
        n = int(rng.integers(3, 140))
        base = rng.random((12, 12, 12)) < 0.2
        grids, cur = [], base.copy()
        for f in range(n):
            if rng.random() < [0.05, 0.3, 0.8][case % 3]:
                cur = cur | (rng.random(cur.shape) < 0.02)    # occasional growth of the occupied set
            if rng.random() < 0.03:
                cur = rng.random(cur.shape) < 0.2             # a jump
            grids.append((cur * 255).astype(np.uint8))
        yield case, grids, [1.05, 1.25, 2.0][case % 3]


def reference_partitioning(ref):
    import contextlib
    import io

    out = {"atp/predefined": json.dumps([type(ref.atp.PREDEFINED_SEGMENT_SIZES).__name__, list(ref.atp.PREDEFINED_SEGMENT_SIZES)]),
           "atp/size": json.dumps([ref.atp.get_segment_size(n) for n in range(1, 260)]),
           "atp/final": json.dumps([ref.atp.get_final_segment_size(n) for n in range(1, 260)])}
    for case, grids, thr in _partitioning_cases():
        with contextlib.redirect_stderr(io.StringIO()):      # tqdm bar
            want = ref.atp.compute_adaptive_segment_sizes(_DS(grids), list(range(len(grids))), thr)
        out[f"atp/want/{case}"] = json.dumps(want, default=int)
    return out


def test_segment_size_rules_and_partitioning_randomized(gold):
    """adaptive_temporal_partitioning.py:28-107 against the oracle restatement (the GPU implementation is compared with
    the same reference decisions through tests/golden/partitioning.npz)."""
    from humanrf_b200 import adaptive_temporal_partitioning as ours
    from oracle import occupancy_tools as O

    kind, sizes = _json(gold, "atp/predefined")
    for x in (ours.PREDEFINED_SEGMENT_SIZES, O.PREDEFINED_SEGMENT_SIZES):
        assert type(x).__name__ == kind and list(x) == sizes
    size, final = _json(gold, "atp/size"), _json(gold, "atp/final")
    for n in range(1, 260):
        assert ours.get_segment_size(n) == size[n - 1] == O.get_segment_size(n)
        assert ours.get_final_segment_size(n) == final[n - 1] == O.get_final_segment_size(n)
    for case, grids, thr in _partitioning_cases():
        assert json.loads(json.dumps(O.compute_adaptive_segment_sizes(grids, thr), default=int)) == _json(gold, f"atp/want/{case}"), case


_MODEL_CACHE = {}


def _import_reference_model():
    """The reference's HumanRF with `tinycudann` and its compiled extension stubbed out: the stubs only RECORD the
    configs they are constructed with and own one flat `.params` (sized by our layout rule -- sizes of tcnn tensors are
    therefore not evidence, the configs / names / first-party tensors are)."""
    from humanrf_b200.scene_representation.grid_layout import GridLayout, MLP_SIGMA_PARAMS, mlp_color_params

    if _MODEL_CACHE:                       # the module stays bound to the stub classes (and their log) of its first import
        _MODEL_CACHE["calls"].clear()
        sys.modules["tinycudann"] = _MODEL_CACHE["tcnn"]
        sys.modules["humanrf.scene_representation.humanrf"] = _MODEL_CACHE["module"]
        return _MODEL_CACHE["module"], _MODEL_CACHE["calls"]
    calls = []

    class _Flat(torch.nn.Module):
        def __init__(self, n):
            super().__init__()
            self.params = torch.nn.Parameter(torch.zeros(n))

    class Encoding(_Flat):
        def __init__(self, n_input_dims, encoding_config, **kw):
            calls.append(("Encoding", n_input_dims, dict(encoding_config)))
            c = encoding_config
            fin = c["base_resolution"] * c["per_level_scale"] ** (c["n_levels"] - 1)
            super().__init__(GridLayout(c["log2_hashmap_size"], c["n_levels"], c["base_resolution"], int(round(fin))).n_params)

    class Network(_Flat):
        def __init__(self, n_input_dims, n_output_dims, network_config, **kw):
            calls.append(("Network", n_input_dims, n_output_dims, dict(network_config)))
            super().__init__(MLP_SIGMA_PARAMS)

    class NetworkWithInputEncoding(_Flat):
        def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, **kw):
            calls.append(("NetworkWithInputEncoding", n_input_dims, n_output_dims, dict(encoding_config), dict(network_config)))
            super().__init__(mlp_color_params(n_input_dims - 18))

    tcnn = types.ModuleType("tinycudann")
    tcnn.Encoding, tcnn.Network, tcnn.NetworkWithInputEncoding = Encoding, Network, NetworkWithInputEncoding
    sys.modules["tinycudann"] = tcnn
    sys.modules["humanrf.scene_representation.tensor_composition_native"] = types.ModuleType("tensor_composition_native")
    import humanrf.scene_representation.humanrf as ref_model

    _MODEL_CACHE.update(module=ref_model, calls=calls, tcnn=tcnn)
    return ref_model, calls


MODEL_CASES = [((50,), 15, 50, 0), ((25, 12, 100, 6), 0, 140, 2), ((6, 6), 3, 9, 0)]


def _model_kw(cam_emb):
    from humanrf_b200.synthetic import MODEL_KW

    return {**MODEL_KW, "camera_embedding_dim": cam_emb, "temporal_partitioning": "adaptive", "fixed_segment_size": 6}


def _model_record(m):
    return {"f2s": m.frame_numbers_to_segment_numbers.numpy(), "f2t": m.frame_numbers_to_normalized_local_frame_numbers.numpy(),
            "scalars": json.dumps([m.num_frames, m.num_segments, m.total_feature_dim, m.density_scale]),
            "state": json.dumps([[k, list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()]),
            "groups": json.dumps([[len(list(g["params"])), g["lr"]] for g in m.get_params(1e-2)])}


def reference_model(ref):
    out = {}
    for idx, (segment_sizes, first, count, cam_emb) in enumerate(MODEL_CASES):
        try:
            ref_model, calls = _import_reference_model()
            theirs = ref_model.HumanRF(sorted_frame_numbers=tuple(range(first, first + count)), segment_sizes=segment_sizes,
                                       **_model_kw(cam_emb))
        finally:
            sys.modules.pop("tinycudann", None)
        out.update({f"model/{idx}/{k}": v for k, v in _model_record(theirs).items()})
        out[f"model/{idx}/calls"] = json.dumps(calls)
    return out


@pytest.mark.parametrize("segment_sizes,first,count,cam_emb", MODEL_CASES)
def test_model_constructor_against_the_reference(gold, segment_sizes, first, count, cam_emb):
    """humanrf.py:68-156 + decomposition4d.py:73-122 run for real (only tcnn is a recording stub): frame LUTs, per-segment
    hash-map sizes, encoding / network configs, state-dict key names and the shapes of the first-party tensors."""
    from humanrf_b200.scene_representation.grid_layout import GridLayout
    from humanrf_b200.scene_representation.humanrf import HumanRF

    idx = MODEL_CASES.index((segment_sizes, first, count, cam_emb))     # the key of this case in the stored outputs
    ours = HumanRF(sorted_frame_numbers=tuple(range(first, first + count)), segment_sizes=segment_sizes, **_model_kw(cam_emb))
    mine = _model_record(ours)
    # frame -> segment / local-time look-up tables
    for k in ("f2s", "f2t"):
        theirs = gold[f"model/{idx}/{k}"]
        assert mine[k].dtype == theirs.dtype and np.array_equal(mine[k], theirs), k
    assert json.loads(mine["scalars"]) == _json(gold, f"model/{idx}/scalars")
    # what the reference asks tcnn for, segment by segment
    calls = _json(gold, f"model/{idx}/calls")
    enc = [c for c in calls if c[0] == "Encoding"]
    assert len(enc) == 4 * len(segment_sizes)
    for s, fg in enumerate(ours.feature_grids):
        for c in enc[4 * s:4 * s + 4]:
            cfg = c[2]
            assert c[1] == 3 and cfg["otype"] == "HashGrid" and cfg["n_levels"] == 16 and cfg["n_features_per_level"] == 2
            assert cfg["log2_hashmap_size"] == fg.layout.log2_hashmap_size
            assert cfg["base_resolution"] == 32 and np.float32(cfg["per_level_scale"]) == np.float32(np.exp(np.log(2048 / 32) / 15))
            assert GridLayout(cfg["log2_hashmap_size"]).n_params == fg.layout.n_params
    net = [c for c in calls if c[0] == "Network"][0]
    assert net[1:3] == [32, 16] and net[3] == {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None",
                                              "n_neurons": 64, "n_hidden_layers": 1}
    col = [c for c in calls if c[0] == "NetworkWithInputEncoding"][0]
    assert col[1:3] == [18 + cam_emb, 3] and col[4]["output_activation"] == "Sigmoid" and col[4]["n_hidden_layers"] == 2
    assert col[3]["nested"][0] == {"n_dims_to_encode": 3, "otype": "SphericalHarmonics", "degree": 4}
    # state dict: same keys in the same order, same shapes and dtypes (first-party tensors: vectors, LUT buffers, embeddings)
    assert json.loads(mine["state"]) == _json(gold, f"model/{idx}/state")
    # optimiser parameter groups (humanrf.py:210-220)
    assert json.loads(mine["groups"]) == _json(gold, f"model/{idx}/groups")


def _scene_density(positions, frame_numbers):
    r2 = (positions ** 2).sum(1)
    return 2500.0 * torch.exp(-60.0 * r2) * (1.0 + 0.25 * (frame_numbers.reshape(-1) % 3).float())


def _scene_radiance(positions, directions):
    return torch.sigmoid(3.0 * positions + directions)


def _render_inputs():
    from helpers import synthetic_rays

    b = synthetic_rays(64, 40, tuple(range(15, 27)), ragged=True, seed=8)
    bg = torch.rand(64, 3, generator=torch.Generator().manual_seed(1))
    parts = [(torch.rand(n, 3, generator=torch.Generator().manual_seed(n)), torch.rand(n, 1, generator=torch.Generator().manual_seed(9 + n)))
             for n in (3, 0, 5)]
    return b, bg, parts


def reference_render(ref):
    """The reference's own prune_samples / render / merge_render_outputs (volume_rendering.py:26-150) on the CPU, with
    `nerfacc` replaced by the oracle's restatement of its three functions and a closed-form scene representation."""
    from oracle import rendering as R

    nerfacc = types.ModuleType("nerfacc")
    nerfacc.render_visibility = lambda alphas, ray_indices, early_stop_eps, alpha_thre, n_rays: \
        R.render_visibility(alphas, ray_indices, early_stop_eps, alpha_thre)

    def render_weight_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays):
        sdt = sigmas.reshape(-1) * (t_ends - t_starts).reshape(-1)
        return (torch.exp(-R._exclusive_by_ray(sdt, ray_indices, "sum")) * (1.0 - torch.exp(-sdt))).unsqueeze(-1)

    nerfacc.render_weight_from_density = render_weight_from_density
    nerfacc.accumulate_along_rays = lambda weights, ray_indices, values=None, n_rays=None: R.accumulate(weights, ray_indices, values, n_rays)
    try:
        _import_reference_model()
        sys.modules["nerfacc"] = nerfacc
        import humanrf.volume_rendering as vr
    finally:
        sys.modules.pop("tinycudann", None)
        sys.modules.pop("nerfacc", None)
    QueryOutput = ref.qio.QueryOutput

    class Scene:
        def density(self, q):
            return QueryOutput(density=_scene_density(q.positions, q.frame_numbers))

        def __call__(self, q):
            return QueryOutput(density=self.density(q).density, radiance=_scene_radiance(q.positions, q.directions))

    b, bg, parts = _render_inputs()
    o, d, fr, ri = b["o"], b["d"], b["frames"].view(-1, 1), b["ri"]
    out = {}
    for is_training in (False, True):
        ib = ref.ib.InputBatch(ray_origins=o, ray_directions=d, frame_numbers=fr, unique_frame_numbers=torch.unique(fr).view(-1, 1),
                               camera_numbers=torch.zeros_like(fr), sample_distances=b["t"].clone().view(-1, 1),
                               ray_indices=ri.clone(), rgba=b["rgba"], width=8, height=8)
        torch.manual_seed(5)
        vr.prune_samples(ib, Scene(), is_training=is_training)
        r = vr.render(ib, Scene(), bg, is_training=is_training)
        nobg = vr.render(ib, Scene(), None, is_training=is_training)
        out.update({f"render/{is_training}/t": ib.sample_distances.numpy(), f"render/{is_training}/ri": ib.ray_indices.numpy(),
                    f"render/{is_training}/color": r.color.numpy(), f"render/{is_training}/wsum": r.weights_sum.numpy(),
                    f"render/{is_training}/color_nobg": nobg.color.numpy()})
    merged = vr.RenderOutput.merge_render_outputs([vr.RenderOutput(color=c, weights_sum=w) for c, w in parts])
    out["render/merged_color"], out["render/merged_wsum"] = merged.color.numpy(), merged.weights_sum.numpy()
    try:
        vr.RenderOutput.merge_render_outputs([vr.RenderOutput(color=torch.rand(2, 3))])
    except RuntimeError as e:
        out["render/merge_error"] = str(e)
    return out


def test_prune_and_render_glue_against_the_reference(gold):
    """Pins everything the oracle restates AROUND nerfacc (positions, jitter, alpha, t_ends = t + step, mask application,
    background blend, output shapes) against the reference's own glue.  nerfacc's own arithmetic stays unpinned."""
    from humanrf_b200.volume_rendering import RenderOutput as OurRenderOutput
    from oracle import rendering as R

    b, bg, parts = _render_inputs()
    o, d, fr, ri = b["o"], b["d"], b["frames"].view(-1, 1), b["ri"]
    for is_training in (False, True):
        g = {k: torch.from_numpy(gold[f"render/{is_training}/{k}"]) for k in ("t", "ri", "color", "wsum", "color_nobg")}
        torch.manual_seed(5)
        t = b["t"].view(-1, 1) + (torch.rand_like(b["t"].view(-1, 1)) * R.STEP if is_training else 0)
        keep = R.prune_mask(_scene_density(o[ri] + t * d[ri], fr[ri]), ri)
        assert 0 < int(keep.sum()) < keep.numel()
        assert torch.equal(g["t"], t[keep]) and torch.equal(g["ri"], ri[keep])
        assert g["t"].shape == (int(keep.sum()), 1)
        tk, rk = t[keep], ri[keep]
        pk = o[rk] + tk * d[rk]
        sigma, rgb = _scene_density(pk, fr[rk]), _scene_radiance(pk, d[rk])
        col, ws = R.render(tk, sigma, rgb, rk, 64, bg)
        assert torch.equal(g["color"], col) and torch.equal(g["wsum"], ws)
        assert g["color"].shape == (64, 3) and g["wsum"].shape == (64, 1)
        assert torch.equal(g["color_nobg"], R.render(tk, sigma, rgb, rk, 64, None)[0])
    # merge_render_outputs: same concatenation, same error for a field that is not a tensor
    c = OurRenderOutput.merge_render_outputs([OurRenderOutput(color=cc, weights_sum=w) for cc, w in parts])
    assert torch.equal(torch.from_numpy(gold["render/merged_color"]), c.color)
    assert torch.equal(torch.from_numpy(gold["render/merged_wsum"]), c.weights_sum)
    assert "Unknown data type" in str(gold["render/merge_error"])
    with pytest.raises(RuntimeError, match="Unknown data type"):
        OurRenderOutput.merge_render_outputs([OurRenderOutput(color=torch.rand(2, 3))])


SCENE_SIZES, SCENE_E = (6, 12, 6), 2


def _scene_inputs():
    from helpers import positions_of, synthetic_rays
    from oracle import field as OF

    frames = tuple(range(15, 15 + sum(SCENE_SIZES)))
    om = OF.make_model(SCENE_SIZES, frames, seed=5, table_init="trained", bf16=False, table_std=0.5, camera_embedding_dim=SCENE_E)
    b = synthetic_rays(96, 24, frames, ragged=True, seed=12, n_distinct_frames=len(frames))
    return frames, om, b, positions_of(b)


def reference_scene(ref):
    """The reference's HumanRF.density / forward and Decomposition4D.forward (humanrf.py:158-208, decomposition4d.py:124-135)
    with every tcnn module and the composition extension answering through the ORACLE's restatement of that one module."""
    from humanrf_b200.synthetic import MODEL_KW
    from oracle import field as OF
    from oracle import hashgrid

    frames, om, b, pos = _scene_inputs()
    try:
        ref_model, _ = _import_reference_model()
        theirs = ref_model.HumanRF(sorted_frame_numbers=frames, segment_sizes=SCENE_SIZES, **{**MODEL_KW, "camera_embedding_dim": SCENE_E})
    finally:
        sys.modules.pop("tinycudann", None)
    import humanrf.scene_representation.decomposition4d as d4

    d4.Decomposition4D.to = lambda self, *a, **k: self                       # the reference parks idle segments on the CPU
    d4.tensor_composition_native.compose_tensors_forward = \
        lambda xyz, xyt, yzt, xzt, vectors, coords: OF.compose(xyz.float(), xyt.float(), yzt.float(), xzt.float(), vectors, coords).half()
    for s, fg in enumerate(theirs.feature_grids):
        with torch.no_grad():
            fg.vectors.copy_(om.segments[s].vectors)
        for k, name in enumerate(("xyz_encoding", "xyt_encoding", "yzt_encoding", "xzt_encoding")):
            enc = getattr(fg, name)
            enc.forward = (lambda x, s=s, k=k: hashgrid.encode(om.segments[s].grids[k], x.float(), om.segments[s].log2T).half())
    theirs.sigma_net.forward = lambda f: torch.relu(f.float() @ om.w_sigma[0].t()) @ om.w_sigma[1].t()

    def color_net(x):                                                        # [ (d+1)/2 | geo 15 | embedding E ] -> rgb
        d, rest = x[:, :3].float() * 2 - 1, x[:, 3:].float()
        inp = torch.cat((OF.sh4(d), rest, torch.ones((x.shape[0], 48 - 16 - rest.shape[1]))), dim=1)
        w1, w2, w3 = om.w_color
        h = torch.relu(torch.relu(inp @ w1.t()) @ w2.t())
        return torch.sigmoid((h @ w3.t())[:, :3])

    theirs.color_net.forward = color_net
    with torch.no_grad():
        theirs.camera_embeddings.weight.copy_(om.camera_embeddings)
    ri = b["ri"]
    dirs, fr, cams = b["d"][ri], b["frames"][ri].view(-1, 1), b["cams"][ri].view(-1, 1)
    out = {}
    for is_training in (True, False):
        q = ref.qio.QueryInput(is_training=is_training, positions=pos, directions=dirs, frame_numbers=fr,
                               unique_frame_numbers=torch.unique(b["frames"]).view(-1, 1), camera_numbers=cams)
        with torch.no_grad():
            r, dens = theirs(q), theirs.density(q)
        out.update({f"scene/{is_training}/density": r.density.numpy(), f"scene/{is_training}/density_only": dens.density.numpy(),
                    f"scene/{is_training}/geo": r.geometry_features.numpy(), f"scene/{is_training}/radiance": r.radiance.numpy()})
    return out


def test_scene_representation_glue_against_the_reference(gold):
    """What is compared is the glue the oracle restates around tcnn / the composition extension: frame -> segment routing,
    the +0.5 shift, local time, grid axis selection (xyz, xyt, yzt, xzt), composition call, truncated_exp * density_scale,
    geometry-feature slicing, (d+1)/2, camera embeddings while training / zeros otherwise.  The reference stores the
    composed features in fp16, hence the tolerances."""
    frames, om, b, pos = _scene_inputs()
    ri = b["ri"]
    dirs, fr, cams = b["d"][ri], b["frames"][ri].view(-1, 1), b["cams"][ri].view(-1, 1)
    touched = set(om.f2s[b["frames"].numpy()].tolist())
    assert len(touched) == 3                                                 # all three segments are exercised
    for is_training in (True, False):
        g = {k: torch.from_numpy(gold[f"scene/{is_training}/{k}"]) for k in ("density", "density_only", "geo", "radiance")}
        with torch.no_grad():
            sigma, geo, rgb = om.forward(pos, dirs, fr.view(-1), cams.view(-1) if is_training else None)
        assert g["density"].shape == sigma.shape and g["geo"].shape == (pos.shape[0], 15) and g["radiance"].shape == rgb.shape
        assert torch.equal(g["density"], g["density_only"])
        rel = ((g["density"] - sigma).abs() / sigma.abs().clamp_min(1e-3)).max().item()
        dg = (g["geo"].float() - geo).abs().max().item()
        dc = (g["radiance"] - rgb).abs().max().item()
        print(f"is_training={is_training}: density rel {rel:.2e}, geometry abs {dg:.2e}, radiance abs {dc:.2e}")
        assert rel < 2e-3 and dg < 2e-3 and dc < 1e-3       # measured 5e-5 / 5e-5 / 5e-6 (the fp16 feature buffer)
    # the embedding really is dropped at evaluation: the two passes differ in radiance only
    assert (torch.from_numpy(gold["scene/False/radiance"]) - torch.from_numpy(gold["scene/True/radiance"])).abs().max() > 1e-3
