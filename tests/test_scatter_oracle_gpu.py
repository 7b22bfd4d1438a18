"""The table / vector gradient scatter (hrf_field_backward_tables, HRF_SCATTER = 6 and 5) against the rounding-aware
float64 reference tests/scatter_oracle.py, entry by entry: every table and vector entry, touched or not, must lie within
its own error bound, and an entry no sample touches must still hold, bit for bit, what the buffer held before the launch
(a random fp32 base pattern in a third of the entries, +0 elsewhere).

Inputs (tests/scatter_cases.py; the CPU tests rebuild sets B-E from the same seeds and show that every mutant of
scatter_oracle.MUTANTS exceeds twice the bound on them):
  A  train-like: ragged synthetic rays on segments (100, 100, 50), ~250k samples, a device live count below the
     capacity and not a multiple of 8, NaN d(features) past it;
  B  edges, C  collisions, D  segments, E  live counts 0 / 1 / 1023 / 1025 / capacity (device scalar), on segments of 6
     frames.
Paths: both generations; egrid read through a survivor index (a column stride wider than n), egrid with identity
columns, the re-gather of the bf16 tables; vectors_t set and NULL; one launch of 4 grids, four one-grid launches, and
(0, 2) + (2, 2).  Sets B-E run the full cross, set A v6 x {egrid + index, re-gather} x {one, four}.
The last test checks the workspace hrf_field_backward_mlp writes (the scatter's producer) and scatters from it.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import encode_oracle as E
import scatter_cases as SC
import scatter_oracle as SO
from encode_oracle import F32, N_LEVELS
from helpers import MODEL_KW, field_without_vectors_t, positions_of, scatter_workspace, segment_grads, synthetic_rays
from humanrf_b200 import _lib as L

pytestmark = pytest.mark.gpu
SCHEDULES = {"one": ((0, 4),), "four": ((0, 1), (1, 1), (2, 1), (3, 1)), "pairs": ((0, 2), (2, 2))}
SOURCES = ("egrid+index", "egrid", "regather")
_CACHE = {}


def _module(fa, cuda):
    from humanrf_b200.scene_representation.humanrf import HumanRF

    m = HumanRF(sorted_frame_numbers=fa.sorted_frame_numbers, segment_sizes=tuple(fa.segment_sizes), **MODEL_KW)
    with torch.no_grad():
        for s, fg in enumerate(m.feature_grids):
            for k, g in enumerate(fg.grids()):
                src = E.bf16_to_f32(fa.tables[s][k]).reshape(-1)
                assert g.numel() == src.size, (s, k)
                g.copy_(torch.from_numpy(src))
            assert tuple(fg.vectors.shape) == fa.vectors[s].shape
            fg.vectors.copy_(torch.from_numpy(fa.vectors[s]))
    m = m.to(cuda)
    nat = m.native()
    nat.refresh()
    return m, nat


def _base(m, seed):
    """Base values of every gradient buffer (device), from a seeded generator."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for p in m.hot_parameters()[: 5 * m.num_segments]:
        b = torch.randn(p.shape, generator=g, device=p.device) * torch.exp2(torch.empty(p.shape, device=p.device).uniform_(-12, 2, generator=g))
        b[torch.rand(p.shape, generator=g, device=p.device) < 2 / 3] = 0
        out.append(b)
    return out


class _Dev:
    """One input set on the device: workspace, the three feature sources, samples with a host or device live count."""

    def __init__(self, inp: SO.ScatterInputs, egrid: np.ndarray, cuda, device_count: bool, seed: int):
        n = inp.n
        d_out = torch.from_numpy(np.ascontiguousarray(inp.dfeat.transpose(1, 0, 2).reshape(n, 32)))
        self.ws = scatter_workspace(d_out, torch.from_numpy(inp.pos4), inp.seg8, cuda)
        rng = np.random.default_rng(seed)
        stride = n + 37
        perm = rng.permutation(stride)[:n]
        wide = np.zeros((64, stride), np.uint32)
        wide[:, perm] = egrid
        self.egrid_wide = torch.from_numpy(wide.view(np.int32)).to(cuda)
        self.feat_index = torch.from_numpy(perm.astype(np.int32)).to(cuda)
        self.egrid = torch.from_numpy(np.ascontiguousarray(egrid).view(np.int32)).to(cuda)
        self.stride = stride
        self.samples = L.Samples()
        self.samples.num_samples = n
        self.count = torch.tensor([inp.live], dtype=torch.int64, device=cuda)
        if device_count:
            self.samples.num_samples_dev = self.count.data_ptr()
        else:
            assert inp.live == n

    def source(self, name):
        if name == "egrid+index":
            return self.egrid_wide.data_ptr(), self.feat_index.data_ptr(), self.stride
        if name == "egrid":
            return self.egrid.data_ptr(), None, 0
        return None, None, 0


def _run(m, nat, dev: _Dev, base, monkeypatch, gen, source, vt, schedule):
    monkeypatch.setenv("HRF_SCATTER", gen)
    grads, sg_dev = segment_grads(m)
    for g, b in zip(grads, base):
        g.copy_(b)
    field, keep = (nat.field, None) if vt else field_without_vectors_t(nat)
    eg, fi, stride = dev.source(source)
    for first, count in SCHEDULES[schedule]:
        L.check(L.lib().hrf_field_backward_tables(C.byref(field), C.byref(dev.samples), sg_dev.data_ptr(), eg, fi, stride,
                                                  dev.ws.data_ptr(), first, count, L.stream()))
    torch.cuda.synchronize()
    del keep
    return grads[: 5 * m.num_segments]


class _Stats:
    def __init__(self):
        self.worst = {}
        self.m_hist = np.zeros(3, np.int64)
        self.checked = 0

    def add(self, key, r, m):
        self.worst[key] = max(self.worst.get(key, 0.0), float(r.max()) if r.size else 0.0)
        mm = m[m > 0]
        self.m_hist += [(mm == 1).sum(), ((mm >= 2) & (mm <= 8)).sum(), (mm > 8).sum()]
        self.checked += r.size

    def report(self, tag):
        tab = np.zeros((4, N_LEVELS))
        for (kind, k, l), v in self.worst.items():
            if kind == "t":
                tab[k, l] = max(tab[k, l], v)
        vec = [max([v for (kind, a, _), v in self.worst.items() if kind == "v" and a == ax] or [0.0]) for ax in range(4)]
        tot = max(self.m_hist.sum(), 1)
        print(f"[{tag}] entries checked {self.checked}; worst error/bound {max(self.worst.values()):.3g}; touched with m=1 "
              f"{self.m_hist[0] / tot:.1%}, m=2-8 {self.m_hist[1] / tot:.1%}, m>8 {self.m_hist[2] / tot:.1%}")
        print(f"[{tag}]   per grid (max over levels): {np.array2string(tab.max(axis=1), precision=3)}; per level (max over "
              f"grids): {np.array2string(tab.max(axis=0), precision=2, max_line_width=300)}; vector axes x,y,z,t: "
              f"{np.array2string(np.array(vec), precision=3)}")
        return max(self.worst.values())


def _check(tag, got, base_np, sums: SO.Sums, st: _Stats, key):
    """One gradient array (any shape, fp32) against the reference sums plus its base values."""
    got = got.reshape(sums.val.shape)
    b = base_np.reshape(sums.val.shape)
    r = SO.ratio(got, sums.val + b.astype(np.float64), sums.bound(b))
    untouched = sums.m == 0
    assert (got[untouched].view(np.uint32) == b[untouched].view(np.uint32)).all(), \
        f"{tag} {key}: an entry no sample touches changed ({int((got[untouched] != b[untouched]).sum())} of them)"
    bad = np.argwhere(r > 1.0)
    assert bad.size == 0, f"{tag} {key}: {bad.shape[0]} entries beyond the bound, first {bad[:3].tolist()}, worst {r.max():.3g}"
    st.add(key, r, sums.m)


# ------------------------------------------------------------------------------------------------------ sets B-E
def _small(cuda):
    if "small" not in _CACHE:
        fa = SC.model()
        m, nat = _module(fa, cuda)
        _CACHE["small"] = (fa, m, nat, _base(m, 9))
    return _CACHE["small"]


@pytest.mark.parametrize("gen", ["6", "5"])
@pytest.mark.parametrize("name", SC.SMALL_SETS)
def test_scatter_small_sets(cuda, monkeypatch, name, gen):
    t0 = time.time()
    fa, m, nat, base = _small(cuda)
    key = ("inputs", name)
    if key not in _CACHE:
        inp = SC.small_set(fa, name)
        eg = SC.egrid_of(fa, inp.pos4, inp.seg8)
        inp_e = SO.ScatterInputs(inp.pos4, inp.seg8, inp.dfeat, inp.live, eg)
        refs = {"egrid": SO.reference(fa, inp_e), "regather": SO.reference(fa, inp)}
        dev = _Dev(inp, eg, cuda, device_count=name.startswith("live"), seed=len(name))
        _CACHE[key] = (inp, refs, dev)
    inp, refs, dev = _CACHE[key]
    base_np = [b.cpu().numpy() for b in base]
    worst = 0.0
    for source in SOURCES:
        ref = refs["regather" if source == "regather" else "egrid"]
        for vt in (True, False):
            for sched in SCHEDULES:
                tag = f"{name} v{gen} {source} vectors_t={'set' if vt else 'NULL'} {sched}"
                got = [g.cpu().numpy() for g in _run(m, nat, dev, base, monkeypatch, gen, source, vt, sched)]
                st = _Stats()
                for s in range(len(fa.tables)):
                    lt = fa.levels[s]
                    for k in range(4):
                        g2 = got[5 * s + k].reshape(-1, 2)
                        b2 = base_np[5 * s + k].reshape(-1, 2)
                        for l in range(N_LEVELS):
                            sl = slice(int(lt.offset[l]), int(lt.offset[l]) + int(lt.size[l]))
                            sums = SO.Sums(*(getattr(ref.tables[s][k], f)[sl] for f in ("val", "err", "mag", "m")))
                            _check(tag, g2[sl], b2[sl], sums, st, ("t", k, l))
                    gv, bv = got[5 * s + 4], base_np[5 * s + 4]
                    for ax in range(4):
                        sums = SO.Sums(*(getattr(ref.vectors[s], f)[ax] for f in ("val", "err", "mag", "m")))
                        _check(tag, gv[ax], bv[ax], sums, st, ("v", ax, s))
                if sched == "one" and vt:
                    worst = max(worst, st.report(tag))
                else:
                    worst = max(worst, max(st.worst.values()))
    print(f"[{name} v{gen}] 36 paths, worst error/bound {worst:.3g}, {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------------ set A
def _train_like(cuda):
    if "A" in _CACHE:
        return _CACHE["A"]
    segs = (100, 100, 50)
    fa = SC.model(segs, seed=11)
    m, nat = _module(fa, cuda)
    frames = fa.sorted_frame_numbers
    b = synthetic_rays(4608, 128, frames, ragged=True, seed=61)
    pos = positions_of(b).numpy()
    fr = b["frames"][b["ri"]].numpy()
    f2s, f2t = E.frame_luts(frames, segs)
    x = E.fadd(pos, F32(0.5))
    n_live = pos.shape[0] - pos.shape[0] % 8 - 3
    cap = n_live + 1000
    pos4 = np.full((cap, 4), 0.5, F32)
    pos4[:n_live, :3] = x[:n_live]
    pos4[:n_live, 3] = f2t[fr[:n_live]]
    seg8 = np.zeros(cap, np.uint8)
    seg8[:n_live] = f2s[fr[:n_live]]
    rng = np.random.default_rng(62)
    df = SC.d_features(rng, cap)
    df[:, n_live:] = np.nan
    # the saved per-grid features from the training forward itself (bit-exact with the encode reference elsewhere)
    s_q = nat.samples_query(torch.from_numpy(pos[:n_live]).to(cuda), None, torch.from_numpy(fr[:n_live].astype(np.int32)).to(cuda))
    _, _, _, saved = nat.forward(s_q, 0, False, True)
    torch.cuda.synchronize()
    eg = np.zeros((64, cap), np.uint32)
    eg[:, :n_live] = saved[32 * n_live:].view(torch.int32).cpu().numpy().view(np.uint32).reshape(64, n_live)
    inp = SO.ScatterInputs(pos4, seg8, df, n_live)
    inp_e = SO.ScatterInputs(pos4, seg8, df, n_live, eg)
    assert 240_000 < n_live < 270_000 and n_live % 8 != 0
    dev = _Dev(inp, eg, cuda, device_count=True, seed=63)
    _CACHE["A"] = (fa, m, nat, inp, inp_e, dev, _base(m, 64))
    return _CACHE["A"]


def test_scatter_train_like(cuda, monkeypatch):
    t0 = time.time()
    fa, m, nat, inp, inp_e, dev, base = _train_like(cuda)
    ns = len(fa.tables)
    paths = [(src, sched) for src in ("egrid+index", "regather") for sched in ("one", "four")]
    runs = {p: _run(m, nat, dev, base, monkeypatch, "6", p[0], True, p[1]) for p in paths}
    t1 = time.time()
    stats = {p: _Stats() for p in paths}
    vec = {mode: [SO.Sums.zeros((4, fa.vec_res, 32)) for _ in range(ns)] for mode in ("egrid", "regather")}
    coarse_max, fine_terms = 0.0, []
    for k in range(4):
        for l in range(N_LEVELS):
            tabs = SO.reference_level(fa, inp_e, k, l, vec["egrid"])
            SO.reference_level(fa, inp, k, l, vec["regather"])
            for s in range(ns):
                lt = fa.levels[s]
                sl = slice(2 * int(lt.offset[l]), 2 * (int(lt.offset[l]) + int(lt.size[l])))
                b = base[5 * s + k][sl].cpu().numpy().reshape(-1, 2)
                coarse_max = max(coarse_max, float(np.abs(tabs[s].val).max()))
                if l == N_LEVELS - 1:
                    one = tabs[s].m == 1
                    fine_terms.append(np.abs(tabs[s].val[one]))
                for p in paths:
                    got = runs[p][5 * s + k][sl].cpu().numpy().reshape(-1, 2)
                    _check(f"A {p}", got, b, tabs[s], stats[p], ("t", k, l))
    for p in paths:
        mode = "regather" if p[0] == "regather" else "egrid"
        for s in range(ns):
            got, b = runs[p][5 * s + 4].cpu().numpy(), base[5 * s + 4].cpu().numpy()
            for ax in range(4):
                sums = SO.Sums(*(getattr(vec[mode][s], f)[ax] for f in ("val", "err", "mag", "m")))
                _check(f"A {p}", got[ax], b[ax], sums, stats[p], ("v", ax, s))
        stats[p].report(f"A v6 {p[0]} {p[1]}")
    ft = np.concatenate(fine_terms)
    print(f"[A] {inp.live} live of {inp.n}; finest level, entries with one term: median |S| {np.median(ft):.3g}, "
          f"smallest {ft[ft > 0].min():.3g}; largest |S| of any table entry {coarse_max:.3g} (median ratio "
          f"{np.median(ft) / coarse_max:.2e}); kernels {t1 - t0:.1f} s, check {time.time() - t1:.1f} s")


# ------------------------------------------------------------------------------------------------------ producer
def test_workspace_contract(cuda, monkeypatch):
    """hrf_field_backward_mlp writes what the scatter reads: d(features) [16][n] float2 at 0, (x, y, z, t) float4 at
    128 n, the segment byte at 144 n, n the capacity; rows below a device live count only.  Then the scatter on that
    workspace and the forward's egrid against the reference fed with the workspace's own d(features)."""
    fa, m, nat, _ = _small(cuda)
    frames = fa.sorted_frame_numbers
    b = synthetic_rays(160, 64, list(frames) + [frames[-1] + 3], ragged=True, seed=71, n_distinct_frames=len(frames) + 1)
    n = int(b["t"].numel())
    live = n - 333
    g = {k: v.to(cuda).contiguous() for k, v in b.items() if k in ("o", "d", "frames", "t", "ri")}
    count = torch.tensor([live], dtype=torch.int64, device=cuda)
    s = nat.samples_rays(g["o"], g["d"], g["frames"], g["t"], g["ri"], count_dev=count)
    sigma, _, rgb, saved = nat.forward(s, 1, False, True)
    ws = torch.full((n * 40,), float("nan"), dtype=torch.float32, device=cuda)
    d_sigma = torch.randn(n, device=cuda)
    d_rgb = torch.randn(n, 3, device=cuda)
    d_mlp = torch.zeros(m.mlp_grad_elems, dtype=torch.float32, device=cuda)
    L.check(L.lib().hrf_field_backward_mlp(C.byref(nat.field), C.byref(s), d_sigma.data_ptr(), d_rgb.data_ptr(), None,
                                           saved.data_ptr(), None, d_mlp.data_ptr(), None, ws.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    raw = ws.cpu().numpy()
    x, fr = E.load_rays(b["o"].numpy(), b["d"].numpy(), b["frames"].numpy(), b["t"].numpy(), b["ri"].numpy())
    seg, t = E.segment_and_time(fa, fr)
    pos4 = raw[32 * n: 36 * n].reshape(n, 4)[:live]
    want = np.concatenate((x, t[:, None]), axis=1)[:live].astype(F32)
    has = seg[:live] >= 0
    assert (pos4[has].view(np.uint32) == want[has].view(np.uint32)).all(), "workspace positions"
    seg8 = raw.view(np.uint8)[144 * n: 145 * n][:live]
    assert (seg8 == np.where(seg[:live] >= 0, seg[:live], 255)).all(), "workspace segment bytes"
    assert (seg8 == 255).any() and (seg8 != 255).any()
    egrid = saved[32 * n:].view(torch.int32).cpu().numpy().view(np.uint32).reshape(64, n)
    enc = E.encode(fa, x[:live], fr[:live])
    em = E.egrid_mismatch(enc, egrid[:, :live])
    assert em["words"] == 0, em
    dfeat = raw[: 32 * n].reshape(16, n, 2)
    inp = SO.ScatterInputs(raw[32 * n: 36 * n].reshape(n, 4).copy(), raw.view(np.uint8)[144 * n: 145 * n].copy(),
                           dfeat.copy(), live, egrid)
    inp.pos4[live:] = 0.5
    ref = SO.reference(fa, inp)
    base = _base(m, 72)
    monkeypatch.setenv("HRF_SCATTER", "6")
    grads, sg_dev = segment_grads(m)
    for gg, bb in zip(grads, base):
        gg.copy_(bb)
    L.check(L.lib().hrf_field_backward_tables(C.byref(nat.field), C.byref(s), sg_dev.data_ptr(), saved.data_ptr() + 64 * n,
                                              None, 0, ws.data_ptr(), 0, 4, L.stream()))
    torch.cuda.synchronize()
    st = _Stats()
    for sgi in range(len(fa.tables)):
        for k in range(4):
            _check("producer", grads[5 * sgi + k].cpu().numpy(), base[5 * sgi + k].cpu().numpy(), ref.tables[sgi][k], st, ("t", k, 0))
        _check("producer", grads[5 * sgi + 4].cpu().numpy(), base[5 * sgi + 4].cpu().numpy(), ref.vectors[sgi], st, ("v", 3, sgi))
    st.report(f"producer: {live} live of {n}")
