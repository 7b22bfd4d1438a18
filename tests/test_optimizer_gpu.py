"""The fused Adam kernels against the float64 reference of tests/adam_oracle.py, entry by entry:

* hrf_adam_multi over one descriptor table of edge cases (sizes around the 4096-element block, float4 and scalar paths,
  a blob permutation, vectors with their transposed copy), gradients from 0 to overflowing squares, grad_scale 1 and
  1/3, zero_grad on and off, steps 1..10 and a large step count, an inactive tensor;
* the float4 and the scalar path, and hrf_adam_multi and hrf_dp_reduce_adam, give the same bits;
* hrf_dp_reduce_adam at world sizes 1, 2, 3, 5 and 8 simulated on one device (W gradient buckets, W shadow buffers, one
  launch per rank), in one launch and as five region launches;
* FusedTrainer's descriptor table at world 1: every hot parameter, its moments, the bf16 shadows, the packed MLP blob
  and the transposed vectors;
* hrf_adam_step.
Every case prints its worst err/bound per output and regime."""
import ctypes as C

import numpy as np
import pytest
import torch

import adam_oracle as A
from humanrf_b200 import _lib as L
from humanrf_b200.parallel import shard_bounds

pytestmark = pytest.mark.gpu

BLOCK = 4096
SENTINEL = -16447                      # bf16 bits 0xBFC1 (-1.5078125): a value no shadow write produces here


def _struct_array(items, dev):
    raw = b"".join(bytes(x) for x in items)
    return torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).to(dev)


def _np(t):
    return t.detach().cpu().numpy().copy()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint16)


def _bf16_bits(p32):
    return torch.from_numpy(np.ascontiguousarray(p32, np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


class Report:
    """Worst err/bound per (case, output/regime) over a test, printed at the end."""

    def __init__(self, title):
        self.title, self.rows = title, {}

    def add(self, case, stats):
        for k, (w, n) in stats.items():
            w0, n0 = self.rows.get((case, k), (None, 0))
            self.rows[(case, k)] = (w if w0 is None else (w0 if w is None else max(w0, w)), n0 + n)

    def regime_entries(self, regime):
        return sum(n for (_, k), (_, n) in self.rows.items() if k.startswith(f"m/{regime}"))

    def show(self):
        print(f"\n{self.title}: max err/bound")
        for (case, k) in sorted(self.rows):
            w, n = self.rows[(case, k)]
            print(f"  {case:<22} {k:<22} {'rule' if w is None else f'{w:.3f}':>8}  ({n} entries)")
        worst = [w for w, _ in self.rows.values() if w is not None]
        assert max(worst) <= 1.0, max(worst)


# --------------------------------------------------------------------------------------------------------------------
# hrf_adam_multi over an edge-case table
# name, n, float offset (mod 4) in the flat buffers, shadow ("f4": 8-byte aligned, "odd": 2 bytes off, None),
# blob permutation, vec_res (vectors with a transposed copy), twin (same data as that tensor)
EDGE = [
    ("n1", 1, 0, "f4", False, 0, None),
    ("n3_off1", 3, 1, "f4", False, 0, None),
    ("n4", 4, 0, "f4", False, 0, None),
    ("n4095", 4095, 0, "f4", False, 0, None),
    ("n4096", 4096, 0, "f4", False, 0, None),
    ("n4097", 4097, 0, "f4", False, 0, None),
    ("n12293", 3 * 4096 + 5, 0, "f4", False, 0, None),
    ("n12293_off2", 3 * 4096 + 5, 2, "f4", False, 0, None),
    ("n4096_shadow_odd", 4096, 0, "odd", False, 0, None),
    ("n4096_off3", 4096, 3, None, False, 0, None),
    ("blob_perm", 5000, 0, "f4", True, 0, None),
    ("vectors_vr1", 4 * 1 * 32, 0, None, False, 1, None),
    ("vectors_vr2048", 4 * 2048 * 32, 0, None, False, 2048, None),
    ("twin_f4", 8192, 0, "f4", False, 0, None),
    ("twin_scalar", 8192, 1, "f4", False, 0, "twin_f4"),
    ("inactive", 4097, 0, "f4", False, 0, None),
]
LAUNCHES = list(range(1, 11)) + [1_000_000]          # step counter after each launch (the last one set directly)


def _inactive_at(launch_idx):
    return launch_idx % 3 == 1                        # the "inactive" tensor sits out launches 2, 5, 8, 11


class EdgeTable:
    def __init__(self, dev, seed=11):
        self.dev, self.specs = dev, EDGE
        names = [s[0] for s in EDGE]
        self.pos, self.spos, pos, spos = [], [], 0, 0
        for name, n, off, sh, perm, vr, twin in EDGE:
            pos = -(-pos // 4) * 4 + off
            self.pos.append(pos)
            pos += n
            if sh is None:
                self.spos.append(None)
            else:
                spos = -(-spos // 4) * 4 + (1 if sh == "odd" else 0)
                self.spos.append(spos)
                spos += n
        total, stotal = pos + 4, spos + 4
        self.p, self.m, self.v, self.g = (torch.zeros(total, device=dev) for _ in range(4))
        self.shadow = torch.zeros(stotal, dtype=torch.bfloat16, device=dev)
        self.rngs, self.perms, self.vt = [], [], []
        p_host = np.zeros(total, np.float32)
        for i, (name, n, off, sh, perm, vr, twin) in enumerate(EDGE):
            rng = np.random.default_rng((seed, i))
            self.rngs.append(rng)
            p0, _, _ = A.edge_state(rng, n)
            if twin is not None:
                j = names.index(twin)
                p0 = p_host[self.pos[j]:self.pos[j] + n].copy()
            p_host[self.pos[i]:self.pos[i] + n] = p0
            self.perms.append(torch.randperm(n, generator=torch.Generator().manual_seed(i)).to(torch.int32).to(dev) if perm else None)
            self.vt.append(torch.zeros(n, device=dev) if vr else None)
        self.p.copy_(torch.from_numpy(p_host))
        self.twin_of = {i: names.index(s[6]) for i, s in enumerate(EDGE) if s[6] is not None}
        self.active = torch.ones(len(EDGE), dtype=torch.int32, device=dev)
        self.steps = torch.zeros(len(EDGE), dtype=torch.int32, device=dev)
        items, first = [], 0
        for i, (name, n, off, sh, perm, vr, twin) in enumerate(EDGE):
            t = L.AdamTensor()
            a = self.pos[i]
            t.param, t.exp_avg, t.exp_avg_sq, t.grad = (x[a:].data_ptr() for x in (self.p, self.m, self.v, self.g))
            t.shadow_bf16 = self.shadow[self.spos[i]:].data_ptr() if sh is not None else None
            t.blob_perm = self.perms[i].data_ptr() if perm else None
            t.active, t.step, t.n, t.first_block = self.active[i:].data_ptr(), self.steps[i:].data_ptr(), n, first
            t.vectors_t, t.vec_res = (self.vt[i].data_ptr(), vr) if vr else (None, 0)
            first += -(-n // BLOCK)
            items.append(t)
        self.blocks = first
        self.desc = _struct_array(items, dev)

    def sl(self, i):
        return slice(self.pos[i], self.pos[i] + self.specs[i][1])

    def write_gradients(self):
        g = _np(self.g)
        for i, (name, n, *_rest) in enumerate(self.specs):
            if i in self.twin_of:
                continue
            gi = A.edge_gradients(self.rngs[i], n)[0]
            g[self.sl(i)] = gi
        for i, j in self.twin_of.items():
            g[self.sl(i)] = g[self.sl(j)]
        self.g.copy_(torch.from_numpy(g))

    def snapshot(self):
        torch.cuda.synchronize()
        return dict(p=_np(self.p), m=_np(self.m), v=_np(self.v), g=_np(self.g), sh=_np(self.shadow.view(torch.int16)).view(np.uint16),
                    steps=_np(self.steps), vt=[None if x is None else _np(x) for x in self.vt])


@pytest.mark.parametrize("zero_grad", [1, 0], ids=["zero_grad", "keep_grad"])
@pytest.mark.parametrize("gscale", [1.0, 1.0 / 3.0], ids=["gscale1", "gscale1_3"])
def test_adam_multi_edge_table_against_the_reference(cuda, gscale, zero_grad):
    """hrf_adam_multi, one launch per step over the whole edge-case table: p', m', v' within the reference's bound (or by
    its underflow / overflow rules), the bf16 shadow equal to torch's bf16 of the kernel's p' (through blob_perm where
    there is one), vectors_t in the transposed layout, gradients cleared only with zero_grad; the inactive tensor, its
    counter and its gradient bit-unchanged; the float4 twin and the scalar twin bit-identical."""
    lib = L.lib()
    tab = EdgeTable(cuda)
    sc = A.Scalars(gscale=gscale)
    rep = Report(f"hrf_adam_multi, grad_scale {gscale:.4f}, zero_grad {zero_grad}")
    expect_steps = np.zeros(len(EDGE), np.int64)
    for li, k_after in enumerate(LAUNCHES):
        if k_after == LAUNCHES[-1]:                  # a long run: set every counter directly
            expect_steps[:] = k_after - 1
            tab.steps.fill_(k_after - 1)
        act = np.ones(len(EDGE), np.int32)
        act[-1] = 0 if _inactive_at(li) else 1
        tab.active.copy_(torch.from_numpy(act))
        tab.write_gradients()
        before = tab.snapshot()
        L.check(lib.hrf_adam_multi(tab.desc.data_ptr(), len(EDGE), tab.blocks, sc.lr, sc.b1, sc.b2, sc.eps, sc.gscale,
                                     zero_grad, L.stream()))
        after = tab.snapshot()
        expect_steps += act
        assert np.array_equal(after["steps"], expect_steps), (after["steps"], expect_steps)
        for i, (name, n, off, sh, perm, vr, twin) in enumerate(EDGE):
            s = tab.sl(i)
            p0, m0, v0, g0 = before["p"][s], before["m"][s], before["v"][s], before["g"][s]
            p1, m1, v1, g1 = after["p"][s], after["m"][s], after["v"][s], after["g"][s]
            shs = slice(tab.spos[i], tab.spos[i] + n) if sh is not None else None
            if not act[i]:
                for key in ("p", "m", "v", "g"):
                    assert np.array_equal(_bits(after[key][s]), _bits(before[key][s])), (name, key)
                if shs is not None:
                    assert np.array_equal(after["sh"][shs], before["sh"][shs]), name
                continue
            ref = A.reference(p0, m0, v0, [g0], int(expect_steps[i]), sc, m1, v1)
            rep.add(name, A.check(p1, m1, v1, p0, ref))
            if zero_grad:
                assert np.array_equal(_bits(g1), np.zeros(n, np.uint32)), name
            else:
                assert np.array_equal(_bits(g1), _bits(g0)), name
            if shs is not None:
                got = after["sh"][shs]
                if perm:
                    got = got[tab.perms[i].cpu().numpy().astype(np.int64)]
                assert np.array_equal(got, _bf16_bits(p1)), name
            if vr:
                assert np.array_equal(_bits(after["vt"][i]), _bits(A.transpose_vectors(p1))), name
        for i, j in tab.twin_of.items():
            for key in ("p", "m", "v"):
                assert np.array_equal(_bits(after[key][tab.sl(i)]), _bits(after[key][tab.sl(j)])), ("twin", key, li)
        # the shadow outside every table keeps its initial zeros
        inside = np.zeros(after["sh"].size, bool)
        for i, spec in enumerate(EDGE):
            if tab.spos[i] is not None:
                inside[tab.spos[i]:tab.spos[i] + spec[1]] = True
        assert not after["sh"][~inside].any()
    rep.show()
    for regime in ("subnormal", "underflow", "overflow"):
        assert rep.regime_entries(regime) > 0, regime


# --------------------------------------------------------------------------------------------------------------------
# hrf_dp_reduce_adam, W simulated ranks on one device
# name, n, sharded, segment (active flag index; None = always active), local shadow ("blob" with a permutation,
# "f4" plain, None), vec_res
DP = [
    ("grid_big", 8 * 4096 * 2 + 77, True, 0, None, 0),
    ("grid_mid", 3 * 4096 + 5, True, 0, None, 0),
    ("grid_tiny", 100, True, 1, None, 0),
    ("grid_seg1", 9000, True, 1, None, 0),
    ("vectors", 4 * 3 * 32, False, 1, None, 3),
    ("mlp", 5000, False, None, "blob", 0),
    ("embeddings", 640, False, None, None, 0),
    ("replicated_f4", 4096 + 8, False, None, "f4", 0),
]
REGIONS = [(0,), (1,), (2, 3), (4,), (5, 6, 7)]        # tensors per region launch (descriptor order)
SHADOW_GAP = 16


class DpRank:
    """One simulated rank's own state: masters and moments, step counters, active flags, replicated copies."""

    def __init__(self, dev, init, perms):
        self.p = [torch.from_numpy(x.copy()).to(dev) for x in init]
        self.m = [torch.zeros(x.size, device=dev) for x in init]
        self.v = [torch.zeros(x.size, device=dev) for x in init]
        self.steps = torch.zeros(len(DP), dtype=torch.int32, device=dev)
        self.active = torch.ones(2, dtype=torch.int32, device=dev)
        self.local = [torch.zeros(spec[1], dtype=torch.bfloat16, device=dev) if spec[4] else None for spec in DP]
        self.vt = [torch.zeros(spec[1], device=dev) if spec[5] else None for spec in DP]
        self.perms = perms

    def state(self):
        return dict(p=[_np(x) for x in self.p], m=[_np(x) for x in self.m], v=[_np(x) for x in self.v], steps=_np(self.steps),
                    local=[None if x is None else _np(x.view(torch.int16)).view(np.uint16) for x in self.local],
                    vt=[None if x is None else _np(x) for x in self.vt])


class DpWorld:
    def __init__(self, dev, world, seed=5):
        self.dev, self.W = dev, world
        self.rngs = [np.random.default_rng((seed, world, i)) for i in range(len(DP))]
        init = [A.edge_state(self.rngs[i], spec[1])[0] for i, spec in enumerate(DP)]
        perms = [torch.randperm(spec[1], generator=torch.Generator().manual_seed(i)).to(torch.int32).to(dev) if spec[4] == "blob" else None
                 for i, spec in enumerate(DP)]
        self.goff = np.concatenate(([0], np.cumsum([spec[1] for spec in DP]))).astype(np.int64)
        self.soff, pos = [], SHADOW_GAP
        for spec in DP:
            if spec[2]:
                self.soff.append(pos)
                pos += spec[1] + SHADOW_GAP
            else:
                self.soff.append(-1)
        self.shadow_len = pos
        self.buckets = [torch.zeros(int(self.goff[-1]) + 4, device=dev) for _ in range(world)]
        self.shadows = [torch.full((pos,), SENTINEL, dtype=torch.int16, device=dev) for _ in range(world)]
        self.ranks = [DpRank(dev, init, perms) for _ in range(world)]
        self.descs, self.blocks, self.firsts, self.bounds = [], [], [], []
        for r, rk in enumerate(self.ranks):
            items, first, firsts, bounds = [], 0, [], []
            for i, (name, n, sharded, seg, local, vr) in enumerate(DP):
                t = L.DpTensor()
                t.param, t.exp_avg, t.exp_avg_sq = rk.p[i].data_ptr(), rk.m[i].data_ptr(), rk.v[i].data_ptr()
                t.grad_offset, t.n = int(self.goff[i]), n
                t.blob_perm = perms[i].data_ptr() if perms[i] is not None else None
                t.active = rk.active[seg:].data_ptr() if seg is not None else None
                t.step = rk.steps[i:].data_ptr()
                t.vectors_t, t.vec_res = (rk.vt[i].data_ptr(), vr) if vr else (None, 0)
                if sharded:
                    t.sharded, t.shadow_offset, t.local_shadow_bf16 = 1, self.soff[i], None
                    t.shard_begin, t.shard_end = shard_bounds(n, r, world, BLOCK)
                else:
                    t.sharded, t.shadow_offset = 0, -1
                    t.local_shadow_bf16 = rk.local[i].data_ptr() if local else None
                    t.shard_begin, t.shard_end = 0, n
                bounds.append((t.shard_begin, t.shard_end))
                t.first_block = first
                firsts.append(first)
                first += -(-(t.shard_end - t.shard_begin) // BLOCK)
                items.append(t)
            self.descs.append(_struct_array(items, dev))
            self.blocks.append(first)
            self.firsts.append(firsts + [first])
            self.bounds.append(bounds)

    def peers(self, r):
        P = L.DpPeers()
        for q in range(self.W):
            P.grad[q], P.shadow[q] = self.buckets[q].data_ptr(), self.shadows[q].data_ptr()
        P.world, P.rank = self.W, r
        return P

    def write_gradients(self, cancel=True):
        grads = [A.edge_gradients(self.rngs[i], spec[1], ranks=self.W, cancel=cancel) for i, spec in enumerate(DP)]
        for r in range(self.W):
            flat = np.zeros(self.buckets[r].numel(), np.float32)
            for i in range(len(DP)):
                flat[self.goff[i]:self.goff[i + 1]] = grads[i][r]
            self.buckets[r].copy_(torch.from_numpy(flat))
        return grads

    def launch(self, sc, regions=False):
        lib = L.lib()
        for r in range(self.W):
            P = self.peers(r)
            if not regions:
                L.check(lib.hrf_dp_reduce_adam(C.byref(P), self.descs[r].data_ptr(), len(DP), 0, self.blocks[r], 1, sc.lr, sc.b1,
                                                 sc.b2, sc.eps, sc.gscale, L.stream()))
                continue
            f = self.firsts[r]
            for j, group in enumerate(REGIONS):
                a, b = f[group[0]], f[group[-1] + 1]
                L.check(lib.hrf_dp_reduce_adam(C.byref(P), self.descs[r].data_ptr(), len(DP), a, b - a, 1 if j == 0 else 0, sc.lr,
                                                 sc.b1, sc.b2, sc.eps, sc.gscale, L.stream()))

    def state(self):
        torch.cuda.synchronize()
        return dict(ranks=[rk.state() for rk in self.ranks], shadows=[_np(s).view(np.uint16) for s in self.shadows],
                    buckets=[_np(b) for b in self.buckets])


def _same_state(a, b, what):
    for r, (x, y) in enumerate(zip(a["ranks"], b["ranks"])):
        assert np.array_equal(x["steps"], y["steps"]), (what, r)
        for key in ("p", "m", "v"):
            for i in range(len(DP)):
                assert np.array_equal(_bits(x[key][i]), _bits(y[key][i])), (what, r, key, DP[i][0])
        for key in ("local", "vt"):
            for i in range(len(DP)):
                if x[key][i] is not None:
                    assert np.array_equal(_bits(x[key][i]), _bits(y[key][i])), (what, r, key, DP[i][0])
    for r in range(len(a["shadows"])):
        assert np.array_equal(a["shadows"][r], b["shadows"][r]), (what, "shadow", r)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_dp_reduce_adam_world_sizes_on_one_device(cuda, world):
    """hrf_dp_reduce_adam with W gradient buckets and W shadow buffers on one device, one launch per simulated rank:
    the union of the rank shards of each sharded tensor matches the reference on the fp32 rank-order sum with
    grad_scale 1/W (cancelling gradients make the order visible); entries outside a rank's shard stay bit-unchanged on it;
    all W shadow buffers equal the bf16 of the assembled masters and keep the sentinel outside the tables; replicated
    tensors are bit-identical on all ranks and match the reference; counters advance once per step; the buckets are
    left untouched; a segment sits out step 2.  The same steps as five region launches give the same bits."""
    A_, B_ = DpWorld(cuda, world), DpWorld(cuda, world)
    sc = A.Scalars(gscale=1.0 / world)
    rep = Report(f"hrf_dp_reduce_adam, world {world}")
    expect = np.zeros(len(DP), np.int64)
    empty = sum(1 for r in range(world) for (a, b), spec in zip(A_.bounds[r], DP) if spec[2] and b == a)
    if world >= 2:
        assert empty > 0          # grid_tiny leaves every rank but the first without a shard
    for step in range(3):
        seg1 = 0 if step == 1 else 1
        for wd in (A_, B_):
            for rk in wd.ranks:
                rk.active.copy_(torch.tensor([1, seg1], dtype=torch.int32))
        grads = A_.write_gradients()
        B_.write_gradients()
        before = A_.state()
        A_.launch(sc)
        B_.launch(sc, regions=True)
        after, after_b = A_.state(), B_.state()
        _same_state(after, after_b, f"regions, step {step}")
        act = np.array([1 if spec[3] is None or spec[3] == 0 or seg1 else 0 for spec in DP])
        expect += act
        for r in range(world):
            assert np.array_equal(after["ranks"][r]["steps"], expect), (r, after["ranks"][r]["steps"], expect)
            assert np.array_equal(_bits(after["buckets"][r]), _bits(before["buckets"][r])), r
        inside = np.zeros(A_.shadow_len, bool)
        for i, (name, n, sharded, seg, local, vr) in enumerate(DP):
            if sharded:
                inside[A_.soff[i]:A_.soff[i] + n] = True
            if not act[i]:
                for r in range(world):
                    for key in ("p", "m", "v"):
                        assert np.array_equal(_bits(after["ranks"][r][key][i]), _bits(before["ranks"][r][key][i])), (name, r, key)
                continue
            k = int(expect[i])
            if sharded:
                asm = {key: np.zeros(n, np.float32) for key in ("p0", "m0", "v0", "p1", "m1", "v1")}
                for r in range(world):
                    a, b = A_.bounds[r][i]
                    for key in ("p", "m", "v"):
                        asm[key + "0"][a:b] = before["ranks"][r][key][i][a:b]
                        asm[key + "1"][a:b] = after["ranks"][r][key][i][a:b]
                        out = np.ones(n, bool)
                        out[a:b] = False
                        assert np.array_equal(_bits(after["ranks"][r][key][i][out]), _bits(before["ranks"][r][key][i][out])), (name, r, key)
                ref = A.reference(asm["p0"], asm["m0"], asm["v0"], list(grads[i]), k, sc, asm["m1"], asm["v1"])
                rep.add(name, A.check(asm["p1"], asm["m1"], asm["v1"], asm["p0"], ref))
                want = _bf16_bits(asm["p1"])
                for r in range(world):
                    assert np.array_equal(after["shadows"][r][A_.soff[i]:A_.soff[i] + n], want), (name, "shadow", r)
            else:
                x0, x1 = before["ranks"][0], after["ranks"][0]
                for r in range(1, world):
                    for key in ("p", "m", "v", "local", "vt"):
                        if x1[key][i] is not None:
                            assert np.array_equal(_bits(after["ranks"][r][key][i]), _bits(x1[key][i])), (name, r, key)
                ref = A.reference(x0["p"][i], x0["m"][i], x0["v"][i], list(grads[i]), k, sc, x1["m"][i], x1["v"][i])
                rep.add(name, A.check(x1["p"][i], x1["m"][i], x1["v"][i], x0["p"][i], ref))
                if local == "blob":
                    got = x1["local"][i][A_.ranks[0].perms[i].cpu().numpy().astype(np.int64)]
                    assert np.array_equal(got, _bf16_bits(x1["p"][i])), name
                elif local == "f4":
                    assert np.array_equal(x1["local"][i], _bf16_bits(x1["p"][i])), name
                if vr:
                    assert np.array_equal(_bits(x1["vt"][i]), _bits(A.transpose_vectors(x1["p"][i]))), name
        for r in range(world):
            assert np.all(after["shadows"][r][~inside] == np.uint16(SENTINEL & 0xFFFF)), r
    rep.show()


def test_adam_multi_and_dp_reduce_adam_agree_bit_for_bit(cuda):
    """Replicated tensors rely on every rank producing the same bits: hrf_adam_multi and hrf_dp_reduce_adam (world 1,
    grad_scale 1) on the same tensors, float4- and scalar-path alike, give identical p, m, v and shadows."""
    lib = L.lib()
    world = DpWorld(cuda, 1, seed=9)
    single = DpWorld(cuda, 1, seed=9)            # the same data, stepped by hrf_adam_multi
    rk = single.ranks[0]
    items, first = [], 0
    grad = single.buckets[0]
    shadow = single.shadows[0]
    for i, (name, n, sharded, seg, local, vr) in enumerate(DP):
        t = L.AdamTensor()
        t.param, t.exp_avg, t.exp_avg_sq = rk.p[i].data_ptr(), rk.m[i].data_ptr(), rk.v[i].data_ptr()
        t.grad = grad[int(single.goff[i]):].data_ptr()
        if sharded:
            t.shadow_bf16, t.blob_perm = shadow[single.soff[i]:].data_ptr(), None
        else:
            t.shadow_bf16 = rk.local[i].data_ptr() if local else None
            t.blob_perm = rk.perms[i].data_ptr() if local == "blob" else None
        t.active = rk.active[seg:].data_ptr() if seg is not None else None
        t.step, t.n, t.first_block = rk.steps[i:].data_ptr(), n, first
        t.vectors_t, t.vec_res = (rk.vt[i].data_ptr(), vr) if vr else (None, 0)
        first += -(-n // BLOCK)
        items.append(t)
    desc = _struct_array(items, cuda)
    sc = A.Scalars(gscale=1.0)
    for step in range(3):
        world.write_gradients(cancel=False)
        single.write_gradients(cancel=False)
        world.launch(sc)
        L.check(lib.hrf_adam_multi(desc.data_ptr(), len(DP), first, sc.lr, sc.b1, sc.b2, sc.eps, 1.0, 0, L.stream()))
        a, b = world.state(), single.state()
        _same_state(a, b, f"adam_multi vs dp_reduce_adam, step {step}")


# --------------------------------------------------------------------------------------------------------------------
def test_fused_trainer_descriptor_table_at_world_1(cuda):
    """FusedTrainer's own descriptor table (two segments, camera embeddings): a known random bucket through
    _exchange_and_adam; every hot parameter and its exp_avg / exp_avg_sq slice against the reference, the bf16 shadow
    tables, the packed MLP blob (through mlp_blob_permutation, so the colour net's blob_perm[n_sig:] slice is checked)
    and the transposed vectors against the bf16 / layout rules; the bucket zeroed afterwards."""
    from humanrf_b200.scene_representation.grid_layout import mlp_blob_permutation
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW
    from humanrf_b200.training import FusedTrainer

    kw = {**MODEL_KW, "camera_embedding_dim": 4, "log2_hashmap_size": 15}
    frames = tuple(range(15, 21))
    torch.manual_seed(0)
    model = HumanRF(sorted_frame_numbers=frames, segment_sizes=(3, 3), **kw).to(cuda)
    with torch.no_grad():
        for p in model.hot_parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(p.numel())).to(cuda) * 0.5)
    tr = FusedTrainer(model, prune=False)
    tr.keep_grad = False
    params = model.hot_parameters()
    assert len(params) == 2 * 5 + 3
    rep = Report("FusedTrainer descriptor table, world 1")
    rng = np.random.default_rng(3)
    total = tr.grad.numel()
    dst, src = mlp_blob_permutation(model.camera_embedding_dim)
    for k in (1, 2):
        bucket = (rng.standard_normal(total) * 10.0 ** rng.uniform(-4, 1, total)).astype(np.float32)
        tr.grad.copy_(torch.from_numpy(bucket))
        torch.cuda.synchronize()
        p0 = [_np(p).reshape(-1) for p in params]
        m0, v0 = _np(tr.exp_avg), _np(tr.exp_avg_sq)
        sc = A.Scalars(lr=tr.current_lr(), b1=tr.betas[0], b2=tr.betas[1], eps=tr.eps, gscale=1.0)
        tr._exchange_and_adam()
        torch.cuda.synchronize()
        m1, v1 = _np(tr.exp_avg), _np(tr.exp_avg_sq)
        assert tr.steps == [k] * len(params)
        assert not _np(tr.grad).any()
        for i, p in enumerate(params):
            a, b = tr.slices[i]
            p1 = _np(p).reshape(-1)
            ref = A.reference(p0[i], m0[a:b], v0[a:b], [bucket[a:b]], k, sc, m1[a:b], v1[a:b])
            rep.add(f"param {i}", A.check(p1, m1[a:b], v1[a:b], p0[i], ref))
        nat = tr.nat
        for s_, fg in enumerate(model.feature_grids):
            for kk, g in enumerate(fg.grids()):
                assert np.array_equal(_np(nat.shadows[s_][kk].view(torch.int16)).view(np.uint16), _bf16_bits(_np(g).reshape(-1))), (s_, kk)
            assert np.array_equal(_bits(_np(nat.vec_t[s_])), _bits(A.transpose_vectors(_np(fg.vectors).reshape(-1)))), s_
        flat = np.concatenate([_np(model.sigma_net.params).reshape(-1), _np(model.color_net.params).reshape(-1)])
        blob = _np(nat.blob.view(torch.int16)).view(np.uint16)
        assert np.array_equal(blob[dst], _bf16_bits(flat[src]))
    rep.show()


def test_adam_step_against_the_reference(cuda):
    """hrf_adam_step (one tensor per launch, bias corrections from the host): within the reference's bound at steps 1, 2
    and 10, and its bf16 shadow equal to torch's bf16 of p'."""
    lib = L.lib()
    n = 10007
    rng = np.random.default_rng(21)
    p0, _, _ = A.edge_state(rng, n)
    p = torch.from_numpy(p0).to(cuda)
    m, v = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=cuda)
    sc = A.Scalars(gscale=0.5)
    rep = Report("hrf_adam_step")
    for k in range(1, 11):
        g = torch.from_numpy(A.edge_gradients(rng, n)[0]).to(cuda)
        b = [_np(p), _np(m), _np(v)]
        L.check(lib.hrf_adam_step(p.data_ptr(), m.data_ptr(), v.data_ptr(), g.data_ptr(), shadow.data_ptr(), n, sc.lr, sc.b1,
                                    sc.b2, sc.eps, k, sc.gscale, L.stream()))
        torch.cuda.synchronize()
        p1, m1, v1 = _np(p), _np(m), _np(v)
        ref = A.reference(b[0], b[1], b[2], [_np(g)], k, sc, m1, v1)
        rep.add("n10007", A.check(p1, m1, v1, b[0], ref))
        assert np.array_equal(_np(shadow.view(torch.int16)).view(np.uint16), _bf16_bits(p1))
    rep.show()
