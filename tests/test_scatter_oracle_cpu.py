"""The gradient-scatter reference (tests/scatter_oracle.py) on the CPU: it is the adjoint of the encode reference, it
agrees with float64 autograd, its per-entry bound holds for fp32 sums in legal orders, its walk restatement agrees with
the plain sum, and every deliberately wrong reference (scatter_oracle.MUTANTS) exceeds twice the bound on the inputs the
GPU test feeds the kernels (tests/scatter_cases.py, rebuilt here from the same seeds)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import encode_oracle as E
import scatter_cases as SC
import scatter_oracle as SO
from encode_oracle import F32, F64, N_LEVELS
from helpers import scatter_autograd_reference
from oracle import field as OF

_CACHE = {}


def _fa():
    if "fa" not in _CACHE:
        _CACHE["fa"] = SC.model()
    return _CACHE["fa"]


def _set(name, egrid=False):
    key = ("set", name, egrid)
    if key not in _CACHE:
        fa = _fa()
        inp = SC.small_set(fa, name)
        if egrid:
            inp.egrid = SC.egrid_of(fa, inp.pos4, inp.seg8)
        _CACHE[key] = inp
    return _CACHE[key]


def _blend64(fa, s, k, l, x, table64):
    """sum_c w_c table[idx_c] in float64 with the encode reference's fp32 weights and corner indices."""
    lt = fa.levels[s]
    cells = [E.to_cell(lt.scale[l], x[:, a]) for a in E.GRID_AXES[k]]
    (ga, fa_), (gb, fb), (gc, fc) = cells
    one = F32(1)
    wd = ((E.fsub(one, fa_), fa_), (E.fsub(one, fb), fb), (E.fsub(one, fc), fc))
    out = np.zeros((x.shape[0], 2), F64)
    for c in range(8):
        w = E.fmul(E.fmul(wd[0][c & 1], wd[1][(c >> 1) & 1]), wd[2][(c >> 2) & 1])
        idx = E.corner_index(c, bool(lt.hashed[l]), int(lt.res[l]), int(lt.size[l]), ga, gb, gc).astype(np.int64)
        out += w.astype(F64)[:, None] * table64[int(lt.offset[l]) + idx]
    return out


@pytest.mark.parametrize("name", ["edges", "segments"])
def test_adjoint_of_the_encode(name):
    """sum_entries S * delta == sum_samples dO * (v (.) blend of delta) for random table perturbations, and the same for
    the vectors (sum_rows S_v * delta_v == sum_samples dO * e (.) lerp of delta_v), in float64."""
    fa = _fa()
    inp = _set(name, egrid=True)
    ref = SO.reference(fa, inp)
    rng = np.random.default_rng(5)
    ok = SO.counted(inp, len(fa.tables))
    for s in range(len(fa.tables)):
        rows = np.nonzero(ok & (inp.seg8 == s))[0]
        x = inp.pos4[rows]
        vec = fa.vectors[s].astype(F64)
        dvec = rng.standard_normal(vec.shape)
        lhs_v = float((ref.vectors[s].val * dvec).sum())
        rhs_v = 0.0
        for k in range(4):
            delta = rng.standard_normal((fa.levels[s].n_entries, 2))
            lhs = float((ref.tables[s][k].val * delta).sum())
            a = E.VECTOR_OF_TERM[k]
            i0, i1, frac = E.row_tap(x[:, a], fa.vec_res)
            fr = frac.astype(F64)[:, None]
            rhs = 0.0
            for l in range(N_LEVELS):
                dO = inp.dfeat[l, rows].astype(F64)
                v = vec[a][i0, 2 * l:2 * l + 2] + fr * (vec[a][i1, 2 * l:2 * l + 2] - vec[a][i0, 2 * l:2 * l + 2])
                rhs += float((dO * v * _blend64(fa, s, k, l, x, delta)).sum())
                word = inp.egrid[4 * l + k, rows]
                e = np.stack((E.bf16_to_f32((word & 0xFFFF).astype(np.uint16)),
                              E.bf16_to_f32((word >> 16).astype(np.uint16))), axis=1).astype(F64)
                dv = dvec[a][i0, 2 * l:2 * l + 2] + fr * (dvec[a][i1, 2 * l:2 * l + 2] - dvec[a][i0, 2 * l:2 * l + 2])
                rhs_v += float((dO * e * dv).sum())
            scale = float((np.abs(ref.tables[s][k].val) * np.abs(delta)).sum())
            assert abs(lhs - rhs) <= 1e-12 * scale, (name, s, k, lhs, rhs)
        assert abs(lhs_v - rhs_v) <= 1e-12 * float((np.abs(ref.vectors[s].val) * np.abs(dvec)).sum()), (name, s)


def test_agrees_with_float64_autograd():
    """Against float64 autograd through oracle.hashgrid and oracle.field.lerp_vectors (test_scatter_gpu's reference) on
    in-cube ray samples (both feature sources)."""
    fa = _fa()
    inp = _set("segments", egrid=True)
    ok = SO.counted(inp, len(fa.tables))
    rows = np.nonzero(ok)[0][:1500]
    sub = SO.ScatterInputs(inp.pos4[rows], inp.seg8[rows], inp.dfeat[:, rows], rows.size, inp.egrid[:, rows])
    om = SimpleNamespace(segments=[SimpleNamespace(grids=[torch.from_numpy(E.bf16_to_f32(t)) for t in fa.tables[s]],
                                                   vectors=torch.from_numpy(fa.vectors[s]), log2T=fa.log2T[s])
                                   for s in range(len(fa.tables))])
    d_out = torch.from_numpy(sub.dfeat.transpose(1, 0, 2).reshape(rows.size, 32).copy())
    ref_tab, ref_vec, _ = scatter_autograd_reference(om, sub.seg8.astype(np.int64), torch.from_numpy(sub.pos4), d_out,
                                                     OF.lerp_vectors)
    for mode in ("egrid", "gather"):
        r = SO.reference(fa, sub if mode == "egrid" else SO.ScatterInputs(sub.pos4, sub.seg8, sub.dfeat, sub.live))
        for s in range(len(fa.tables)):
            for k in range(4):
                a, b = r.tables[s][k].val.reshape(-1), ref_tab[s][k].numpy()
                assert np.linalg.norm(a - b) <= 1e-9 * np.linalg.norm(b), (mode, s, k)
            a, b = r.vectors[s].val, ref_vec[mode][s].numpy()
            e = np.linalg.norm(a - b) / np.linalg.norm(b)
            print(f"{mode} segment {s}: vectors relnorm {e:.2e}")
            assert e <= 1e-6, (mode, s, e)     # autograd's fp32 lerp coordinate (c * VR - 0.5 unfused), same taps


def _ordered_sums(entries, leaves, order, base):
    """fp32 sums of `leaves` (exact float64 products) per entry in a legal order: forward (acc = fl(leaf + acc), the fma
    run, starting from the base value), reverse, or pairwise (the first round adds two leaves, then fp32 adds)."""
    o = np.argsort(entries, kind="stable")
    e, v = entries[o], leaves[o]
    if order == "reverse":
        e, v = e[::-1], v[::-1]
    out = base.astype(F32).copy()
    if order in ("forward", "reverse"):
        start = np.r_[0, np.nonzero(e[1:] != e[:-1])[0] + 1]
        rank = np.arange(e.size) - np.repeat(start, np.diff(np.r_[start, e.size]))
        for r in range(int(rank.max()) + 1 if e.size else 0):
            sel = rank == r
            out[e[sel]] = (out[e[sel]].astype(F64) + v[sel]).astype(F32)
        return out
    vals, keys, first = v, e, True
    while keys.size:
        start = np.r_[0, np.nonzero(keys[1:] != keys[:-1])[0] + 1]
        rank = np.arange(keys.size) - np.repeat(start, np.diff(np.r_[start, keys.size]))
        last = np.r_[keys[1:] != keys[:-1], True]
        single = (rank == 0) & last
        out[keys[single]] = (out[keys[single]].astype(F64) + vals[single]).astype(F32)
        a = (rank % 2 == 0) & ~last
        b = np.nonzero(a)[0] + 1
        odd_tail = (rank % 2 == 0) & last & ~single
        nv = (vals[a].astype(F64) + vals[b].astype(F64)).astype(F32) if first else (vals[a] + vals[b]).astype(F32)
        vals = np.concatenate((nv, vals[odd_tail].astype(F32) if not first else vals[odd_tail].astype(F32)))
        keys = np.concatenate((keys[a], keys[odd_tail]))
        o = np.argsort(keys, kind="stable")
        vals, keys, first = vals[o], keys[o], False
    return out


@pytest.mark.parametrize("name", ["edges", "collisions", "segments"])
@pytest.mark.parametrize("lerp", ["fused", "unfused"])
def test_bound_holds_for_legal_orders(name, lerp):
    """fp32 evaluations of every leaf (both lerp contractions, the 8-fma re-gather chain) summed forward from a nonzero
    base, in reverse, and pairwise stay within the per-entry bound, table and vector entries alike."""
    fa = _fa()
    inp = _set(name)
    worst = 0.0
    for k in range(4):
        for l in (0, 3, 9, 15):
            lt = SO.level_terms(fa, inp, k, l, lerp=lerp)
            for s in range(len(fa.tables)):
                sel = lt.seg == s
                size = int(fa.levels[s].size[l])
                base = SC.base_values((size, 2), 100 * s + 10 * k + l)
                ref = SO.Sums.zeros((size, 2))
                ref.add(lt.idx[sel].reshape(-1), *(a[sel].reshape(-1, 2) for a in (lt.t_val, lt.t_err, lt.t_mag, lt.t_nz)))
                vref = SO.Sums.zeros((4 * fa.vec_res * N_LEVELS, 2))
                vi = SO._vec_flat(fa.vec_res, E.VECTOR_OF_TERM[k], lt.vrow[sel], l).reshape(-1)
                vref.add(vi, *(a[sel].reshape(-1, 2) for a in (lt.v_val, lt.v_err, lt.v_mag, lt.v_nz)))
                for f in range(2):
                    ent, lv = lt.idx[sel].reshape(-1), lt.t_leaf[sel][..., f].reshape(-1)
                    vent, vlv = vi, lt.v_leaf[sel][..., f].reshape(-1)
                    for order in ("forward", "reverse", "pairwise"):
                        b = base[:, f] if order == "forward" else np.zeros(size, F32)
                        got = _ordered_sums(ent, lv, order, b)
                        bound = ref.bound(np.stack((b, b), 1))[:, f] if order == "forward" else ref.bound()[:, f]
                        r = SO.ratio(got, ref.val[:, f] + b.astype(F64), bound)
                        worst = max(worst, float(r.max()))
                        assert r.max() <= 1.0, (name, lerp, k, l, s, order, float(r.max()))
                        gv = _ordered_sums(vent, vlv, order, np.zeros(vref.val.shape[0], F32))
                        rv = SO.ratio(gv, vref.val[:, f], vref.bound()[:, f])
                        worst = max(worst, float(rv.max()))
                        assert rv.max() <= 1.0, (name, lerp, k, l, s, order, "vectors", float(rv.max()))
    print(f"{name} lerp={lerp}: worst error / bound of the fp32 orders {worst:.3f}")


@pytest.mark.parametrize("name", ["edges", "collisions", "segments"])
def test_walk_matches_plain_reference(name):
    """Routing every hot leaf through the restated walk (the run's slot entry, the run's tap row) gives the plain sum."""
    fa = _fa()
    inp = _set(name)
    a, b = SO.reference(fa, inp), SO.walk_sum(fa, inp)
    for s in range(len(fa.tables)):
        for k in range(4):
            for fld in ("val", "m"):
                x, y = getattr(a.tables[s][k], fld), getattr(b.tables[s][k], fld)
                assert np.allclose(x, y, rtol=1e-12, atol=0), (name, s, k, fld)
        assert np.allclose(a.vectors[s].val, b.vectors[s].val, rtol=1e-12, atol=0)
        assert (a.vectors[s].m == b.vectors[s].m).all()


# mutant -> (input set, feature source, grids, levels) of the GPU test's inputs where it shows
MUTANT_CASES = {
    "to_cell_unfused": ("edges", "egrid", range(4), range(N_LEVELS)),
    "scale_ulp_up": ("edges", "egrid", range(4), (E.MUTANT_SCALE_LEVEL,)),
    "parity_weight_swap": ("edges", "egrid", range(4), range(N_LEVELS)),
    "chunk_tail_unflushed": ("segments", "egrid", range(4), range(N_LEVELS)),
    "segment_change_misrouted": ("segments", "egrid", range(4), range(N_LEVELS)),
    "cold_as_hot": ("edges", "egrid", range(4), range(0, N_LEVELS, 5)),
    "vector_taps_swapped": ("edges", "egrid", range(4), range(0, N_LEVELS, 5)),
    "time_rows_keyed_by_row": ("segments", "egrid", (0,), range(N_LEVELS)),
    "regather_one_lane": ("edges", "gather", range(4), range(0, N_LEVELS, 5)),
    "past_live_scattered": ("live1023", "egrid", range(4), range(0, N_LEVELS, 5)),
}


def test_mutants_exceed_the_bound():
    assert set(MUTANT_CASES) == set(SO.MUTANTS)
    fa = _fa()
    lines = []
    for mutant, (name, mode, grids, levels) in MUTANT_CASES.items():
        inp = _set(name, egrid=mode == "egrid")
        key = ("faithful", name, mode, tuple(grids), tuple(levels))
        if key not in _CACHE:
            _CACHE[key] = SO.reference(fa, inp, grids=grids, levels=levels)
        good = _CACHE[key]
        bad = SO.reference(fa, inp, mutant=mutant, grids=grids, levels=levels)
        worst, where = 0.0, None
        for s in range(len(fa.tables)):
            for k in grids:
                r = SO.ratio(bad.tables[s][k].val, good.tables[s][k].val, good.tables[s][k].bound())
                if r.max() > worst:
                    worst, where = float(r.max()), f"segment {s} grid {k}"
            r = SO.ratio(bad.vectors[s].val, good.vectors[s].val, good.vectors[s].bound())
            if r.max() > worst:
                worst, where = float(r.max()), f"segment {s} vectors"
        lines.append(f"wrong reference '{mutant}' on set {name} ({mode}): worst error / bound {worst:.3g} at {where}")
        print(lines[-1])
    for mutant, line in zip(MUTANT_CASES, lines):
        assert float(line.split("bound ")[1].split(" ")[0]) >= 2.0, line
