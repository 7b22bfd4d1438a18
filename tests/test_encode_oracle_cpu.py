"""Checks of the rounding-faithful encode reference (tests/encode_oracle.py) itself: its fused multiply-add against exact
rational arithmetic, its bf16 rounding, its level table against the product's GridLayout, its agreement with
oracle/hashgrid.py, its edge set, and that each deliberately wrong reference it offers is told apart on that edge set."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import encode_oracle as E
from humanrf_b200.scene_representation.grid_layout import GridLayout, segment_log2_hashmap_size
from oracle import hashgrid
from oracle import sampler as OS


def _round_f32(x: Fraction) -> np.float32:
    """Round a rational to the nearest fp32, ties to even, with subnormals (no overflow)."""
    if x == 0:
        return np.float32(0.0)
    sign, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)
    ulp = Fraction(2) ** (e - 23)
    q, r = divmod(a / ulp, 1)
    q = int(q)
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and q & 1):
        q += 1
    return np.float32(sign * float(q * ulp))


def _exact(a, b, c):
    return np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)],
                    np.float32)


def _naive(a, b, c):
    """The double rounding the exact fma replaces: float64 sum, then float32."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def test_fma32_matches_exact_rationals_on_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    c[::3] = (-a[::3].astype(np.float64) * b[::3]).astype(np.float32)       # heavy cancellation
    got, want = E.fma32(a, b, c), _exact(a, b, c)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    assert (OS.fma32(a, b, c).view(np.uint32) == want.view(np.uint32)).all()   # the sampler oracle's round-to-odd form


def test_fma32_decides_double_rounding_cases_and_subnormals():
    # a*b = 2^-24 + 2^-60: 1 + a*b rounds in float64 onto the fp32 midpoint 1 + 2^-24 and a second rounding ties to 1.0,
    # but the exact sum lies above the midpoint: 1 + 2^-23.  Mirrored, scaled, and with the tail on the other side.
    a = np.float32(1 + 2.0 ** -12)
    b = np.float32((2.0 ** 24 - 4095) * 2.0 ** -48)
    assert Fraction(float(a)) * Fraction(float(b)) == Fraction(2) ** -24 + Fraction(2) ** -60
    A = np.array([a, -a, a, a, a * np.float32(2 ** 20)], np.float32)
    B = np.array([b, b, -b, b, b], np.float32)
    C = np.array([1.0, -1.0, np.float32(1 + 2.0 ** -22), 3.0, np.float32(2 ** 20)], np.float32)
    want = _exact(A, B, C)
    got = E.fma32(A, B, C)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    assert (_naive(A, B, C) != want).any(), "the constructed cases must defeat the double rounding"
    # subnormal results, and subnormal inputs
    rng = np.random.default_rng(1)
    n = 2000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-80, -60, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-80, -60, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-149, -126, n)).astype(np.float32)
    want = _exact(a, b, c)
    assert (np.abs(want) < np.finfo(np.float32).tiny).mean() > 0.5
    assert (E.fma32(a, b, c).view(np.uint32) == want.view(np.uint32)).all()


def test_bf16_round_to_nearest_even_ties():
    bits = np.array([0x3F808000, 0x3F818000, 0x3F808001, 0x3F807FFF, 0xBF808000, 0xBF818000, 0x00008000, 0x00018000,
                     0x7F7F8000, 0x00000000, 0x80000000], np.uint32)
    x = bits.view(np.float32)
    want = np.array([0x3F80, 0x3F82, 0x3F81, 0x3F80, 0xBF80, 0xBF82, 0x0000, 0x0002, 0x7F80, 0x0000, 0x8000], np.uint16)
    assert (E.bf16_bits(x) == want).all()
    assert (E.bf16_bits(x) == torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)).all()
    rng = np.random.default_rng(2)
    r = rng.integers(0, 2 ** 32, 100000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    r = r[np.isfinite(r)]
    assert (E.bf16_bits(r) == torch.from_numpy(r).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)).all()
    assert (E.bf16_bits(np.float32(1 + 2.0 ** -8 + 2.0 ** -9), truncate=True) == 0x3F80)


@pytest.mark.parametrize("log2T", [14, 15, 16, 17, 18, 19])
def test_level_table_matches_grid_layout(log2T):
    lt, lay = E.level_table(log2T), GridLayout(log2T)
    assert (lt.scale.view(np.uint32) == lay.scale.view(np.uint32)).all()
    assert (lt.res == lay.res).all() and (lt.offset == lay.offset).all() and (lt.size == lay.size).all()
    assert sum(1 << l for l in range(16) if lt.hashed[l]) == lay.hashed_mask and lt.n_entries == lay.n_entries


@pytest.mark.parametrize("segment_size", [6, 12, 25, 50, 100])
def test_segment_log2_and_dense_sizes(segment_size):
    l2 = E.segment_log2_hashmap_size(segment_size)
    assert l2 == segment_log2_hashmap_size(segment_size, 19)
    lt = E.level_table(l2)
    dense = [int(lt.size[l]) for l in range(16) if not lt.hashed[l]]
    assert dense[0] == 32768
    if segment_size >= 50:      # the non-power-of-two dense levels of the baseline sizes (test_baseline_sizes_gpu.py)
        assert dense[:3] == [32768, 79512, 175616]
        assert (segment_size == 100) == (len(dense) == 4 and dense[3] == 405224)


def test_frame_rule_matches_the_product_luts():
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    frames = tuple(range(15, 15 + 18))
    m = HumanRF(sorted_frame_numbers=frames, segment_sizes=(6, 12), **MODEL_KW)
    f2s, f2t = E.frame_luts(frames, (6, 12))
    assert (f2s == m.frame_numbers_to_segment_numbers.numpy()).all()
    assert (f2t.view(np.uint32) == m.frame_numbers_to_normalized_local_frame_numbers.numpy().view(np.uint32)).all()


def _small_field(rng, wide=False, segs=(6,)):
    frames = tuple(range(15, 15 + sum(segs)))
    grids, vecs = [], []
    for s in segs:
        lt = E.level_table(E.segment_log2_hashmap_size(s))
        g = [(rng.standard_normal(2 * lt.n_entries) * 6).astype(np.float32) for _ in range(4)]
        v = (rng.standard_normal((4, 2048, 32)) * 0.1).astype(np.float32)
        if wide:
            g = [_widen(x, rng) for x in g]
            v = _widen(v, rng)
        grids.append(g)
        vecs.append(v)
    return E.field_from_fp32(grids, vecs, frames, segs), frames


def _widen(x, rng):
    y = (np.abs(x) * 2.0 ** rng.uniform(-24, 8, x.shape) * np.where(rng.random(x.shape) < 0.5, -1, 1)).astype(np.float32)
    y[rng.random(x.shape) < 0.05] = 0
    return y


def test_agrees_with_hashgrid_oracle():
    """Cell, corner indices and weights of oracle/hashgrid.py equal the reference's bit for bit on the edge set (exact
    fma in both); its unfused blend lies within an fp32 accumulation bound of the fused chain."""
    rng = np.random.default_rng(3)
    fa, frames = _small_field(rng)
    lt = fa.levels[0]
    p = E.edge_positions([lt], 3000, rng, outside=0.0)
    x, _ = E.load_query(p, np.full(p.shape[0], frames[0]))
    for l in range(16):
        idx, w = hashgrid.corner_indices_and_weights(x, lt.scale[l], int(lt.res[l]), int(lt.size[l]), bool(lt.hashed[l]))
        cells = [E.to_cell(lt.scale[l], x[:, d]) for d in range(3)]
        for k in range(8):
            assert (idx[:, k] == E.corner_index(k, bool(lt.hashed[l]), int(lt.res[l]), int(lt.size[l]),
                                                *[c[0] for c in cells])).all(), (l, k)
            wd = [(E.fsub(np.float32(1), c[1]), c[1]) for c in cells]
            wk = E.fmul(E.fmul(wd[0][k & 1], wd[1][(k >> 1) & 1]), wd[2][(k >> 2) & 1])
            assert (w[:, k].view(np.uint32) == wk.view(np.uint32)).all(), (l, k)
    tab = torch.from_numpy(E.bf16_to_f32(fa.tables[0][0]).astype(np.float32))
    ref = hashgrid.encode(tab, torch.from_numpy(x), fa.log2T[0]).numpy().reshape(-1, 16, 2)
    enc = E.encode(fa, x, np.full(x.shape[0], frames[0]))
    eg = enc.egrid[0::4]                                           # grid 0 (xyz), [16, N]
    got = np.stack((E.bf16_to_f32((eg & 0xFFFF).astype(np.uint16)), E.bf16_to_f32((eg >> 16).astype(np.uint16))), axis=2)
    got = got.transpose(1, 0, 2)
    bound = 2.0 ** -8 * np.abs(ref) + 8 * 2.0 ** -24 * np.abs(E.bf16_to_f32(fa.tables[0][0])).max()
    assert (np.abs(got - ref) <= bound).all()


def test_edge_set_reaches_every_boundary():
    rng = np.random.default_rng(4)
    lts = [E.level_table(l2) for l2 in (15, 19)]
    for lt in lts:
        e = E.level_edges(lt, rng)
        for l in range(16):
            exact, below = 0, 0
            p = E.fma32(lt.scale[l], e, np.float32(0.5))
            on = p == np.floor(p)
            exact_prod = [Fraction(float(lt.scale[l])) * Fraction(float(v)) + Fraction(1, 2) for v in e[on]]
            exact = sum(1 for q in exact_prod if q.denominator == 1)
            below = sum(1 for q, v in zip(exact_prod, p[on]) if q < Fraction(float(v)))
            assert on.sum() >= 4 and below + exact >= 1, (l, int(on.sum()), exact, below)
    p = E.edge_positions(lts, 4000, rng)
    x, _ = E.load_query(p, np.zeros(p.shape[0], np.int64))
    assert ((x < -1) & (x >= -4)).any() and ((x > 2) & (x <= 4)).any()
    assert (x == 0).any() and (x == 1).any() and (x == np.float32(2.0 ** -25)).any()
    i0, i1, _ = E.row_tap(x[:, 0], 2048)
    assert (i0 == 0).any() and (i1 == 0).any() and (i0 == 2047).any() and (i1 == 2047).any()


@pytest.mark.parametrize("mutant", E.MUTANTS)
def test_every_mutant_is_told_apart_on_the_edge_set(mutant):
    """The comparators, run with each deliberately wrong reference on the correct reference's own output (variant 0),
    report at least one mismatch: the edge set reaches the boundary each mutant moves."""
    rng = np.random.default_rng(5)
    fa, frames = _small_field(rng, wide=True, segs=(6, 12))
    n = 3000
    p = E.edge_positions(fa.levels, n, rng)
    fr = np.array(list(frames) * (n // len(frames) + 1))[:n]
    x, fr = E.load_query(p, fr)
    good = E.encode(fa, x, fr, feat_gpu=E.encode(fa, x, fr).feat)
    assert good.check["mismatch"] == 0
    bad = E.encode(fa, x, fr, feat_gpu=good.feat, mutant=mutant)
    eg = E.egrid_mismatch(bad, good.egrid)
    print(f"{mutant}: egrid words differing {eg['words']} of {eg['checked']}, composed outputs outside the candidate set "
          f"{bad.check['mismatch']} of {bad.check['outputs']}")
    assert eg["words"] + bad.check["mismatch"] > 0
