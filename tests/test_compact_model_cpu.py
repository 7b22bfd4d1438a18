"""The 8-bit table format of the compact model on the CPU: the numpy quantiser (tests/quant_oracle.py) -- codes in
range, the zero slice, the clip-ratio argmin and its tie rule, the pairing of grids with vector axes -- and the int8
encode built on tests/encode_oracle.py against the float64 encode of the dequantised tables with unfolded vectors.
Every check is also run on the oracle's deliberately wrong formats (quant_oracle.MUTANTS) and must reject the one it
targets.  Last, the file reader's checks on malformed files."""
import numpy as np
import pytest
import torch

import encode_oracle as E
import quant_oracle as Q

F32 = np.float32


def _heavy(rng, n):
    """A trained-like slice: N(0, 0.05) with a Student-t tail and one outlier."""
    x = (rng.standard_t(3, n) * 0.05).astype(F32)
    x[rng.integers(0, n)] = F32(1.5)
    return x


# ------------------------------------------------------------------------------------------------ the quantiser
def _codes_in_range(mutant=None) -> bool:
    rng = np.random.default_rng(1)
    x = _heavy(rng, 4096)
    x[0] = -F32(np.max(np.abs(x)))            # -absmax: below -127 s for every c < 1
    absmax = F32(np.max(np.abs(x)))
    for c in Q.CLIP_RATIOS:
        q = Q.codes_of(x, Q.scale_of(c, absmax), mutant)
        if q.min() < -127 or q.max() > 127:
            return False
    return True


def _half_to_even(mutant=None) -> bool:
    s = Q.scale_of(F32(1), F32(127) * F32(2.0 ** -10))    # exactly 2^-10
    assert s == F32(2.0 ** -10)
    x = np.array([2.5, -2.5, 0.5, 3.5], F32) * s          # x / s lands on the halves exactly
    return Q.codes_of(x, s, mutant).tolist() == [2, -2, 0, 4]


def _zero_slice(mutant=None) -> bool:
    _, scales, errs = Q.slice_errors(np.zeros(100, F32))
    ci = Q.choose(errs, mutant)
    return bool((scales == 0).all() and ci == 0 and (Q.codes_of(np.zeros(100, F32), scales[ci]) == 0).all())


def _argmin(mutant=None) -> bool:
    x = _heavy(np.random.default_rng(2), 1 << 18)   # a hashed level of a 50-frame segment
    absmax, scales, errs = Q.slice_errors(x)
    ci = Q.choose(errs, mutant)
    brute = [float(np.sum((x.astype(np.float64) - np.float64(s) * Q.codes_of(x, s).astype(np.float64)) ** 2))
             for s in scales]
    return ci == int(np.argmin(brute)) and ci > 0 and Q.decided(errs)


@pytest.mark.parametrize("check,mutant", [(_codes_in_range, "allow_m128"), (_half_to_even, "half_away"),
                                          (_zero_slice, "ties_smaller"), (_argmin, None)])
def test_quantiser(check, mutant):
    assert check(None)
    if mutant is not None:
        assert not check(mutant), f"{check.__name__} does not reject {mutant}"


def test_clip_ratio_helps_heavy_tails():
    """The outlier is what c < 1 is for: the chosen ratio's error is well below c = 1's (0.54 x here)."""
    x = _heavy(np.random.default_rng(3), 1 << 18)
    _, _, errs = Q.slice_errors(x)
    ci = Q.choose(errs)
    print(f"c = {Q.CLIP_RATIOS[ci]}, error {errs[ci]:.4g} against {errs[0]:.4g} at c = 1")
    assert errs[ci] < 0.75 * errs[0]


def test_scale_and_code_roundings():
    """s = (c * absmax) / 127 in two fp32 roundings, q = rint(x / s) in fp32: not a float64 shortcut."""
    rng = np.random.default_rng(4)
    a = (rng.random(2000) * 3).astype(F32)
    for c in Q.CLIP_RATIOS:
        s = np.array([Q.scale_of(c, v) for v in a], F32)
        assert (s == (F32(c) * a) / F32(127)).all()
    x = rng.standard_normal(5000).astype(F32)
    s = Q.scale_of(F32(0.7), F32(np.max(np.abs(x))))
    assert (Q.codes_of(x, s) == np.clip(np.rint(x / s), -127, 127)).all()


# ------------------------------------------------------------------------------------------------ fold + encode
@pytest.fixture(scope="module")
def segment():
    """A (6,) segment: master tables with heavy tails, vectors, its level table, and points over its frames."""
    rng = np.random.default_rng(5)
    lt = E.level_table(E.segment_log2_hashmap_size(6))
    grids = [np.concatenate([_heavy(rng, 2 * int(lt.size[l])) for l in range(16)]) for _ in range(4)]
    vectors = (rng.standard_normal((4, 2048, 32)) * 0.1).astype(F32)
    frames = tuple(range(15, 21))
    n = 400
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(F32)
    fr = np.array(frames)[rng.integers(0, 6, n)]
    return lt, grids, vectors, frames, x, fr


def _fold_pairing(mutant=None) -> bool:
    rng = np.random.default_rng(6)
    v = rng.standard_normal((4, 8, 32)).astype(F32)
    scales = rng.random((4, 16, 2)).astype(F32)
    f = Q.fold_vectors(v, scales, mutant)
    return all((f[E.VECTOR_OF_TERM[k]] == v[E.VECTOR_OF_TERM[k]] * scales[k].reshape(1, 32)).all() for k in range(4))


def _encode_matches_dequantised(segment, mutant=None) -> bool:
    """The int8 encode (bf16 tables holding the codes, folded vectors) against the float64 encode of s * q with the
    unfolded vectors: every composed feature within its bf16 rounding plus the fp32 rounding of the sums."""
    lt, grids, vectors, frames, x, fr = segment
    scales, _, _, codes, folded = Q.quantize_segment(grids, vectors, lt, mutant)
    if mutant == "allow_m128":
        codes = [c.astype(np.int8) for c in codes]
    fa = Q.int8_field([codes], [folded], frames, (6,))
    enc = E.encode(fa, x, fr)
    _, t = E.segment_and_time(fa, fr)
    ref = Q.dequantised_encode(codes, scales, vectors, lt, x, t)
    mag = Q.dequantised_encode(codes, scales, vectors, lt, x, t, absolute=True)
    got = E.bf16_to_f32(enc.feat).astype(np.float64)
    tol = 2.0 ** -8 * np.abs(ref) + 2.0 ** -18 * mag + 1e-30    # bf16 half ulp + fp32 sums (few ulps of the terms)
    worst = float(np.max(np.abs(got - ref) / tol))
    print(f"mutant {mutant}: worst |int8 - dequantised| / bound = {worst:.3f}")
    return worst <= 1.0


def test_fold_pairing():
    assert _fold_pairing(None)
    assert not _fold_pairing("wrong_axis")


def test_int8_encode_is_the_dequantised_encode(segment):
    assert _encode_matches_dequantised(segment)


@pytest.mark.parametrize("mutant", ["wrong_axis", "not_folded"])
def test_int8_encode_rejects(segment, mutant):
    assert not _encode_matches_dequantised(segment, mutant)


def test_grid_quantiser_layout(segment):
    """quantize_grid walks every level's slice: each slice's codes reproduce from its own scale alone."""
    lt, grids, *_ = segment
    scale, clip, errs, codes = Q.quantize_grid(grids[0], lt)
    t = grids[0].reshape(-1, 2)
    for l in range(16):
        a, b = int(lt.offset[l]), int(lt.offset[l] + lt.size[l])
        for f in range(2):
            assert (codes[a:b, f] == Q.codes_of(t[a:b, f], scale[l, f])).all()
            assert scale[l, f] == Q.scale_of(Q.CLIP_RATIOS[clip[l, f]], np.max(np.abs(t[a:b, f])))
    assert codes.min() >= -127


# ------------------------------------------------------------------------------------------------ the file reader
def _payload(segment):
    from humanrf_b200.scene_representation.grid_layout import MLP_BLOB_ELEMS
    from humanrf_b200.toolbox import compact_model as CM

    lt, grids, vectors, frames, *_ = segment
    scales, clip, errs, codes, folded = Q.quantize_segment(grids, vectors, lt)
    f2s, f2t = E.frame_luts(frames, (6,))
    return dict(format=CM.FORMAT_TAG, version=CM.FORMAT_VERSION,
                config=dict(density_scale=100.0, sorted_frame_numbers=frames, segment_sizes=(6,), log2_hashmap_size=19,
                            coarsest_resolution=32, finest_resolution=2048, camera_embedding_dim=0),
                codes=[[torch.from_numpy(c) for c in codes]], scales=torch.from_numpy(scales[None]),
                vectors=[torch.from_numpy(folded)], mlp_blob=torch.zeros(MLP_BLOB_ELEMS, dtype=torch.bfloat16),
                frame_to_segment=torch.from_numpy(f2s), frame_to_tlocal=torch.from_numpy(f2t), camera_embeddings=None,
                clip=torch.from_numpy(clip[None]), rms=torch.zeros((1, 4, 16, 2)))


def _malformed(p, how):
    if how == "version":
        p["version"] = 99
    elif how == "table_length":
        p["codes"][0][2] = p["codes"][0][2][:-8]
    elif how == "dtype":
        p["codes"][0][1] = p["codes"][0][1].to(torch.int16)
    elif how == "scale_nan":
        p["scales"][0, 1, 3, 0] = float("nan")
    elif how == "code_m128":
        p["codes"][0][0][5, 1] = -128
    elif how == "lut":
        p["frame_to_segment"] = p["frame_to_segment"][:-1]
    return p


@pytest.mark.parametrize("how", ["version", "table_length", "dtype", "scale_nan", "code_m128", "lut", "truncated"])
def test_reader_refuses_malformed_files(tmp_path, segment, how):
    from humanrf_b200.toolbox.compact_model import CompactHumanRF, _validate

    _validate(_payload(segment))                       # the well-formed payload passes
    path = tmp_path / "m.pt"
    if how == "truncated":
        torch.save(_payload(segment), path)
        path.write_bytes(path.read_bytes()[: path.stat().st_size // 2])
    else:
        torch.save(_malformed(_payload(segment), how), path)
    with pytest.raises(ValueError) as e:
        CompactHumanRF.load(path, "cpu")
    print(how, "->", e.value)
