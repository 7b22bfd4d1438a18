"""LPIPS pieces that need no GPU: the fp32 input scaling against torch, the tf32 rounding helper, the float64 oracle
against torchvision's module, the 31-pixel rule, the weight loader's checks, the tables' LPIPS column, and that
deliberately wrong oracles fail the end-to-end bar of test_lpips_gpu.py."""
import csv
import math

import numpy as np
import pytest
import torch

from lpips_oracle import PAIR_KINDS, SCALE, SHIFT, Oracle, make_pair, rna_tf32, scale_input, seeded_state_dicts

REL_BAR, ABS_FLOOR = 5e-3, 1e-6      # test_lpips_gpu.py's end-to-end bar


@pytest.fixture(scope="module")
def state():
    return seeded_state_dicts(0)


def test_input_scaling_matches_torch_bit_for_bit():
    # every uint8 value in every channel, as evaluate.py (u8 / 255.0 on the CPU) and lpips (2x - 1, ScalingLayer) do it
    img = np.stack([np.roll(np.arange(256, dtype=np.uint8), 85 * c) for c in range(3)], -1)[None]    # [1,256,3]
    t = torch.from_numpy(img).permute(2, 0, 1) / 255.0
    t = t * 2 - 1
    ref = (t - torch.tensor(SHIFT)[:, None, None]) / torch.tensor(SCALE)[:, None, None]
    assert ref.dtype == torch.float32
    assert np.array_equal(scale_input(img).view(np.uint32), ref.numpy().view(np.uint32))
    # float32 input: v is taken as given
    f = np.random.default_rng(0).random((5, 7, 3), dtype=np.float32)
    t = torch.from_numpy(f).permute(2, 0, 1) * 2 - 1
    ref = (t - torch.tensor(SHIFT)[:, None, None]) / torch.tensor(SCALE)[:, None, None]
    assert np.array_equal(scale_input(f).view(np.uint32), ref.numpy().view(np.uint32))


def test_rna_tf32_helper():
    bits = np.array([0x3F800000, 0x3F801000, 0x3F800FFF, 0x3F801001, 0x3F802000 | 0x1000, 0x3F803FFF,
                     0x7F7FFFFF, 0x7F7FE000, 0x7F7FEFFF, 0x7F7FF000, 0x00000FFF, 0x00001000, 0x7F800000, 0x7FC00000],
                    np.uint32)
    want = np.array([0x3F800000, 0x3F802000, 0x3F800000, 0x3F802000, 0x3F804000, 0x3F804000,
                     0x7F800000, 0x7F7FE000, 0x7F7FE000, 0x7F800000, 0x00000000, 0x00002000, 0x7F800000, 0x7FC00000],
                    np.uint32)
    for sign in (0, 0x80000000):
        x = (bits | np.uint32(sign)).view(np.float32)
        w = want | np.uint32(sign)
        got = rna_tf32(x).view(np.uint32)
        nan = np.isnan(x)
        assert np.array_equal(got[~nan], w[~nan]) and np.isnan(got.view(np.float32)[nan]).all()
        assert np.array_equal(rna_tf32(torch.from_numpy(x)).numpy().view(np.uint32)[~nan], got[~nan])
    # random values: tf32-valued, within half a tf32 ulp, ties away from zero
    x = np.random.default_rng(1).standard_normal(100000).astype(np.float32) * np.float32(1e3)
    r = rna_tf32(x)
    assert not (r.view(np.uint32) & 0x1FFF).any()
    ulp = np.ldexp(1.0, np.frexp(np.abs(x).astype(np.float64))[1] - 11)
    assert (np.abs(r.astype(np.float64) - x) <= ulp / 2).all()


def test_oracle_equals_torchvision_layer_by_layer(state):
    o = Oracle(*state)
    x = o.prepare(make_pair("noise", 67, 45)[0])
    with torch.no_grad():
        for a, b in zip(o.trunk(x), o.trunk_torchvision(x)):
            assert a.shape == b.shape and torch.equal(a, b)


def test_31_pixel_rule(state):
    o = Oracle(*state)
    for w, h in ((31, 31), (31, 40), (40, 31)):
        pred, gt = make_pair("noise", w, h)
        assert math.isfinite(o(pred, gt))
        with torch.no_grad():
            o.trunk_torchvision(o.prepare(pred))
    for w, h in ((30, 40), (40, 30)):
        pred, gt = make_pair("noise", w, h)
        assert math.isnan(o(pred, gt))
        with pytest.raises(RuntimeError), torch.no_grad():
            o.trunk_torchvision(o.prepare(pred))
    pred, gt = make_pair("noise", 64, 64)
    assert math.isnan(o(pred, gt, (0, 0, 0, 0))) and math.isnan(o(pred, gt, (3, 3, 30, 50)))


def test_loader_rejects_missing_keys_and_wrong_shapes(state, tmp_path):
    from humanrf_b200.toolbox.lpips import load_lpips_alex, lpips_alex_from_state_dicts

    alex, lin = state
    cases = []
    a = dict(alex)
    del a["features.8.bias"]
    cases.append((a, lin, "features.8.bias"))
    a = dict(alex)
    a["features.3.weight"] = a["features.3.weight"][:, :63]
    cases.append((a, lin, "features.3.weight"))
    a = dict(alex)
    a["features.0.weight"] = a["features.0.weight"].permute(0, 2, 3, 1)        # OHWI instead of OIHW
    cases.append((a, lin, "features.0.weight"))
    li = dict(lin)
    del li["lin4.model.1.weight"]
    cases.append((alex, li, "lin4.model.1.weight"))
    li = dict(lin)
    li["lin2.model.1.weight"] = li["lin2.model.1.weight"].reshape(384)
    cases.append((alex, li, "lin2.model.1.weight"))
    li = dict(lin)
    li["lin3.model.1.weight"], li["lin4.model.1.weight"] = li["lin4.model.1.weight"], li["lin3.model.1.weight"][:, :255]
    cases.append((alex, li, "lin4.model.1.weight"))
    for i, (a, li, key) in enumerate(cases):
        with pytest.raises(RuntimeError, match=key.replace(".", r"\.")):
            lpips_alex_from_state_dicts(a, li, "cuda")
        # and through the files, as torch.save writes them
        torch.save(a, tmp_path / f"alex{i}.pth")
        torch.save(li, tmp_path / f"lin{i}.pth")
        with pytest.raises(RuntimeError, match=key.replace(".", r"\.")):
            load_lpips_alex(tmp_path / f"alex{i}.pth", tmp_path / f"lin{i}.pth", "cuda")


def test_tables_with_lpips_follow_evaluate_py(tmp_path):
    from humanrf_b200.toolbox.evaluation import ViewScore, write_metric_tables

    scores = [ViewScore(0, 15, 30.5, 0.91, (1, 2, 40, 50), 0.125), ViewScore(2, 16, 28.0, 0.85, (0, 0, 64, 48), 0.25)]
    write_metric_tables(tmp_path / "a", scores)
    rows = list(csv.reader(open(tmp_path / "a" / "metrics.csv", newline="")))
    assert rows == [["camera", "frame", "PSNR", "LPIPS", "SSIM"], ["1", "15", "30.5", "0.125", "0.91"],
                    ["3", "16", "28.0", "0.25", "0.85"]]
    avg = list(csv.reader(open(tmp_path / "a" / "averages.csv", newline="")))
    assert avg[0] == ["PSNR", "LPIPS", "SSIM"] and [float(v) for v in avg[1]] == [29.25, 0.1875, 0.88]
    # without LPIPS nothing changes
    write_metric_tables(tmp_path / "b", [ViewScore(0, 15, 30.5, 0.91, (1, 2, 40, 50))])
    assert list(csv.reader(open(tmp_path / "b" / "metrics.csv", newline="")))[0] == ["camera", "frame", "PSNR", "SSIM"]
    assert list(csv.reader(open(tmp_path / "b" / "averages.csv", newline="")))[0] == ["PSNR", "SSIM"]


# the GPU test's end-to-end pairs at the sizes a CPU runs quickly
CPU_PAIRS = [((31, 31), k) for k in PAIR_KINDS] + [((32, 47), k) for k in PAIR_KINDS]


def _bgr(o, pred, gt, roi=None):
    return Oracle.__call__(o, np.ascontiguousarray(np.asarray(pred)[..., ::-1]),
                           np.ascontiguousarray(np.asarray(gt)[..., ::-1]), roi)


@pytest.mark.parametrize("variant", ["bgr", "conv1_pad1", "lin34_swapped"])
def test_wrong_oracles_fail_the_end_to_end_bar(state, variant):
    good = Oracle(*state)
    bad = Oracle(*state)
    if variant == "conv1_pad1":
        bad.specs[0] = (4, 1)
    elif variant == "lin34_swapped":
        bad.lin[3], bad.lin[4] = bad.lin[4], bad.lin[3]
    fails = []
    for (W, H), kind in CPU_PAIRS:
        pred, gt = make_pair(kind, W, H, seed=W + H)
        ref = good(pred, gt)
        try:
            got = _bgr(bad, pred, gt) if variant == "bgr" else bad(pred, gt)
        except RuntimeError:        # conv1 padding 1 leaves pool2 empty at 31 pixels: no value at all
            got = float("nan")
        fails.append(not abs(got - ref) <= REL_BAR * ref + ABS_FLOOR)
    assert all(fails), [p for p, f in zip(CPU_PAIRS, fails) if not f]
