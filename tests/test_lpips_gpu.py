"""LPIPS on the H100 (csrc/lpips.cu, hrf_lpips, toolbox/lpips.py), with seeded random weights in the real file formats:
each stored layer against a float64 convolution of the kernel's own stored input, the tail against a float64
recomputation from the stored layers, the whole score against the float64 oracle of tests/lpips_oracle.py, the ROI and
NaN rules, input types, identities, determinism, graph capture, and evaluate_sequence's LPIPS column."""
import csv
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lpips_oracle import CONV_KEYS, CONV_SPECS, PAIR_KINDS, Oracle, make_pair, rna_tf32, scale_input, seeded_state_dicts

pytestmark = pytest.mark.gpu

# End-to-end bar against the unrounded float64 oracle: |kernel - oracle| <= REL_BAR * oracle + ABS_FLOOR.  Rounding
# every conv operand to tf32 (2^-11 relative) perturbs each layer's features by up to ~1e-3 relative of their size, and
# LPIPS is a squared difference of the two images' features, so the error scales with the features while the score
# scales with their difference: relative to the score it is largest where the images nearly agree.  On an H100 the
# pairs with LPIPS above 1e-3 stay within 2.4e-3 relative; the quantisation-only pairs (LPIPS 2e-5 to 8e-5, whose
# feature difference sits near the tf32 rounding scale) differ by up to 5e-7 absolute, 1.2e-2 relative on the smallest
# images, where the deep layers are 1 or 2 pixels.  ABS_FLOOR = 1e-6 is three orders below the precision LPIPS is
# reported at; every deliberately wrong oracle of test_lpips_cpu.py still fails the bar on every pair.
REL_BAR, ABS_FLOOR = 5e-3, 1e-6
U = 2.0 ** -24
WORST = []


@pytest.fixture(scope="module")
def weights(cuda, tmp_path_factory):
    from humanrf_b200.toolbox.lpips import load_lpips_alex

    alex, lin = seeded_state_dicts(0)
    d = tmp_path_factory.mktemp("lpips_weights")
    torch.save(alex, d / "alexnet-owt-7be5be79.pth")
    torch.save(lin, d / "alex.pth")
    return alex, lin, load_lpips_alex(d / "alexnet-owt-7be5be79.pth", d / "alex.pth", cuda)


@pytest.fixture(scope="module")
def oracle(weights, cuda):
    alex, lin, _ = weights
    return Oracle(alex, lin, device=cuda)


def _ellipse_roi(W, H, fx=0.35, fy=0.42):
    """Bounding box of eval_bench.py's centred ellipse mask (2878 x 2526 at 4112 x 3008)."""
    y, x = np.mgrid[0:H, 0:W]
    m = ((x + 0.5 - W / 2) / (fx * W)) ** 2 + ((y + 0.5 - H / 2) / (fy * H)) ** 2 <= 1
    ys, xs = np.nonzero(m)
    return (int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1))


def _dev(img, cuda):
    return torch.from_numpy(np.ascontiguousarray(img)).to(cuda)


def _roi_t(roi, cuda):
    return None if roi is None else torch.tensor(roi, dtype=torch.int32, device=cuda)


def _run(pred, gt, w, cuda, roi=None, keep=False):
    from humanrf_b200.toolbox.lpips import lpips, workspace_bytes

    H, W = pred.shape[:2]
    ws = torch.empty(workspace_bytes(W, H), dtype=torch.uint8, device=cuda) if keep else None
    out = lpips(_dev(pred, cuda), _dev(gt, cuda), w, roi=_roi_t(roi, cuda), workspace=ws)
    return float(out.item()), ws


# ---- per layer --------------------------------------------------------------------------------------------------------
def _conv_check(x, y, w, b, stride, pad, n_sample, seed):
    """Largest |error| / bound of the stored conv output y [2,ho,wo,Co] against relu(conv(x) + b) in float64 from the
    stored input x [2,hi,wi,Ci] and the tf32 weights w [Co,Ci',KS,KS], at every output pixel or a seeded sample of
    n_sample.  Bound: the fp32 any-order
    accumulation bound (n + 1) 2^-23 (sum |a w| + |b|) for the pre-activation, then one tf32 rounding (2^-11 relative)."""
    ks, ci = w.shape[2], w.shape[1]
    _, ho, wo, co = y.shape
    total = 2 * ho * wo
    g = torch.Generator(device="cpu").manual_seed(seed)
    idx = torch.arange(total) if total <= n_sample else torch.randperm(total, generator=g)[:n_sample]
    idx = idx.to(x.device)
    img, oy, ox = idx // (ho * wo), (idx // wo) % ho, idx % wo
    xp = F.pad(x[..., :ci].double(), (0, 0, pad, pad, pad, pad))
    k = torch.arange(ks, device=x.device)
    iy = (oy * stride)[:, None] + k[None]
    ix = (ox * stride)[:, None] + k[None]
    wt = w.double().permute(0, 2, 3, 1)                              # [Co, KS, KS, Ci]
    got = y.reshape(-1, co)[idx].double()
    worst = 0.0
    for c0 in range(0, len(idx), 4096):
        sl = slice(c0, c0 + 4096)
        patch = xp[img[sl, None, None], iy[sl, :, None], ix[sl, None, :]]   # [n, KS, KS, Ci]
        pre = torch.einsum("nyxc,oyxc->no", patch, wt) + b.double()
        mag = torch.einsum("nyxc,oyxc->no", patch.abs(), wt.abs()) + b.double().abs()
        ref = torch.relu(pre)
        e = (ks * ks * ci + 1) * 2.0 ** -23 * mag
        bound = e + 2.0 ** -11 * (ref + e) + 1e-30
        err = (got[sl] - ref).abs()
        assert bool((err <= bound).all()), f"conv: max excess {float((err - bound).max()):.3e}"
        worst = max(worst, float((err / bound).max()))
    return worst


def _tail_reference(t, lin):
    """LPIPS from the stored layers in float64, and a bound on the kernel's fp32 tail error (per pixel: the channel sums
    (C + 1) u relative, the norm (C/2 + 4) u, the difference, square, lin product and channel sum, u = 2^-24)."""
    total, bound = 0.0, 0.0
    for k, name in enumerate(("conv1", "conv2", "conv3", "conv4", "conv5")):
        a, b = t[name][0].double(), t[name][1].double()
        C = a.shape[-1]
        na = a / (torch.sqrt((a * a).sum(-1, keepdim=True)) + 1e-10)
        nb = b / (torch.sqrt((b * b).sum(-1, keepdim=True)) + 1e-10)
        e = na - nb
        lw = lin[k].double()
        total += float((lw * e * e).sum(-1).mean())
        de = (C / 2 + 4) * U * (na.abs() + nb.abs()) + U * e.abs()
        ep = (lw * (2 * e.abs() * de + de * de + U * e * e)).sum(-1) + (C + 2) * U * (lw * e * e).sum(-1)
        bound += float(ep.mean())
    return total, bound + 1e-12 * abs(total)


LAYER_CASES = [((32, 47), "noise", None), ((752, 1028), "unrelated", (1, 6, 513, 700)),
               ((1028, 752), "saturated", None), ((4112, 3008), "noise", "ellipse")]


@pytest.mark.parametrize("size,kind,roi", LAYER_CASES, ids=[f"{s[0]}x{s[1]}-{k}" for s, k, _ in LAYER_CASES])
def test_layers_and_tail_match_float64(cuda, weights, size, kind, roi):
    from humanrf_b200.toolbox.lpips import workspace_tensors

    alex, lin, w = weights
    W, H = size
    if roi == "ellipse":
        roi = _ellipse_roi(W, H)
    pred, gt = make_pair(kind, W, H, seed=W)
    got, ws = _run(pred, gt, w, cuda, roi, keep=True)
    rw, rh = (W, H) if roi is None else roi[2:]
    t = workspace_tensors(ws, W, H, rw, rh)
    # input: the fp32 scaling of step 1, rounded to tf32, bit for bit; the 4th channel is zero
    x0, y0 = (0, 0) if roi is None else roi[:2]
    for i, img in enumerate((pred, gt)):
        ref = rna_tf32(scale_input(img[y0:y0 + rh, x0:x0 + rw])).transpose(1, 2, 0)
        assert np.array_equal(t["input"][i, ..., :3].cpu().numpy(), ref)
    assert not t["input"][..., 3].any()
    # every stored activation is tf32-valued
    for name in ("conv1", "pool1", "conv2", "pool2", "conv3", "conv4", "conv5"):
        assert not (t[name].view(torch.int32) & 0x1FFF).any(), name
    # pools are exact
    for src, dst in (("conv1", "pool1"), ("conv2", "pool2")):
        ref = F.max_pool2d(t[src].permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
        assert torch.equal(ref, t[dst]), dst
    ins = ("input", "pool1", "pool2", "conv3", "conv4")
    outs = ("conv1", "conv2", "conv3", "conv4", "conv5")
    rel = []
    for k in range(5):
        wk = rna_tf32(alex[CONV_KEYS[k] + ".weight"].float()).to(cuda)
        bk = alex[CONV_KEYS[k] + ".bias"].float().to(cuda)
        rel.append(_conv_check(t[ins[k]], t[outs[k]], wk, bk, *CONV_SPECS[k], n_sample=20000, seed=k))
    total, bound = _tail_reference(t, [l.to(cuda).reshape(-1) for l in
                                        (lin[f"lin{k}.model.1.weight"] for k in range(5))])
    print(f"{W}x{H} roi {roi}: lpips {got:.9g}, tail |kernel - float64| {abs(got - total):.2e} (bound {bound:.2e}); "
          f"conv |error| / bound per layer {', '.join(f'{r:.2f}' for r in rel)}")
    assert abs(got - total) <= bound


# ---- end to end -------------------------------------------------------------------------------------------------------
E2E_CASES = ([((31, 31), k, None) for k in PAIR_KINDS] + [((32, 47), k, None) for k in PAIR_KINDS]
             + [((752, 1028), k, (3, 5, 749, 1019)) for k in PAIR_KINDS]
             + [((1028, 752), k, r) for k, r in zip(PAIR_KINDS, (None, (0, 0, 1021, 745), (7, 2, 1021, 750),
                                                                   (1, 0, 1027, 752), (0, 9, 1028, 743)))]
             + [((4112, 3008), "noise", "ellipse")])


@pytest.mark.parametrize("size,kind,roi", E2E_CASES, ids=[f"{s[0]}x{s[1]}-{k}-{r}" for s, k, r in E2E_CASES])
def test_end_to_end_matches_oracle(cuda, weights, oracle, size, kind, roi):
    W, H = size
    if roi == "ellipse":
        roi = _ellipse_roi(W, H)
    pred, gt = make_pair(kind, W, H, seed=W + H)
    got, _ = _run(pred, gt, weights[2], cuda, roi)
    ref = oracle(pred, gt, roi)
    rel = abs(got - ref) / ref
    WORST.append((rel, abs(got - ref)))
    print(f"{W}x{H} {kind} roi {roi}: lpips {got:.9g} oracle {ref:.9g} relative {rel:.2e} absolute {abs(got - ref):.2e}"
          f" (worst so far {max(w[0] for w in WORST):.2e} relative, {max(w[1] for w in WORST):.2e} absolute)")
    assert math.isfinite(got) and abs(got - ref) <= REL_BAR * ref + ABS_FLOOR


# ---- ROI, NaN, input types, identities ----------------------------------------------------------------------------------
def test_roi_equals_precropped_image(cuda, weights):
    W, H = 1028, 752
    pred, gt = make_pair("noise", W, H, seed=4)
    for roi in ((5, 3, 1023, 749), (0, 0, 31, 31), (997, 721, 31, 31), (2, 1, 513, 389)):
        x, y, w, h = roi
        a, _ = _run(pred, gt, weights[2], cuda, roi)
        b, _ = _run(pred[y:y + h, x:x + w], gt[y:y + h, x:x + w], weights[2], cuda, (0, 0, w, h))
        c, _ = _run(pred[y:y + h, x:x + w], gt[y:y + h, x:x + w], weights[2], cuda, None)
        assert np.float64(a).tobytes() == np.float64(b).tobytes() == np.float64(c).tobytes(), roi


def test_nan_rule(cuda, weights):
    W, H = 96, 80
    pred, gt = make_pair("noise", W, H, seed=5)
    for roi in ((3, 2, 30, 60), (3, 2, 60, 30), (0, 0, 0, 0), (70, 0, 31, 40), (0, 50, 40, 31), (-1, 0, 40, 40)):
        got, _ = _run(pred, gt, weights[2], cuda, roi)
        assert math.isnan(got), roi
    assert math.isfinite(_run(pred, gt, weights[2], cuda, (65, 49, 31, 31))[0])
    got, _ = _run(pred[:30], gt[:30], weights[2], cuda)
    assert math.isnan(got)


def test_float_input_equals_uint8(cuda, weights):
    pred, gt = make_pair("blur", 1028, 752, seed=6)
    a, _ = _run(pred, gt, weights[2], cuda, (3, 1, 1001, 700))
    b, _ = _run(pred.astype(np.float32) / np.float32(255), gt.astype(np.float32) / np.float32(255), weights[2], cuda,
                (3, 1, 1001, 700))
    assert np.float64(a).tobytes() == np.float64(b).tobytes()


def test_identities_determinism_and_graph(cuda, weights):
    from humanrf_b200.toolbox.lpips import lpips

    w = weights[2]
    pred, gt = make_pair("noise", 1028, 752, seed=7)
    p, g = _dev(pred, cuda), _dev(gt, cuda)
    roi = _roi_t((2, 3, 1001, 701), cuda)
    a = lpips(p, g, w, roi=roi).clone()
    b = lpips(p, g, w, roi=roi).clone()
    s = lpips(g, p, w, roi=roi).clone()
    z = lpips(g, g.clone(), w, roi=roi).clone()
    torch.cuda.synchronize()
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() == s.cpu().numpy().tobytes()
    assert z.item() == 0.0 and a.item() > 0
    # an element of a larger tensor, read back once
    rows = torch.full((3, 3), -1.0, dtype=torch.float64, device=cuda)
    lpips(p, g, w, roi=roi, out=rows[1, 2])
    assert rows[1, 2].item() == a.item() and (rows.view(-1)[[0, 1, 2, 3, 4, 6, 7, 8]] == -1).all()
    # captured in a CUDA graph: no host synchronisation inside; a replay writes the same bytes
    out = torch.zeros((), dtype=torch.float64, device=cuda)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        lpips(p, g, w, roi=roi, out=out)
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lpips(p, g, w, roi=roi, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == a.cpu().numpy().tobytes()


def test_lpips_rejects_bad_inputs(cuda, weights):
    from humanrf_b200.toolbox.lpips import lpips

    w = weights[2]
    x = torch.zeros(40, 36, 3, dtype=torch.uint8, device=cuda)
    bad = [(x.double(), x), (x, x[:, :35].contiguous()), (x, x.float()), (x, x.cpu()), (x[..., :2].contiguous(), x),
           (x.transpose(0, 1), x.transpose(0, 1))]
    for args in bad:
        with pytest.raises(RuntimeError):
            lpips(*args, w)
    with pytest.raises(RuntimeError):
        lpips(x, x, w, roi=torch.zeros(4, dtype=torch.int64, device=cuda))
    with pytest.raises(RuntimeError):
        lpips(x, x, w, out=torch.empty(2, dtype=torch.float64, device=cuda))


# ---- evaluate_sequence ----------------------------------------------------------------------------------------------
def test_evaluate_sequence_with_lpips(cuda, tmp_path, weights):
    import cv2

    from test_evaluation_gpu import _loader
    from test_learned_occupancy_gpu import confined_teacher
    from humanrf_b200.toolbox.evaluation import evaluate_sequence, image_metrics
    from humanrf_b200.toolbox.lpips import lpips

    w = weights[2]
    m = confined_teacher(cuda)
    ds, dl = _loader(cuda)
    pairs = [(0, 15), (2, 15), (1, 16)]
    out = tmp_path / "eval"
    scores = evaluate_sequence(m, dl, pairs, out, lpips_weights=w)
    plain = evaluate_sequence(m, dl, pairs, tmp_path / "plain", save_frames=False)
    rows = list(csv.reader(open(out / "metrics.csv", newline="")))
    assert rows[0] == ["camera", "frame", "PSNR", "LPIPS", "SSIM"]
    names = ["Cam001_rgb000015.png", "Cam003_rgb000015.png", "Cam002_rgb000016.png"]
    for (c, f), name, s, p, row in zip(pairs, names, scores, plain, rows[1:]):
        assert (s.psnr, s.ssim, s.roi) == (p.psnr, p.ssim, p.roi) and p.lpips is None
        png = np.ascontiguousarray(cv2.imread(str(out / "test_frames" / name), cv2.IMREAD_UNCHANGED)[..., ::-1])
        gt = np.ascontiguousarray(np.rint(ds.get_rgb(c, f) * 255).astype(np.uint8)[..., ::-1])
        mask = (ds.get_mask(c, f)[..., 0] * 255).astype(np.uint8)
        _, roi = image_metrics(_dev(png, cuda), _dev(gt, cuda), _dev(mask, cuda))
        ref = lpips(_dev(png, cuda), _dev(gt, cuda), w, roi=roi).item()
        print(f"cam {c} frame {f}: LPIPS {s.lpips:.9g} roi {s.roi}")
        assert s.roi[2] >= 31 and s.roi[3] >= 31
        assert np.float64(s.lpips).tobytes() == np.float64(ref).tobytes()
        assert float(row[3]) == s.lpips and float(row[2]) == s.psnr and float(row[4]) == s.ssim
    avg = list(csv.reader(open(out / "averages.csv", newline="")))
    assert avg[0] == ["PSNR", "LPIPS", "SSIM"]
    assert float(avg[1][1]) == pytest.approx(np.mean([s.lpips for s in scores]), rel=1e-12)
    assert list(csv.reader(open(tmp_path / "plain" / "metrics.csv", newline="")))[0] == ["camera", "frame", "PSNR", "SSIM"]

    # a view whose mask's bounding box is 20 x 20 pixels: SSIM is defined, LPIPS is not, and the error names the view
    get_mask = ds.get_mask

    def small_mask(cam, frame, normalize=True):
        mk = get_mask(cam, frame)
        if (cam, frame) == (1, 16):
            keep = np.zeros_like(mk)
            keep[10:30, 20:40] = 1
            mk = mk * keep
            mk[10, 20] = mk[29, 39] = 1
        return mk

    ds.get_mask = small_mask
    with pytest.raises(RuntimeError, match=r"LPIPS.*\(1, 16\)"):
        evaluate_sequence(m, dl, [(0, 15), (1, 16)], tmp_path / "small", save_frames=False, lpips_weights=w)
    assert not (tmp_path / "small" / "metrics.csv").exists()
