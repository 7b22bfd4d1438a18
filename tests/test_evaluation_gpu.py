"""Image scores on the H100 (csrc/image_metrics.cu, hrf_image_metrics, toolbox/evaluation.py): the kernel against the
float64 oracle of tests/eval_oracle.py, determinism, graph capture, and evaluate_sequence against evaluate.py's
pipeline restated on the files it writes."""
import csv
import math

import numpy as np
import pytest
import torch

from eval_oracle import evaluate_pair
from test_learned_occupancy_gpu import _sphere, confined_teacher

pytestmark = pytest.mark.gpu

SSIM_TOL, PSNR_TOL = 1e-10, 1e-9


def _images(W, H, seed):
    """gt uniform in 0..255; pred = gt + noise, clipped; blocks of 0 and 255 in both (the largest window sums)."""
    rng = np.random.default_rng(seed)
    gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    pred = np.clip(gt.astype(np.int32) + rng.integers(-30, 31, gt.shape), 0, 255).astype(np.uint8)
    bh, bw = max(1, H // 5), max(1, W // 5)
    gt[:bh, :bw] = 255
    pred[:bh, :bw] = 255
    gt[H - bh:, W - bw:] = 0
    pred[H - bh:, :bw] = 0
    pred[H // 2:H // 2 + bh, W // 2:W // 2 + bw] = 255
    return pred, gt


def _ellipse(W, H, fx=0.35, fy=0.42):
    y, x = np.mgrid[0:H, 0:W]
    return (((x + 0.5 - W / 2) / (fx * W)) ** 2 + ((y + 0.5 - H / 2) / (fy * H)) ** 2 <= 1).astype(np.uint8) * 255


def _mask(kind, W, H, seed):
    rng = np.random.default_rng(seed + 1)
    m = np.zeros((H, W), np.uint8)
    if kind == "full":
        m[:] = 1
    elif kind == "random":
        m = (rng.random((H, W)) < 0.3).astype(np.uint8)
    elif kind == "ellipse":
        m = _ellipse(W, H)
    elif kind == "borders":          # touches all four borders, with holes
        m = (rng.random((H, W)) < 0.7).astype(np.uint8) * 200
        m[0, W // 3] = m[H - 1, W // 2] = m[H // 3, 0] = m[H // 2, W - 1] = 1
    elif kind == "sparse_rect":      # random pixels inside a sub-rectangle
        x0, y0 = W // 7, H // 5
        m[y0:H - H // 6, x0:W - W // 9] = rng.random((H - H // 6 - y0, W - W // 9 - x0)) < 0.02
        m[y0, x0] = m[H - H // 6 - 1, W - W // 9 - 1] = 1
    elif kind.startswith("w") or kind.startswith("h"):   # an ROI exactly N wide (w7, w6) or N tall (h7)
        n = int(kind[1:])
        if kind[0] == "w":
            m[H // 4:H - 2, W // 3:W // 3 + n] = rng.random((H - 2 - H // 4, n)) < 0.5
            m[H // 4, W // 3] = m[H - 3, W // 3 + n - 1] = 1
        else:
            m[H // 3:H // 3 + n, 2:W - 1] = rng.random((n, W - 3)) < 0.5
            m[H // 3, 2] = m[H // 3 + n - 1, W - 2] = 1
    elif kind != "empty":
        raise ValueError(kind)
    return m


CASES = [(7, 7, "full"), (13, 9, "random"), (13, 9, "borders"), (1028, 752, "ellipse"), (752, 1028, "sparse_rect"),
         (1028, 752, "borders"), (100, 60, "w7"), (100, 60, "h7"), (100, 60, "w6"), (64, 48, "empty"),
         (4112, 3008, "ellipse")]


@pytest.mark.parametrize("W,H,kind", CASES)
def test_kernel_matches_oracle(cuda, W, H, kind):
    from humanrf_b200.toolbox.evaluation import image_metrics

    seed = W * 7 + H
    pred, gt = _images(W, H, seed)
    mask = _mask(kind, W, H, seed)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    out, roi = image_metrics(t(pred), t(gt), t(mask))
    torch.cuda.synchronize()
    p, s = out.cpu().numpy()
    rp, rs, rroi = evaluate_pair(pred, gt, mask)
    print(f"{W}x{H} {kind}: roi {tuple(roi.tolist())} PSNR {p:.12f} ({p - rp:+.2e}) SSIM {s:.15f} ({s - rs:+.2e})")
    assert tuple(roi.cpu().tolist()) == rroi
    if kind == "empty":
        assert math.isnan(p) and math.isnan(s) and rroi == (0, 0, 0, 0)
        return
    assert math.isfinite(p) and abs(p - rp) <= PSNR_TOL
    if kind == "w6":
        assert math.isnan(s) and math.isnan(rs)
    else:
        assert math.isfinite(s) and abs(s - rs) <= SSIM_TOL


def test_identical_images_deterministic_and_graph_captured(cuda):
    from humanrf_b200.toolbox.evaluation import image_metrics

    W, H = 1028, 752
    pred, gt = _images(W, H, 3)
    mask = torch.from_numpy(_ellipse(W, H)).to(cuda)
    p, g = torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda)
    same, _ = image_metrics(g, g.clone(), mask > 0)          # a bool mask is taken as it is
    torch.cuda.synchronize()
    assert same[0].item() == float("inf") and same[1].item() >= 1 - 1e-12
    a, ra = image_metrics(p, g, mask)
    b, rb = image_metrics(p, g, mask)
    torch.cuda.synchronize()
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() and torch.equal(ra, rb)
    # rows of one [n, 2] tensor, read back once
    rows = torch.full((3, 2), -1.0, dtype=torch.float64, device=cuda)
    image_metrics(p, g, mask, out=rows[0])
    image_metrics(g, g, mask, out=rows[1])
    image_metrics(p, g, mask, out=rows[2])
    r = rows.cpu().numpy()
    assert r[0].tobytes() == a.cpu().numpy().tobytes() == r[2].tobytes() and r[1, 0] == float("inf")
    # captured in a CUDA graph: no host synchronisation inside; a replay writes the same bytes
    out = torch.zeros(2, dtype=torch.float64, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        image_metrics(p, g, mask, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _, rg = image_metrics(p, g, mask, out=out)
    out.zero_()
    rg.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == a.cpu().numpy().tobytes() and torch.equal(rg, ra)


def test_image_metrics_rejects_bad_inputs(cuda):
    from humanrf_b200.toolbox.evaluation import image_metrics

    x = torch.zeros(16, 12, 3, dtype=torch.uint8, device=cuda)
    m = torch.ones(16, 12, dtype=torch.uint8, device=cuda)
    bad = [(x.float(), x, m), (x, x[:, :11].contiguous(), m), (x, x, m[:15]), (x, x, m.float()),
           (x, x.transpose(0, 1).contiguous().transpose(0, 1), m), (x, x.cpu(), m), (x[..., :2].contiguous(), x, m)]
    for args in bad:
        with pytest.raises(RuntimeError):
            image_metrics(*args)
    with pytest.raises(RuntimeError):
        image_metrics(x, x, m, out=torch.empty(2, dtype=torch.float32, device=cuda))


def _loader(cuda, empty_mask=None):
    """The depth-map tests' scene (SyntheticDataset, sphere hulls), camera 2 made portrait by swapping its size."""
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset

    ds = SyntheticDataset(G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    cam = ds.cameras[2]
    cam.width, cam.height = cam.height, cam.width
    cam.focal_length = np.array([cam.focal_length[0], cam.focal_length[0] * cam.width / cam.height])
    if empty_mask is not None:
        get_mask = ds.get_mask
        ds.get_mask = lambda c, f, normalize=True: (0 * get_mask(c, f) if (c, f) == empty_mask else get_mask(c, f))
    return ds, DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
                  space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=64 * 48, camera_numbers=(0, 1, 2),
                  frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])


def test_evaluate_sequence(cuda, tmp_path):
    import cv2

    from humanrf_b200.toolbox.depth_maps import render_depth_map
    from humanrf_b200.toolbox.evaluation import evaluate_sequence, quantize

    m = confined_teacher(cuda)
    ds, dl = _loader(cuda)
    assert (dl.cameras[2].width, dl.cameras[2].height) == (48, 64)
    pairs = [(0, 15), (2, 15), (1, 16), (0, 16)]
    out = tmp_path / "eval"
    scores = evaluate_sequence(m, dl, pairs, out)
    names = ["Cam001_rgb000015.png", "Cam003_rgb000015.png", "Cam002_rgb000016.png", "Cam001_rgb000016.png"]
    assert sorted(p.name for p in (out / "test_frames").iterdir()) == sorted(names)
    rows = list(csv.reader(open(out / "metrics.csv", newline="")))
    assert rows[0] == ["camera", "frame", "PSNR", "SSIM"]
    assert [r[:2] for r in rows[1:]] == [["1", "15"], ["3", "15"], ["2", "16"], ["1", "16"]]
    ref = []
    for (c, f), name, s, row in zip(pairs, names, scores, rows[1:]):
        # the PNG is the quantised render
        color = render_depth_map(m, dl, c, f).color
        png = cv2.imread(str(out / "test_frames" / name), cv2.IMREAD_UNCHANGED)
        assert png.shape == (dl.cameras[c].height, dl.cameras[c].width, 3)
        assert np.array_equal(png[..., ::-1], quantize(color).cpu().numpy())
        # evaluate.py's pipeline restated: the PNG read back, the dataset's 8-bit image and its mask's first channel
        gt = np.rint(ds.get_rgb(c, f) * 255).astype(np.uint8)[..., ::-1]
        mask = (ds.get_mask(c, f)[..., 0] * 255).astype(np.uint8)
        rp, rs, rroi = evaluate_pair(png[..., ::-1], gt, mask)
        print(f"cam {c} frame {f}: PSNR {s.psnr:.6f} ({s.psnr - rp:+.1e}) SSIM {s.ssim:.6f} ({s.ssim - rs:+.1e}) roi {s.roi}")
        assert (s.camera, s.frame, s.roi) == (c, f, rroi)
        assert abs(s.psnr - rp) <= PSNR_TOL and abs(s.ssim - rs) <= SSIM_TOL
        assert float(row[2]) == s.psnr and float(row[3]) == s.ssim
        ref.append((rp, rs))
    avg = list(csv.reader(open(out / "averages.csv", newline="")))
    assert avg[0] == ["PSNR", "SSIM"]
    assert float(avg[1][0]) == pytest.approx(np.mean([r[0] for r in ref]), abs=1e-9)
    assert float(avg[1][1]) == pytest.approx(np.mean([r[1] for r in ref]), abs=1e-10)
    # the rendered views are not trivially black: the sphere is in view
    assert all(cv2.imread(str(out / "test_frames" / n)).any() for n in names)

    # bad cameras or frames are rejected before anything exists
    for bad in ([(0, 15), (0, 99)], [(7, 15)], [(-1, 15)]):
        with pytest.raises(RuntimeError):
            evaluate_sequence(m, dl, bad, tmp_path / "bad")
        assert not (tmp_path / "bad").exists()
    # an empty mask: the error names the pair, and no table is written
    _, dl_empty = _loader(cuda, empty_mask=(1, 16))
    with pytest.raises(RuntimeError, match=r"\(1, 16\)"):
        evaluate_sequence(m, dl_empty, [(0, 15), (1, 16)], tmp_path / "empty", save_frames=False)
    assert not (tmp_path / "empty" / "metrics.csv").exists()
    # baked grids
    baked = evaluate_sequence(m, dl, [(0, 15), (2, 16)], tmp_path / "baked", bake=True, save_frames=False)
    assert len(baked) == 2 and all(math.isfinite(s.psnr) and math.isfinite(s.ssim) for s in baked)
    assert (tmp_path / "baked" / "metrics.csv").exists() and not (tmp_path / "baked" / "test_frames").exists()
