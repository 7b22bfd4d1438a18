"""Scores of the learned geometry against the dataset's meshes on the GPU.

``mesh_distance`` runs one direction of ``hrf_mesh_distance`` (csrc/mesh_distance.cu, contract in
include/humanrf_b200.h and DESIGN.md §3.11): points sampled on a source mesh by area, each queried for the closest point
on a target mesh's surface through a tree over the target's triangles.  ``compare_meshes`` runs both directions and
returns the usual scores (accuracy, completeness, Chamfer distance, normal consistency, F-score per threshold).
``evaluate_geometry`` meshes each frame of a trained model as ``export_mesh_sequence`` does and scores it against the
dataset's OBJ meshes (``alembic_extractor``'s ``Frame%06d.obj``), writing ``geometry.csv`` and ``geometry_averages.csv``.
``read_obj`` reads the OBJ subset ``alembic_extractor`` and ``write_obj`` write.
"""
from __future__ import annotations

import csv
import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from .. import _lib as L
from .mesh_extraction import Mesh, _check_frame, extract_mesh, scene_normalisation, to_world

MAX_TAUS = 8
DEFAULT_TAUS = (0.005, 0.01, 0.02)


@dataclass
class GeometryScore:
    """Scores of a predicted mesh against a reference mesh, in the meshes' units: accuracy = mean distance pred -> ref,
    completeness = mean distance ref -> pred, chamfer_l1 = their mean, chamfer_l2 = the mean of the two directions' mean
    squared distances, normal_consistency = the mean of the two directions' mean |n_pred . n_ref|, and per threshold
    (taus) precision = share of pred samples within tau of ref, recall = share of ref samples within tau of pred and
    fscore = 2PR / (P + R) (0 when P + R = 0).  frame is set by ``evaluate_geometry``."""
    accuracy: float
    completeness: float
    chamfer_l1: float
    chamfer_l2: float
    normal_consistency: float
    taus: tuple
    precision: tuple
    recall: tuple
    fscore: tuple
    frame: int | None = None


def _line_error(path, lineno, msg):
    return RuntimeError(f"{path}:{lineno}: {msg}")


def read_obj(path, device="cuda") -> Mesh:
    """The triangle mesh of a Wavefront OBJ file, as ``alembic_extractor`` and ``write_obj`` write them: ``v x y z`` lines
    (``v x y z r g b`` give colours) and ``f a b c`` lines with 1-based indices, each also in the ``a/b/c``, ``a//c`` and
    ``a/b`` forms (only the vertex index is used).  Every other line is ignored.  Faces that are not triangles, indices
    that are 0, negative or past the last vertex, and files without faces are rejected, naming the file and line.  The
    numbers are converted by numpy in bulk."""
    with open(path, "r") as fh:
        lines = fh.read().splitlines()
    toks = [ln.split() for ln in lines]
    vi = [i for i, t in enumerate(toks) if t and t[0] == "v"]
    fi = [i for i, t in enumerate(toks) if t and t[0] == "f"]
    vlen = np.fromiter((len(toks[i]) for i in vi), np.int64, len(vi))
    bad = np.nonzero((vlen != 4) & (vlen != 7))[0]
    if len(bad):
        raise _line_error(path, vi[bad[0]] + 1, f"a vertex needs 3 coordinates (and optionally 3 colours): "
                                                f"{lines[vi[bad[0]]]!r}")
    flen = np.fromiter((len(toks[i]) for i in fi), np.int64, len(fi))
    bad = np.nonzero(flen != 4)[0]
    if len(bad):
        raise _line_error(path, fi[bad[0]] + 1, f"only triangles are supported: {lines[fi[bad[0]]]!r}")
    if not fi:
        raise RuntimeError(f"{path}: no faces")
    colors = None
    if vi:
        with_rgb = vlen == 7
        if with_rgb.any() and not with_rgb.all():
            k = int(np.nonzero(with_rgb != with_rgb[0])[0][0])
            raise _line_error(path, vi[k] + 1, "some vertices have colours and some do not")
        width = 6 if with_rgb[0] else 3
        vals = np.array([x for i in vi for x in toks[i][1:]]).astype(np.float64).reshape(-1, width)
        verts = vals[:, :3].astype(np.float32)
        if width == 6:
            colors = vals[:, 3:].astype(np.float32)
    else:
        verts = np.zeros((0, 3), np.float32)
    ftok = np.array([x for i in fi for x in toks[i][1:]])
    try:
        idx = np.char.partition(ftok, "/")[:, 0].astype(np.int64).reshape(-1, 3)
    except ValueError:
        bad = [i for i in fi if not all(t.split("/")[0].lstrip("-").isdigit() for t in toks[i][1:])]
        raise _line_error(path, bad[0] + 1 if bad else fi[0] + 1, "face indices must be integers") from None
    bad = np.nonzero(((idx < 1) | (idx > len(verts))).any(1))[0]
    if len(bad):
        raise _line_error(path, fi[bad[0]] + 1, f"face index outside [1, {len(verts)}]: {lines[fi[bad[0]]]!r}")
    faces = (idx - 1).astype(np.int32)
    dev = torch.device(device)
    return Mesh(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), None,
                None if colors is None else torch.from_numpy(colors).to(dev))


def _check_mesh(mesh, name):
    if not isinstance(mesh, Mesh):
        raise RuntimeError(f"{name} must be a Mesh")
    v, f = mesh.vertices, mesh.faces
    for t, what, dt in ((v, "vertices", torch.float32), (f, "faces", torch.int32)):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError(f"{name}.{what} must be a torch.Tensor")
        L.require_cuda(t, f"{name}.{what}", dt)
        if t.dim() != 2 or t.shape[1] != 3:
            raise RuntimeError(f"{name}.{what} must be [n,3], got {tuple(t.shape)}")
    if v.device != f.device:
        raise RuntimeError(f"{name}.vertices and {name}.faces must be on one device")
    if f.shape[0] >= 2 ** 31:
        raise RuntimeError(f"{name} has {f.shape[0]} faces; at most 2^31 - 1 are supported")


def _check_taus(taus):
    taus = tuple(float(t) for t in taus)
    if len(taus) > MAX_TAUS:
        raise RuntimeError(f"at most {MAX_TAUS} thresholds, got {len(taus)}")
    if any(not math.isfinite(t) or t < 0 for t in taus):
        raise RuntimeError(f"thresholds must be finite and non-negative, got {taus}")
    return taus


def mesh_distance(src: Mesh, dst: Mesh, num_samples: int, seed: int, taus=DEFAULT_TAUS, out=None,
                  per_sample: bool = False):
    """One direction on the device, without synchronising: `num_samples` points sampled on `src` by area (seeded by
    `seed`), each with its distance to the closest point of `dst`'s surface.  Returns ``(out, counts, error, samples)``:
    out float64 [3] = (mean distance, mean squared distance, mean |n_src . n_dst|), counts int64 [len(taus)] = samples
    with distance <= tau (tau rounded to float32), error int32 [1] (bit 0: a src face index out of range, bit 1: a dst
    one), and with `per_sample` a dict of points f32 [N,3], faces i32 [N], distances f32 [N] and closest i32 [N]
    (None without).  `out` may be given (e.g. a row of an [n,3] float64 tensor).  out is NaN and counts -1 when error is
    set or either mesh has no face of non-zero area."""
    _check_mesh(src, "src")
    _check_mesh(dst, "dst")
    dev = src.vertices.device
    if dst.vertices.device != dev:
        raise RuntimeError("src and dst must be on one device")
    n = int(num_samples)
    if not 1 <= n < 2 ** 31:
        raise RuntimeError(f"num_samples must be in [1, 2^31), got {num_samples}")
    taus = _check_taus(taus)
    seed = int(seed)
    if not 0 <= seed < 2 ** 64:
        raise RuntimeError(f"seed must be in [0, 2^64), got {seed}")
    if out is None:
        out = torch.empty(3, dtype=torch.float64, device=dev)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float64 or out.device != dev or out.shape != (3,)
          or not out.is_contiguous()):
        raise RuntimeError(f"out must be a contiguous float64 [3] tensor on {dev}")
    counts = torch.empty(len(taus), dtype=torch.int64, device=dev)
    error = torch.empty(1, dtype=torch.int32, device=dev)
    samples = None
    if per_sample:
        samples = {"points": torch.empty((n, 3), dtype=torch.float32, device=dev),
                   "faces": torch.empty(n, dtype=torch.int32, device=dev),
                   "distances": torch.empty(n, dtype=torch.float32, device=dev),
                   "closest": torch.empty(n, dtype=torch.int32, device=dev)}
    lib = L.lib()
    fs, ft = int(src.faces.shape[0]), int(dst.faces.shape[0])
    nbytes = int(lib.hrf_mesh_distance_workspace_bytes(fs, ft, n, len(taus)))
    if nbytes <= 0:
        raise RuntimeError("bad mesh distance sizes")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    tau_arr = (C.c_float * max(len(taus), 1))(*taus)
    s = samples or {}
    with torch.cuda.device(dev):
        L.check(lib.hrf_mesh_distance(
            L.ptr(src.vertices) if src.vertices.numel() else None, int(src.vertices.shape[0]),
            L.ptr(src.faces) if fs else None, fs,
            L.ptr(dst.vertices) if dst.vertices.numel() else None, int(dst.vertices.shape[0]),
            L.ptr(dst.faces) if ft else None, ft, n, seed, tau_arr, len(taus), out.data_ptr(),
            counts.data_ptr() if taus else None, error.data_ptr(), L.ptr(s.get("points")), L.ptr(s.get("faces")),
            L.ptr(s.get("distances")), L.ptr(s.get("closest")), ws.data_ptr(), L.stream()))
    return out, counts, error, samples


def scores_from(fwd, bwd, cnt_fwd, cnt_bwd, num_samples, taus, frame=None) -> GeometryScore:
    """A ``GeometryScore`` from the two directions' read-back results: fwd / bwd = ``mesh_distance``'s out for
    pred -> ref and ref -> pred, cnt_* its counts, num_samples per direction."""
    n = float(num_samples)
    valid = all(not math.isnan(float(x)) for x in (*fwd, *bwd))
    prec, rec, fs = [], [], []
    for i in range(len(taus)):
        p = float(cnt_fwd[i]) / n if valid else math.nan
        r = float(cnt_bwd[i]) / n if valid else math.nan
        prec.append(p)
        rec.append(r)
        fs.append(math.nan if not valid else (0.0 if p + r == 0 else 2 * p * r / (p + r)))
    acc, comp = float(fwd[0]), float(bwd[0])
    return GeometryScore(acc, comp, (acc + comp) / 2, (float(fwd[1]) + float(bwd[1])) / 2,
                         (float(fwd[2]) + float(bwd[2])) / 2, tuple(taus), tuple(prec), tuple(rec), tuple(fs), frame)


def _launch_pair(pred, ref, num_samples, taus, seed, row_fwd, row_bwd, cnt, err):
    _, c0, e0, _ = mesh_distance(pred, ref, num_samples, seed, taus, out=row_fwd)
    _, c1, e1, _ = mesh_distance(ref, pred, num_samples, seed, taus, out=row_bwd)
    cnt[0].copy_(c0)
    cnt[1].copy_(c1)
    err[0].copy_(e0[0])
    err[1].copy_(e1[0])


def _raise_on_errors(err, pred_name, ref_name):
    """err = the two directions' error words (pred -> ref, ref -> pred): bit 0 names the source, bit 1 the target."""
    bad = [name for name, hit in ((pred_name, (err[0] & 1) | (err[1] & 2)), (ref_name, (err[0] & 2) | (err[1] & 1)))
           if hit]
    if bad:
        raise RuntimeError(f"face indices outside the vertex range in {' and '.join(bad)}")


@torch.no_grad()
def compare_meshes(pred: Mesh, ref: Mesh, num_samples: int = 1_000_000, taus=DEFAULT_TAUS,
                   seed: int = 0) -> GeometryScore:
    """Scores of `pred` against `ref` (both on one CUDA device, same units): `num_samples` points on each, both
    directions with the same `seed`, read back once.  Raises when a face index is out of range; a mesh without a face of
    non-zero area gives NaN scores."""
    taus = _check_taus(taus)
    dev = pred.vertices.device
    vals = torch.empty((2, 3), dtype=torch.float64, device=dev)
    cnt = torch.empty((2, len(taus)), dtype=torch.int64, device=dev)
    err = torch.empty(2, dtype=torch.int32, device=dev)
    _launch_pair(pred, ref, num_samples, taus, seed, vals[0], vals[1], cnt, err)
    v, c, e = vals.cpu().numpy(), cnt.cpu().numpy(), err.cpu().numpy()
    _raise_on_errors(e, "pred", "ref")
    return scores_from(v[0], v[1], c[0], c[1], num_samples, taus)


CSV_BASE = ("frame", "accuracy", "completeness", "chamfer_l1", "chamfer_l2", "normal_consistency")


def csv_columns(taus):
    """``geometry.csv``'s columns: frame, the five distances, then precision, recall and F per threshold."""
    cols = list(CSV_BASE)
    for t in taus:
        cols += [f"precision@{t:g}", f"recall@{t:g}", f"fscore@{t:g}"]
    return cols


def write_geometry_tables(out_dir, scores) -> None:
    """``geometry.csv`` (one row per frame, in order, columns ``csv_columns``) and ``geometry_averages.csv`` (the mean of
    every column but frame)."""
    taus = scores[0].taus
    cols = csv_columns(taus)

    def row(s):
        r = [s.frame, s.accuracy, s.completeness, s.chamfer_l1, s.chamfer_l2, s.normal_consistency]
        for p, q, f in zip(s.precision, s.recall, s.fscore):
            r += [p, q, f]
        return r

    os.makedirs(out_dir, exist_ok=True)
    rows = [row(s) for s in scores]
    with open(os.path.join(out_dir, "geometry.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(cols)
        w.writerows(rows)
    with open(os.path.join(out_dir, "geometry_averages.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(cols[1:])
        w.writerow([float(np.mean([r[k] for r in rows])) for k in range(1, len(cols))])


@torch.no_grad()
def evaluate_geometry(model, dataset, frames, reference_dir, out_dir, level: float, bake: bool = True,
                      num_samples: int = 1_000_000, taus=DEFAULT_TAUS, seed: int = 0,
                      reference_name: str = "Frame{:06d}.obj", render_step_size: float = 4e-4):
    """Scores the learned geometry of every frame of `frames` against the dataset's meshes: the frame's hull from
    ``dataset.get_occupancy_grid`` (tightened by ``bake_occupancy_grid`` first when `bake`), ``extract_mesh`` at `level`
    and ``to_world`` with the DataLoader's normalisation of `dataset`, as ``export_mesh_sequence`` writes it, so
    distances are in the dataset's world units (metres for ActorsHQ); then ``compare_meshes`` against
    ``reference_dir/reference_name.format(frame)`` (``read_obj``).  ``alembic_extractor`` numbers its OBJs by Alembic
    sample index, taken here to be the dataset's 0-based frame number; pass `reference_name` where a take differs.
    Every frame and every reference file is checked before any work; the scores are read back once at the end, and a
    frame without a score (an empty mesh at `level`, or a reference without a face of non-zero area) raises, naming it.
    Writes ``out_dir/geometry.csv`` and ``out_dir/geometry_averages.csv``; returns a ``GeometryScore`` per frame."""
    from .learned_occupancy import bake_occupancy_grid

    frames = [_check_frame(model, f) for f in frames]
    if not frames:
        raise RuntimeError("no frames to evaluate")
    taus = _check_taus(taus)
    paths = [os.path.join(reference_dir, reference_name.format(f)) for f in frames]
    missing = [p for p in paths if not os.path.isfile(p)]
    if missing:
        raise RuntimeError(f"missing reference meshes: {missing}")
    offset, scale = scene_normalisation(dataset)
    dev = model.device
    vals = torch.empty((len(frames), 2, 3), dtype=torch.float64, device=dev)
    cnt = torch.empty((len(frames), 2, len(taus)), dtype=torch.int64, device=dev)
    err = torch.empty((len(frames), 2), dtype=torch.int32, device=dev)
    for k, (frame, path) in enumerate(zip(frames, paths)):
        grid = torch.from_numpy(np.ascontiguousarray(dataset.get_occupancy_grid(frame_number=frame))).to(dev)
        if bake:
            grid = bake_occupancy_grid(model, frame, grid, render_step_size)
        pred = to_world(extract_mesh(model, frame, grid, level), offset, scale)
        ref = read_obj(path, device=dev)
        _launch_pair(pred, ref, num_samples, taus, seed, vals[k, 0], vals[k, 1], cnt[k], err[k])
    v, c, e = vals.cpu().numpy(), cnt.cpu().numpy(), err.cpu().numpy()
    for k, path in enumerate(paths):
        _raise_on_errors(e[k], f"the mesh of frame {frames[k]}", path)
    scores = [scores_from(v[k, 0], v[k, 1], c[k, 0], c[k, 1], num_samples, taus, frame)
              for k, frame in enumerate(frames)]
    bad = [s.frame for s in scores if any(math.isnan(x) for x in (s.accuracy, s.completeness, s.normal_consistency))]
    if bad:
        raise RuntimeError(f"no geometry score for frames {bad}: the mesh at level {level} or the reference mesh has no "
                           "face of non-zero area")
    write_geometry_tables(out_dir, scores)
    return scores
