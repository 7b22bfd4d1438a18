"""Per-frame triangle meshes from a trained model's density field.

``extract_mesh`` evaluates the density on the vertices of a grid (``density_lattice``: the corners of the voxels of a
hull or baked occupancy grid, include/humanrf_b200.h ``hrf_density_lattice``) and runs marching cubes over that lattice
on the GPU (``marching_cubes``, ``hrf_marching_cubes_count`` / ``_emit``).  The only host synchronisation of an
extraction is the read of the two mesh counts that sizes the outputs.  ``write_obj`` writes the OBJ subset the
ActorsHQ toolbox's mesh renderer reads (``v`` and ``f`` lines only), ``write_ply`` binary PLY with normals and colours,
and ``export_mesh_sequence`` one OBJ per frame in world units.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import _lib as L


@dataclass
class Mesh:
    """An indexed triangle mesh on the device: vertices f32 [V,3], faces i32 [F,3] (counter-clockwise seen from the
    outside), per-vertex normals f32 [V,3] and colours f32 [V,3] in [0,1], or None."""
    vertices: torch.Tensor
    faces: torch.Tensor
    normals: Optional[torch.Tensor] = None
    colors: Optional[torch.Tensor] = None


def _check_frame(model, frame_number) -> int:
    frame = int(frame_number)
    if frame not in model.sorted_frame_numbers:
        raise RuntimeError(f"frame {frame} is not one of the model's frames")
    return frame


def _check_grid(grid, name) -> int:
    if not isinstance(grid, torch.Tensor):
        raise RuntimeError(f"{name} must be a torch.Tensor")
    if grid.dtype != torch.uint8:
        raise RuntimeError(f"{name} has dtype {grid.dtype}, expected torch.uint8")
    if grid.dim() != 3 or not (grid.shape[0] == grid.shape[1] == grid.shape[2]):
        raise RuntimeError(f"{name} must be a cubic [G,G,G] grid, got shape {tuple(grid.shape)}")
    if grid.device.type != "cuda":
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if not grid.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    return int(grid.shape[0])


@torch.no_grad()
def density_lattice(model, frame_number: int, mask: Optional[torch.Tensor] = None,
                    resolution: Optional[int] = None) -> torch.Tensor:
    """Density of `model` at `frame_number` on the (G+1)^3 corners of a G^3 grid's voxels, float32 [G+1,G+1,G+1]
    indexed [z][y][x]; vertex i sits at i / G - 0.5 per axis.  With a `mask` (uint8 [G,G,G] CUDA, non-zero = occupied)
    G is the mask's and only the corners of occupied voxels are evaluated (0 elsewhere); without one, `resolution` is
    G and every vertex is evaluated.  Each value is exactly ``model.density`` (query form) at that position."""
    frame = _check_frame(model, frame_number)
    device = model.device
    if mask is not None:
        G = _check_grid(mask, "mask")
        if resolution is not None and int(resolution) != G:
            raise RuntimeError(f"resolution {resolution} differs from the mask's {G}")
        if mask.device != device:
            raise RuntimeError("mask and model must be on the same CUDA device")
    elif resolution is None:
        raise RuntimeError("either a mask or a resolution is needed")
    else:
        G = int(resolution)
    nat = model.native()
    lib = L.lib()
    nbytes = int(lib.hrf_density_lattice_workspace_bytes(G))
    if nbytes <= 0:
        raise RuntimeError(f"grid resolution {G} outside [1, 1024]")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
    sigma = torch.empty((G + 1,) * 3, dtype=torch.float32, device=device)
    L.check(lib.hrf_density_lattice(C.byref(nat.field), frame, L.ptr(mask), G, sigma.data_ptr(), ws.data_ptr(),
                                    L.stream()))
    return sigma


@torch.no_grad()
def marching_cubes(lattice: torch.Tensor, level: float, normals: bool = True) -> Mesh:
    """Surface {lattice >= level} of a float32 [(G+1)]^3 CUDA lattice indexed [z][y][x], in the lattice's normalised
    coordinates (vertex i at i / G - 0.5).  One vertex per crossing lattice edge, shared by the cubes around it; the
    contract (vertex and face order, interpolation, case table) is in include/humanrf_b200.h.  Reads the two mesh
    counts back once."""
    L.require_cuda(lattice, "lattice", torch.float32)
    if lattice.dim() != 3 or not (lattice.shape[0] == lattice.shape[1] == lattice.shape[2]) or lattice.shape[0] < 2:
        raise RuntimeError(f"lattice must be a cubic [G+1,G+1,G+1] volume with G >= 1, got {tuple(lattice.shape)}")
    G = int(lattice.shape[0]) - 1
    lib = L.lib()
    nbytes = int(lib.hrf_marching_cubes_workspace_bytes(G))
    if nbytes <= 0:
        raise RuntimeError(f"grid resolution {G} outside [1, 1024]")
    dev = lattice.device
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    L.check(lib.hrf_marching_cubes_count(lattice.data_ptr(), G, float(level), counts.data_ptr(), ws.data_ptr(),
                                         L.stream()))
    nv, nf = (int(c) for c in counts.cpu())
    if nv > 2 ** 31 - 1:
        raise RuntimeError(f"{nv} vertices do not fit int32 face indices")
    verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    nrm = torch.empty((nv, 3), dtype=torch.float32, device=dev) if normals else None
    faces = torch.empty((nf, 3), dtype=torch.int32, device=dev)
    L.check(lib.hrf_marching_cubes_emit(lattice.data_ptr(), G, float(level), nv, nf, L.ptr(verts) if nv else None,
                                        L.ptr(nrm) if nv else None, L.ptr(faces) if nf else None, ws.data_ptr(),
                                        L.stream()))
    return Mesh(verts, faces, nrm)


@torch.no_grad()
def extract_mesh(model, frame_number: int, grid: torch.Tensor, level: float, colors: bool = False) -> Mesh:
    """Mesh of {density >= level} of `model` at `frame_number` inside `grid` (a hull or baked occupancy grid, uint8
    [G,G,G] CUDA): ``density_lattice`` over the grid's occupied voxels, then ``marching_cubes``.  `level` is in the
    model's density units (after ``density_scale``) and should be positive, so that the vertices outside the grid (0)
    are outside the surface.  Positions are in the model's normalised coordinates ([-0.5, 0.5]^3, see ``to_world``).
    With `colors`, each vertex gets ``model.forward``'s radiance (query form, evaluation mode) seen along -normal."""
    from ..scene_representation.query_io import QueryInput

    frame = _check_frame(model, frame_number)
    mesh = marching_cubes(density_lattice(model, frame, grid), level, normals=True)
    if colors:
        n = mesh.vertices.shape[0]
        frames = torch.full((n,), frame, dtype=torch.int32, device=mesh.vertices.device)
        out = model.forward(QueryInput(is_training=False, positions=mesh.vertices, directions=-mesh.normals,
                                       frame_numbers=frames))
        mesh.colors = out.radiance
    return mesh


def to_world(mesh: Mesh, scene_offset, scene_scale) -> Mesh:
    """`mesh` in world units: undoes the loader's normalisation p = (world + scene_offset) * scene_scale
    (dataset/data_loader.py).  Faces, normals and colours are unchanged (the scale is uniform)."""
    off = torch.as_tensor(np.asarray(scene_offset, np.float64), dtype=torch.float64, device=mesh.vertices.device)
    verts = (mesh.vertices.double() / float(scene_scale) - off).float()
    return Mesh(verts, mesh.faces, mesh.normals, mesh.colors)


def write_obj(path, mesh: Mesh) -> None:
    """Wavefront OBJ with `v x y z` lines (`v x y z r g b` with colours) and 1-based `f a b c` lines, nothing else:
    the ActorsHQ mesh renderer's loader warns on any other token.  Floats are written with 9 significant digits, so a
    float32 value reads back exactly."""
    v = mesh.vertices.detach().cpu().numpy().astype(np.float32)
    if mesh.colors is not None:
        v = np.concatenate([v, mesh.colors.detach().cpu().numpy().astype(np.float32)], 1)
    f = mesh.faces.detach().cpu().numpy().astype(np.int64) + 1
    with open(path, "w") as fh:
        if len(v):
            np.savetxt(fh, v, fmt="v " + " ".join(["%.9g"] * v.shape[1]))
        if len(f):
            np.savetxt(fh, f, fmt="f %d %d %d")


def write_ply(path, mesh: Mesh) -> None:
    """Binary little-endian PLY: float x y z, float nx ny nz (with normals), uchar red green blue (with colours), and
    faces as `uchar`-counted `int` index lists."""
    v = mesh.vertices.detach().cpu().numpy().astype("<f4")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if mesh.normals is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if mesh.colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    rec = np.empty(len(v), dtype=fields)
    rec["x"], rec["y"], rec["z"] = v[:, 0], v[:, 1], v[:, 2]
    if mesh.normals is not None:
        n = mesh.normals.detach().cpu().numpy().astype("<f4")
        rec["nx"], rec["ny"], rec["nz"] = n[:, 0], n[:, 1], n[:, 2]
    if mesh.colors is not None:
        c = np.clip(np.rint(mesh.colors.detach().cpu().numpy().astype(np.float64) * 255.0), 0, 255).astype(np.uint8)
        rec["red"], rec["green"], rec["blue"] = c[:, 0], c[:, 1], c[:, 2]
    f = mesh.faces.detach().cpu().numpy().astype("<i4")
    frec = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frec["n"], frec["i"] = 3, f
    names = {"<f4": "float", "u1": "uchar"}
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    header += [f"property {names[t]} {n}" for n, t in fields]
    header += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(rec.tobytes())
        fh.write(frec.tobytes())


def scene_normalisation(dataset):
    """(scene_offset, scene_scale) the DataLoader derives from `dataset.get_aabb()` (dataset/data_loader.py)."""
    aabb = np.asarray(dataset.get_aabb(), np.float64)
    return -aabb.mean(0), 1 / np.max(aabb[1] - aabb[0])


@torch.no_grad()
def export_mesh_sequence(model, dataset, frames, out_dir, level: float, bake: bool = True,
                         render_step_size: float = 4e-4, colors: bool = False):
    """Writes `out_dir`/frame%06d.obj for every frame of `frames`, in world units: the frame's hull from
    ``dataset.get_occupancy_grid`` (tightened by ``bake_occupancy_grid`` first when `bake`), ``extract_mesh`` at
    `level`, ``to_world`` with the DataLoader's normalisation of `dataset`.  Returns the written paths."""
    from .learned_occupancy import bake_occupancy_grid

    frames = [_check_frame(model, f) for f in frames]
    offset, scale = scene_normalisation(dataset)
    device = model.device
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for frame in frames:
        grid = torch.from_numpy(np.ascontiguousarray(dataset.get_occupancy_grid(frame_number=frame))).to(device)
        if bake:
            grid = bake_occupancy_grid(model, frame, grid, render_step_size)
        mesh = to_world(extract_mesh(model, frame, grid, level, colors=colors), offset, scale)
        path = os.path.join(out_dir, f"frame{frame:06d}.obj")
        write_obj(path, mesh)
        paths.append(path)
    return paths
