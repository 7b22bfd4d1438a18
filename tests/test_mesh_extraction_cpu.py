"""Marching-cubes contract on the CPU oracle (tests/mc_oracle.py) and the mesh writers of toolbox/mesh_extraction.py."""
import numpy as np
import pytest
import torch

import mc_oracle as O


def random_lattice(G, seed):
    """Standard-normal values with a border of -1: every cube case occurs at G = 32 and the surface stays inside."""
    lat = np.random.default_rng(seed).standard_normal((G + 1,) * 3).astype(np.float32)
    lat[0], lat[-1], lat[:, 0], lat[:, -1], lat[:, :, 0], lat[:, :, -1] = (-1,) * 6
    return lat


def sphere_lattice(G, r):
    c = np.arange(G + 1) / G - 0.5
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    return (r - np.sqrt(x * x + y * y + z * z)).astype(np.float32)


def cube_cases(lat, level):
    G = lat.shape[0] - 1
    ins = (lat >= np.float32(level)).astype(np.int64)
    case = np.zeros((G, G, G), np.int64)
    for c in range(8):
        case |= ins[c >> 2:(c >> 2) + G, (c >> 1) & 1:((c >> 1) & 1) + G, c & 1:(c & 1) + G] << c
    return case


def teacher_sign_lattice(G):
    """The sign s of the confined teacher (test_learned_occupancy_gpu.confined_teacher) on the (G+1)^3 lattice:
    trilinear interpolation of the +-1 ellipsoid grid on the dense level 0.  sigma = 100 e^{12 s}, so
    sigma >= 100 <=> s >= 0.  Also returns the level-0 scale."""
    from humanrf_b200.scene_representation.humanrf import HumanRF
    from humanrf_b200.synthetic import MODEL_KW

    lay = HumanRF(sorted_frame_numbers=tuple(range(15, 21)), segment_sizes=(6,), **MODEL_KW).feature_grids[0].layout
    res, scale = int(lay.res[0]), float(lay.scale[0])
    i = np.arange(res)
    c = (i - 0.5) / scale - 0.5
    zz, yy, xx = np.meshgrid(c, c, c, indexing="ij")
    sign = np.where((xx / 0.2) ** 2 + (yy / 0.3) ** 2 + (zz / 0.15) ** 2 <= 1.0, 1.0, -1.0)
    p = np.arange(G + 1) / G                 # p + 0.5 of lattice vertex k
    g = scale * p + 0.5
    g0 = np.floor(g).astype(np.int64)
    w = g - g0
    s = np.zeros((G + 1,) * 3)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                wz = (w if dz else 1 - w)[:, None, None]
                wy = (w if dy else 1 - w)[None, :, None]
                wx = (w if dx else 1 - w)[None, None, :]
                iz, iy, ix = (np.minimum(g0 + d, res - 1) for d in (dz, dy, dx))   # the border is far outside E
                s += wz * wy * wx * sign[np.ix_(iz, iy, ix)]
    return s.astype(np.float32), scale


def test_case_table_is_consistent():
    assert O.NTRI[0] == 0 and O.NTRI[255] == 0
    for case in range(1, 255):
        cross, _ = O._face_rule_segments(case)
        used = O.TRI[case, :3 * O.NTRI[case]]
        assert set(used.tolist()) == {e for e in range(12) if cross[e]}, case


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_lattices_give_closed_oriented_meshes(seed):
    G = 32
    lat = random_lattice(G, seed)
    assert np.unique(cube_cases(lat, 0.0)).size == 256
    v, f, n = O.marching_cubes(lat, 0.0)
    assert O.is_closed_oriented(f)
    assert np.array_equal(np.unique(f), np.arange(len(v)))            # every vertex used
    # one vertex per crossing lattice edge, lying on that edge
    ins = lat >= 0
    ncross = (ins[:, :, 1:] != ins[:, :, :-1]).sum() + (ins[:, 1:] != ins[:, :-1]).sum() + (ins[1:] != ins[:-1]).sum()
    assert len(v) == ncross
    k = np.rint((v + 0.5) * G)
    assert ((np.abs((v + 0.5) * G - k) < 1e-4).sum(1) >= 2).all()
    assert O.signed_volume(v, f) > 0
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)


def test_sphere():
    G, r = 64, 0.3
    v, f, n = O.marching_cubes(sphere_lattice(G, r), 0.0)
    assert O.is_closed_oriented(f) and O.components(len(v), f) == 1
    assert O.euler_characteristic(v, f) == 2
    # a polyhedron inscribed in the sphere loses at most the caps over its facets: with facets of diameter
    # h <= sqrt(2)/G the relative volume error is below 3 h^2 / (8 r^2), about 1 % here
    vol, ref = O.signed_volume(v, f), 4 / 3 * np.pi * r ** 3
    tol = 3 * (np.sqrt(2) / G) ** 2 / (8 * r * r)
    assert abs(vol - ref) <= tol * ref, (vol, ref)
    assert np.abs(np.linalg.norm(v, axis=1) - r).max() <= 1 / G
    radial = v / np.linalg.norm(v, axis=1, keepdims=True)
    assert (np.einsum("ij,ij->i", n, radial) > 0.99).all()          # -grad sigma points outward


def test_teacher_surface_topology():
    """The confined teacher's surface at sigma = 100 is one closed sphere-like component at the GPU test's G."""
    s, scale = teacher_sign_lattice(128)
    v, f, _ = O.marching_cubes(s, 0.0)
    assert O.is_closed_oriented(f)
    assert O.components(len(v), f) == 1 and O.euler_characteristic(v, f) == 2


def parse_obj_like_the_renderer(path):
    """actorshq/toolbox/mesh_tools/renderer/main.cpp load_obj: the first token up to ' ' selects the line kind; 'f'
    takes three 1-based indices, 'v' three floats; anything but '#', '\\r' and 'vt' is reported."""
    verts, idx, unsupported = [], [], []
    for line in open(path).read().split("\n")[:-1]:
        prop, _, rest = line.partition(" ")
        tok = rest.split()
        if prop == "f":
            idx += [int(t) - 1 for t in tok[:3]]
        elif prop == "v":
            verts += [np.float32(t) for t in tok[:3]]
        elif prop not in ("#", "\r", "vt"):
            unsupported.append(prop)
    return np.array(verts, np.float32).reshape(-1, 3), np.array(idx, np.int64).reshape(-1, 3), unsupported


def _mesh(colors):
    from humanrf_b200.toolbox.mesh_extraction import Mesh

    v, f, n = O.marching_cubes(sphere_lattice(16, 0.3), 0.0)
    c = np.random.default_rng(0).random(v.shape).astype(np.float32) if colors else None
    t = torch.from_numpy
    return Mesh(t(v), t(f), t(n), None if c is None else t(c))


@pytest.mark.parametrize("colors", [False, True])
def test_obj_round_trip(tmp_path, colors):
    from humanrf_b200.toolbox.mesh_extraction import write_obj

    m = _mesh(colors)
    write_obj(tmp_path / "m.obj", m)
    v, f, bad = parse_obj_like_the_renderer(tmp_path / "m.obj")
    assert bad == []
    assert np.array_equal(v.view(np.int32), m.vertices.numpy().view(np.int32))
    assert np.array_equal(f, m.faces.numpy())
    if colors:
        rgb = np.array([[np.float32(t) for t in l.split()[4:7]] for l in open(tmp_path / "m.obj") if l[0] == "v"])
        assert np.array_equal(rgb.astype(np.float32), m.colors.numpy())


@pytest.mark.parametrize("colors", [False, True])
def test_ply_round_trip(tmp_path, colors):
    from humanrf_b200.toolbox.mesh_extraction import write_ply

    m = _mesh(colors)
    write_ply(tmp_path / "m.ply", m)
    raw = open(tmp_path / "m.ply", "rb").read()
    head, body = raw.split(b"end_header\n", 1)
    lines = head.decode().split("\n")
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"]
    props = [l.split()[-1] for l in lines if l.startswith("property") and "list" not in l]
    types = {l.split()[-1]: ("<f4" if l.split()[1] == "float" else "u1") for l in lines if l.startswith("property")
             and "list" not in l}
    nv = int([l for l in lines if l.startswith("element vertex")][0].split()[-1])
    nf = int([l for l in lines if l.startswith("element face")][0].split()[-1])
    vd = np.dtype([(p, types[p]) for p in props])
    vr = np.frombuffer(body[:nv * vd.itemsize], vd)
    fr = np.frombuffer(body[nv * vd.itemsize:], np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    assert len(fr) == nf and (fr["n"] == 3).all()
    assert np.array_equal(np.stack([vr["x"], vr["y"], vr["z"]], 1), m.vertices.numpy())
    assert np.array_equal(np.stack([vr["nx"], vr["ny"], vr["nz"]], 1), m.normals.numpy())
    assert np.array_equal(fr["i"], m.faces.numpy())
    if colors:
        c = np.stack([vr["red"], vr["green"], vr["blue"]], 1)
        assert np.array_equal(c, np.rint(m.colors.numpy().astype(np.float64) * 255).astype(np.uint8))
    else:
        assert "red" not in props
