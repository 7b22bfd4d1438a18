"""Mesh extraction on the H100 (csrc/occupancy_bake.cu density_lattice_kernel, csrc/mesh_extract.cu,
toolbox/mesh_extraction.py): the fused lattice against the public query-form density, marching cubes against the CPU
oracle, and the user-visible claims on the confined teacher, whose surface is known."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import mc_oracle as O
from test_learned_occupancy_gpu import _sharp_pair, _sphere, confined_teacher
from test_mesh_extraction_cpu import parse_obj_like_the_renderer, random_lattice, sphere_lattice

pytestmark = pytest.mark.gpu

RADII = np.array([0.2, 0.3, 0.15])


def unfused_lattice(m, frame, mask, G):
    """Vertex positions built in torch -> HumanRF.density (query form) at the corners of occupied voxels, 0 elsewhere."""
    from humanrf_b200.scene_representation.query_io import QueryInput

    dev = m.sigma_net.params.device
    if mask is None:
        corner = torch.ones((G + 1,) * 3, dtype=torch.bool, device=dev)
    else:
        occ = Fn.pad((mask != 0).float()[None, None], (1, 1, 1, 1, 1, 1))
        corner = Fn.max_pool3d(occ, 2, stride=1)[0, 0] > 0
    z, y, x = torch.nonzero(corner, as_tuple=True)
    # a device tensor divisor: torch turns division by a host scalar into a multiplication by its reciprocal, which
    # rounds differently unless G is a power of two
    Gt = torch.tensor(float(G), dtype=torch.float32, device=dev)
    pos = torch.stack([i.to(torch.float32) / Gt - 0.5 for i in (x, y, z)], -1).contiguous()
    out = torch.zeros((G + 1,) * 3, dtype=torch.float32, device=dev)
    with torch.no_grad():
        out[z, y, x] = m.density(QueryInput(is_training=False, positions=pos, frame_numbers=torch.full(
            (pos.shape[0],), frame, dtype=torch.int32, device=dev))).density
    return out


CASES = [((50,), 64, (15, 64), 0, True), ((50,), 256, (40,), 0, True), ((100, 100, 50), 64, (114, 115, 214, 215), 0, True),
         ((100, 100, 50), 256, (114, 115), 0, True), ((50,), 64, (15, 30), 2, True), ((50,), 64, (20,), 0, False),
         ((100, 100, 50), 96, (114, 115), 0, False)]


@pytest.mark.parametrize("segs,G,frames,cam_emb,masked", CASES, ids=[
    "seg50-G64", "seg50-G256", "seg100x2-50-G64", "seg100x2-50-G256", "seg50-G64-camemb2", "seg50-G64-dense",
    "seg100x2-50-G96-dense"])
def test_lattice_equals_unfused_bitwise(cuda, segs, G, frames, cam_emb, masked):
    from humanrf_b200.synthetic_scene import ellipsoid_grid
    from humanrf_b200.toolbox.mesh_extraction import density_lattice

    _, m, _ = _sharp_pair(segs, cuda, cam_emb)
    mask = torch.from_numpy(ellipsoid_grid(G)).to(cuda) if masked else None
    for frame in frames:
        lat = density_lattice(m, frame, mask) if masked else density_lattice(m, frame, resolution=G)
        ref = unfused_lattice(m, frame, mask, G)
        torch.cuda.synchronize()
        assert lat.shape == (G + 1,) * 3 and lat.dtype == torch.float32
        assert torch.equal(lat.view(torch.int32), ref.view(torch.int32)), f"{int((lat != ref).sum())} vertices differ"
        if masked:
            assert torch.equal(density_lattice(m, frame, mask, resolution=G), lat)
        print(f"segs={segs} G={G} frame={frame} mask={masked}: {int((lat != 0).sum())} evaluated vertices")


def _mc_equals_oracle(lat_np, level):
    from humanrf_b200.toolbox.mesh_extraction import marching_cubes

    v, f, n = O.marching_cubes(lat_np, level)
    lat = torch.from_numpy(lat_np).cuda()
    a = marching_cubes(lat, level)
    b = marching_cubes(lat, level)
    av, af, an = a.vertices.cpu().numpy(), a.faces.cpu().numpy(), a.normals.cpu().numpy()
    assert av.shape == v.shape and af.shape == f.shape, (av.shape, v.shape, af.shape, f.shape)
    assert np.array_equal(av.view(np.int32), v.view(np.int32))
    assert np.array_equal(af, f)
    assert np.abs(an - n).max(initial=0) <= 1e-5
    for x, y in ((a.vertices, b.vertices), (a.faces, b.faces), (a.normals, b.normals)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))     # identical bytes
    c = marching_cubes(lat, level, normals=False)
    assert c.normals is None and torch.equal(c.faces, a.faces) and torch.equal(c.vertices, a.vertices)
    return v, f


@pytest.mark.parametrize("seed", [0, 1])
def test_marching_cubes_random_lattices_equal_oracle(cuda, seed):
    lat = random_lattice(32, seed)
    v, f = _mc_equals_oracle(lat, 0.0)
    print(f"random G=32 seed {seed}: {len(v)} vertices {len(f)} faces")


def test_marching_cubes_sphere_and_model_lattice_equal_oracle(cuda):
    from humanrf_b200.toolbox.mesh_extraction import density_lattice

    _mc_equals_oracle(sphere_lattice(128, 0.3), 0.0)
    _, m, _ = _sharp_pair((50,), cuda)
    lat = density_lattice(m, 20, resolution=48)
    level = float(torch.quantile(lat.double().flatten(), 0.5))
    v, f = _mc_equals_oracle(lat.cpu().numpy(), level)
    assert len(f) > 0


def _ellipsoid_distance(p):
    """Distance of points p [n,3] to the surface of the ellipsoid with RADII (closest point x_i = p_i r_i^2 /
    (r_i^2 + lam), lam by bisection)."""
    p = np.asarray(p, np.float64)
    r2 = RADII ** 2
    lo, hi = np.full(len(p), -r2.min() + 1e-12), np.full(len(p), 10.0)
    for _ in range(200):
        lam = (lo + hi) / 2
        g = ((p * RADII / (r2 + lam[:, None])) ** 2).sum(1) - 1
        lo, hi = np.where(g > 0, lam, lo), np.where(g > 0, hi, lam)
    x = p * r2 / (r2 + lam[:, None])
    return np.linalg.norm(p - x, axis=1)


def test_confined_teacher_mesh(cuda):
    """sigma = 100 e^{12 s}, s = trilinear of a +-1 sign grid of the ellipsoid E on the dense level 0: sigma = 100 is the
    sign field's zero set, which lies within one level-0 cell diagonal (sqrt(3) / scale0) of E's surface; marching
    cubes adds at most one lattice spacing (1/G)."""
    from humanrf_b200.scene_representation.query_io import QueryInput
    from humanrf_b200.toolbox.mesh_extraction import extract_mesh

    m = confined_teacher(cuda)
    G, frame = 128, 17
    hull = torch.from_numpy(_sphere(G)).to(cuda)
    mesh = extract_mesh(m, frame, hull, 100.0, colors=True)
    v, f = mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy()
    assert O.is_closed_oriented(f)
    assert O.components(len(v), f) == 1 and O.euler_characteristic(v, f) == 2
    scale0 = float(m.feature_grids[0].layout.scale[0])
    d = _ellipsoid_distance(v)
    band = np.sqrt(3) / scale0 + 1 / G
    assert d.max() <= band, (d.max(), band)
    # the mesh lies in a shell of half-width `band` around E's surface, so its volume differs from E's by at most the
    # shell's volume, about area(E) * band (Knud Thomsen's area formula, within 1.1 %, taken with 2 % slack)
    a, b, c = RADII
    pk = 1.6075
    area = 4 * np.pi * (((a * b) ** pk + (a * c) ** pk + (b * c) ** pk) / 3) ** (1 / pk) * 1.02
    vol, ref = O.signed_volume(v, f), 4 / 3 * np.pi * a * b * c
    assert abs(vol - ref) <= area * band, (vol, ref, area * band)
    # colours: HumanRF.forward in evaluation mode at the vertices, looking along -normal
    n = mesh.vertices.shape[0]
    out = m.forward(QueryInput(is_training=False, positions=mesh.vertices, directions=-mesh.normals,
                               frame_numbers=torch.full((n,), frame, dtype=torch.int32, device=cuda)))
    assert torch.equal(mesh.colors, out.radiance)
    print(f"confined teacher G={G}: {len(v)} vertices {len(f)} faces, max distance {d.max():.4f} (band {band:.4f}), "
          f"volume {vol:.5f} vs {ref:.5f} (tolerance {area * band:.5f})")


def test_export_mesh_sequence(cuda, tmp_path):
    from humanrf_b200.dataset.data_loader import DataLoader as DL
    from humanrf_b200.synthetic_scene import SyntheticDataset
    from humanrf_b200.toolbox.learned_occupancy import bake_occupancy_grid
    from humanrf_b200.toolbox.mesh_extraction import export_mesh_sequence, extract_mesh, to_world

    m = confined_teacher(cuda)
    ds = SyntheticDataset(G=64)
    ds._grids = {f: _sphere(64) for f in ds.frames}
    dl = DL(dataset=ds, device="cuda", mode=DL.Mode.TEST, dataloader_output_mode=DL.OutputMode.RAYS_AND_SAMPLES,
            space_pruning_mode=DL.SpacePruningMode.OCCUPANCY_GRID, batch_size=64 * 48, camera_numbers=(0, 1),
            frame_numbers=tuple(ds.frames), max_buffer_size=1, render_sequence=[(0, 15)])
    frames = (15, 16)
    paths = export_mesh_sequence(m, dl.dataset, frames, tmp_path / "objs", 100.0)
    assert [p.split("/")[-1] for p in paths] == ["frame000015.obj", "frame000016.obj"]
    assert sorted(x.name for x in (tmp_path / "objs").iterdir()) == ["frame000015.obj", "frame000016.obj"]
    for frame, path in zip(frames, paths):
        hull = torch.from_numpy(_sphere(64)).to(cuda)
        ref = to_world(extract_mesh(m, frame, bake_occupancy_grid(m, frame, hull), 100.0), dl.scene_offset,
                       dl.scene_scale)
        v, f, bad = parse_obj_like_the_renderer(path)
        assert bad == [] and len(f) > 0
        assert np.array_equal(v.view(np.int32), ref.vertices.cpu().numpy().view(np.int32))
        assert np.array_equal(f, ref.faces.cpu().numpy())
        # world units: the normalised mesh maps back inside the dataset's box
        assert (v >= ds.aabb[0] - 1e-4).all() and (v <= ds.aabb[1] + 1e-4).all()
    with pytest.raises(RuntimeError):
        export_mesh_sequence(m, ds, (15, 99), tmp_path / "bad", 100.0)
    assert not (tmp_path / "bad" / "frame000015.obj").exists()


def test_mesh_extraction_rejects_bad_inputs(cuda):
    from humanrf_b200.toolbox.mesh_extraction import density_lattice, extract_mesh, marching_cubes

    from helpers import make_pair

    _, m, frames = make_pair((6,), device=cuda)
    good = torch.from_numpy(_sphere(16)).to(cuda)
    assert density_lattice(m, frames[0], good).shape == (17, 17, 17)
    bad = [good.float(), good.bool(), good[:, :, :8].contiguous(), good[0], good.cpu(), good.transpose(0, 2),
           good.cpu().numpy()]
    for h in bad:
        with pytest.raises(RuntimeError):
            density_lattice(m, frames[0], h)
        with pytest.raises(RuntimeError):
            extract_mesh(m, frames[0], h, 1.0)
    for f in (frames[0] - 1, frames[-1] + 1, -1, 10 ** 6):
        with pytest.raises(RuntimeError):
            density_lattice(m, f, good)
        with pytest.raises(RuntimeError):
            extract_mesh(m, f, good, 1.0)
    for G in (0, 1025):
        with pytest.raises(RuntimeError):
            density_lattice(m, frames[0], resolution=G)
    with pytest.raises(RuntimeError):
        density_lattice(m, frames[0])
    with pytest.raises(RuntimeError):
        density_lattice(m, frames[0], good, resolution=8)
    lat = density_lattice(m, frames[0], good)
    for bad_lat in (lat.double(), lat.cpu(), lat[:, :, :8], lat.transpose(0, 2), lat[0], lat[:1, :1, :1].contiguous()):
        with pytest.raises(RuntimeError):
            marching_cubes(bad_lat, 1.0)
    with pytest.raises(RuntimeError):
        marching_cubes(lat, float("nan"))
