"""CPU restatement of the marching-cubes contract (include/humanrf_b200.h, hrf_marching_cubes_*) in numpy float32.

TEST INFRASTRUCTURE ONLY: the case table is generated here from the face rule, independently of the C++ generator in
csrc/mesh_extract.cu, and the mesh is built with the same vertex numbering, interpolation and face order, so the GPU
result can be compared bit for bit."""
import numpy as np

f32 = np.float32


# ------------------------------------------------------------------------------------------------------ case table
def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.int64)


def edge_corners(e):
    """Cube edge e = 4 * axis + idx: its lower and upper corner (corner c = a + 2b + 4d at (a, b, d))."""
    axis, idx = e >> 2, e & 3
    lo = [0, 0, 0]
    others = [a for a in range(3) if a != axis]
    lo[others[0]], lo[others[1]] = idx & 1, idx >> 1
    hi = list(lo)
    hi[axis] = 1
    return lo[0] + 2 * lo[1] + 4 * lo[2], hi[0] + 2 * hi[1] + 4 * hi[2]


EDGES = [edge_corners(e) for e in range(12)]


def _face_rule_segments(case):
    """Oriented segments (A -> B) on the six cube faces.  On a face with two crossing edges they are joined; with four
    (the ambiguous face) the two edges at each inside corner are joined, i.e. the inside corners are not connected.
    A -> B is oriented so that (mid B - mid A) x (inside corner of A - mid A) points into the cube."""
    inside = [(case >> c) & 1 for c in range(8)]
    cross = [inside[a] != inside[b] for a, b in EDGES]
    mid = [(corner_pos(a) + corner_pos(b)) / 2.0 for a, b in EDGES]
    nxt = {}
    for ax in range(3):
        for side in (0, 1):
            n_out = np.zeros(3)
            n_out[ax] = 2 * side - 1
            fe = [e for e in range(12) if (e >> 2) != ax and corner_pos(EDGES[e][0])[ax] == side]
            fc = [e for e in fe if cross[e]]
            if not fc:
                continue
            if len(fc) == 2:
                segs = [tuple(fc)]
            else:
                corners = [c for c in range(8) if corner_pos(c)[ax] == side and inside[c]]
                segs = [tuple(e for e in fe if c in EDGES[e]) for c in corners]
            for a, b in segs:
                ca = EDGES[a][0] if inside[EDGES[a][0]] else EDGES[a][1]
                d = np.cross(mid[b] - mid[a], corner_pos(ca) - mid[a]) @ n_out
                assert d != 0
                if d > 0:
                    a, b = b, a
                assert a not in nxt
                nxt[a] = b
    return cross, nxt


def _edge_faces(e):
    """The two cube faces (axis, side) edge e lies on."""
    p = corner_pos(EDGES[e][0])
    return {(a, int(p[a])) for a in range(3) if a != (e >> 2)}


def case_table():
    """(ntri [256] uint8, tri [256, 3 * max_tri] uint8 cube edges): each case's loops start at their smallest
    unused crossing edge, taken in ascending order.  A loop is fan-triangulated from its first vertex (in loop order)
    whose diagonals join no two edges of a common cube face: such a diagonal could also be drawn by the neighbouring
    cube across that face, and the shared mesh edge would then lie in four triangles."""
    tris = []
    for case in range(256):
        cross, nxt = _face_rule_segments(case)
        used, out = set(), []
        for e in range(12):
            if not cross[e] or e in used:
                continue
            loop = [e]
            x = nxt[e]
            while x != e:
                loop.append(x)
                x = nxt[x]
            used.update(loop)
            n = len(loop)
            for r in range(n):
                lr = loop[r:] + loop[:r]
                if all(not (_edge_faces(lr[0]) & _edge_faces(lr[i])) for i in range(2, n - 1)):
                    break
            else:
                raise AssertionError(f"case {case}: no fan origin")
            for i in range(1, n - 1):
                out.append((lr[0], lr[i], lr[i + 1]))
        tris.append(out)
    max_tri = max(len(t) for t in tris)
    ntri = np.array([len(t) for t in tris], np.uint8)
    tab = np.zeros((256, 3 * max_tri), np.uint8)
    for c, t in enumerate(tris):
        if t:
            tab[c, :3 * len(t)] = np.array(t, np.uint8).reshape(-1)
    return ntri, tab


NTRI, TRI = case_table()


# ---------------------------------------------------------------------------------------------------- extraction
def _gradient(sig, axis):
    """d sigma along `axis` (numpy axis of the [z][y][x] lattice): central differences, one-sided at the border."""
    s = np.moveaxis(sig, axis, 0)
    g = np.empty_like(s)
    g[1:-1] = (s[2:] - s[:-2]).astype(f32) * f32(0.5)
    g[0] = s[1] - s[0]
    g[-1] = s[-1] - s[-2]
    return np.moveaxis(g, 0, axis)


def marching_cubes(lattice, level, normals=True):
    """Mesh of {sigma >= level} on a float32 [(G+1)]^3 lattice indexed [z][y][x]: (vertices f32 [V,3],
    faces int32 [F,3], normals f32 [V,3] or None), in the order of the contract."""
    sig = np.ascontiguousarray(lattice, f32)
    G = sig.shape[0] - 1
    assert sig.shape == (G + 1,) * 3 and G >= 1
    level = f32(level)
    Gp = G + 1
    inside = sig >= level
    cross = np.zeros((Gp, Gp, Gp, 3), bool)            # [z][y][x][axis x,y,z]: edge owned by the lower endpoint
    cross[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    cross[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    cross[:-1, :, :, 2] = inside[:-1, :, :] != inside[1:, :, :]
    flat = cross.reshape(-1)
    ids = np.cumsum(flat, dtype=np.int64) - 1          # vertex id of (owner, axis) where it crosses
    sel = np.nonzero(flat)[0]
    owner, axis = sel // 3, sel % 3
    x, y, z = owner % Gp, (owner // Gp) % Gp, owner // (Gp * Gp)
    stride = np.array([1, Gp, Gp * Gp])[axis]
    sf = sig.reshape(-1)
    s0, s1 = sf[owner], sf[owner + stride]
    t = ((level - s0).astype(f32) / (s1 - s0).astype(f32)).astype(f32)
    Gf = f32(G)
    coord = np.stack([x, y, z], 1).astype(f32)
    base = ((coord / Gf).astype(f32) - f32(0.5)).astype(f32)
    along = ((coord[np.arange(sel.size), axis] + t).astype(f32) / Gf).astype(f32) - f32(0.5)
    verts = base.copy()
    verts[np.arange(sel.size), axis] = along.astype(f32)

    nrm = None
    if normals:
        grads = [_gradient(sig, 2).reshape(-1), _gradient(sig, 1).reshape(-1), _gradient(sig, 0).reshape(-1)]
        n = np.stack([-(g[owner] + (t * (g[owner + stride] - g[owner]).astype(f32)).astype(f32)).astype(f32)
                      for g in grads], 1).astype(f32)
        m = np.abs(n).max(1)
        ok = m > 0
        n[ok] = (n[ok] / m[ok, None]).astype(f32)
        ln = np.sqrt(((n[:, 0] * n[:, 0]).astype(f32) + (n[:, 1] * n[:, 1]).astype(f32)).astype(f32)
                     + (n[:, 2] * n[:, 2]).astype(f32)).astype(f32)
        n[ok] = (n[ok] / ln[ok, None]).astype(f32)
        n[~ok] = 0
        nrm = n

    # faces: cubes in linear order, triangles in table order
    ins = inside.astype(np.int64)
    case = np.zeros((G, G, G), np.int64)
    for c in range(8):
        a, b, d = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= ins[d:d + G, b:b + G, a:a + G] << c
    case = case.reshape(-1)
    nt = NTRI[case].astype(np.int64)
    cubes = np.nonzero(nt)[0]
    reps = nt[cubes]
    cube = np.repeat(cubes, reps)
    tri_i = np.arange(reps.sum()) - np.repeat(np.cumsum(reps) - reps, reps)
    ci, cj, ck = cube % G, (cube // G) % G, cube // (G * G)
    lo = np.array([edge_corners(e)[0] for e in range(12)])
    off = np.stack([lo & 1, (lo >> 1) & 1, lo >> 2], 1)
    faces = np.empty((cube.size, 3), np.int64)
    for q in range(3):
        e = TRI[case[cube], tri_i * 3 + q].astype(np.int64)
        ov = (ci + off[e, 0]) + Gp * ((cj + off[e, 1]) + Gp * (ck + off[e, 2]))
        faces[:, q] = ids[ov * 3 + (e >> 2)]
    return verts.astype(f32), faces.astype(np.int32), nrm


# ---------------------------------------------------------------------------------------------- mesh properties
def edge_use(faces):
    """{(a, b): count} of directed mesh edges."""
    f = np.asarray(faces, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    keys, cnt = np.unique(d[:, 0] * (1 << 32) + d[:, 1], return_counts=True)
    return keys, cnt


def is_closed_oriented(faces):
    """Every undirected edge in exactly two faces, with opposite windings."""
    keys, cnt = edge_use(faces)
    if (cnt != 1).any():
        return False
    a, b = keys >> 32, keys & 0xFFFFFFFF
    rev = b * (1 << 32) + a
    return bool(np.isin(rev, keys).all())


def euler_characteristic(verts, faces):
    f = np.asarray(faces, np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e = np.sort(e, 1)
    ne = np.unique(e[:, 0] * (1 << 32) + e[:, 1]).size
    return len(verts) - ne + len(f)


def components(num_vertices, faces):
    """Number of connected components of the face graph (vertices joined by faces)."""
    parent = np.arange(num_vertices)

    def find(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i

    for a, b, c in np.asarray(faces, np.int64):
        ra, rb, rc = find(a), find(b), find(c)
        parent[rb] = ra
        parent[find(rc)] = ra
    used = np.unique(np.asarray(faces).reshape(-1))
    return len({find(i) for i in used})


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)
