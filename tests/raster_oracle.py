"""numpy restatement of hrf_rasterize_mesh and hrf_depth_metrics (include/humanrf_b200.h, DESIGN.md §3.12), operation
for operation: float64 projection, 8-bit fixed point, exact int64 edge functions with the tie rule, float64 depth
rounded to float32, and the least (z bits << 32 | face) key per pixel."""
import numpy as np

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
MAX_FIXED = 536870912.0        # 2^21 pixels in 8-bit fixed point


def project(V, M, fx, fy, cx, cy, near):
    """Per vertex: U, V (int64 fixed point), Z (float64) and ok (False: in front of near, non-finite or beyond
    +-2^21 pixels)."""
    p = np.asarray(V, F32).astype(np.float64)
    M = np.asarray(M, np.float64).reshape(3, 4)
    c = [((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) + M[r, 3] for r in range(3)]
    with np.errstate(all="ignore"):
        u = (fx * c[0]) / c[2] + cx
        v = (fy * c[1]) / c[2] + cy
        us, vs = u * 256.0, v * 256.0
        ok = (c[2] >= near) & (c[2] <= np.finfo(np.float64).max) & (np.abs(us) <= MAX_FIXED) & (np.abs(vs) <= MAX_FIXED)
    U = np.where(ok, np.rint(np.where(ok, us, 0)), 0).astype(np.int64)
    Vv = np.where(ok, np.rint(np.where(ok, vs, 0)), 0).astype(np.int64)
    return U, Vv, c[2], ok


def setup(U, Vv, ok, F, W, H):
    """Per face: status (0 drawn, 1 index out of range, 2 skipped, 3 zero area, 4 box off the image) and the clipped box
    (x0, y0, x1, y1), inclusive."""
    F = np.asarray(F, np.int64).reshape(-1, 3)
    nv = len(U)
    status = np.zeros(len(F), np.int64)
    bad = ((F < 0) | (F >= nv)).any(1)
    status[bad] = 1
    Fi = np.where(bad[:, None], 0, F)
    skip = ~bad & ~ok[Fi].all(1) if nv else np.zeros(len(F), bool)
    status[skip] = 2
    live = status == 0
    x, y = U[Fi] if nv else np.zeros((len(F), 3), np.int64), Vv[Fi] if nv else np.zeros((len(F), 3), np.int64)
    A = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
    status[live & (A == 0)] = 3
    x0 = np.maximum((x.min(1) + 127) >> 8, 0)
    x1 = np.minimum((x.max(1) - 128) >> 8, W - 1)
    y0 = np.maximum((y.min(1) + 127) >> 8, 0)
    y1 = np.minimum((y.max(1) - 128) >> 8, H - 1)
    status[(status == 0) & ((x0 > x1) | (y0 > y1))] = 4
    return status, x, y, A, np.stack([x0, y0, x1, y1], 1)


def tie_inside(dx, dy):
    return (dy > 0) | ((dy == 0) & (dx < 0))


def fragments(x, y, A, Z3, fi, px, py):
    """For pairs (face fi, pixel (px, py)): covered (bool) and z (float32) per the contract's steps 3 and 4."""
    xf, yf, Af = x[fi], y[fi], A[fi]
    sg = np.where(Af < 0, -1, 1).astype(np.int64)
    sx, sy = 256 * px.astype(np.int64) + 128, 256 * py.astype(np.int64) + 128
    E, inside = [], np.ones(len(fi), bool)
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        dx, dy = xf[:, b] - xf[:, a], yf[:, b] - yf[:, a]
        e = sg * (dx * (sy - yf[:, a]) - dy * (sx - xf[:, a]))
        inside &= (e > 0) | ((e == 0) & tie_inside(sg * dx, sg * dy))
        E.append(e)
    Ad = (sg * Af).astype(np.float64)
    Zf = Z3[fi]
    with np.errstate(all="ignore"):
        b = [e.astype(np.float64) / Ad for e in E]
        s = (b[0] / Zf[:, 0] + b[1] / Zf[:, 1]) + b[2] / Zf[:, 2]
        z = (1.0 / s).astype(F32)
    return inside, z


def _pairs(box, faces):
    """Every (face, pixel) of the faces' clipped boxes, row-major within each box."""
    bw = box[faces, 2] - box[faces, 0] + 1
    bh = box[faces, 3] - box[faces, 1] + 1
    cnt = bw * bh
    fi = np.repeat(faces, cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    p = np.arange(cnt.sum()) - start
    bwr = np.repeat(bw, cnt)
    return fi, box[fi, 0] + p % bwr, box[fi, 1] + p // bwr


def raster_fixed(U, Vv, Z, ok, F, W, H, near, far):
    """The contract from snapped vertices on: dict of z f32 [H,W], mask u8, face i32, hits i32, error, skipped."""
    status, x, y, A, box = setup(U, Vv, ok, F, W, H)
    Z3 = np.asarray(Z, np.float64)[np.where((status == 1)[:, None], 0, np.asarray(F, np.int64).reshape(-1, 3))] \
        if len(Z) else np.zeros((len(status), 3))
    keys = np.full(W * H, EMPTY, np.uint64)
    hits = np.zeros(W * H, np.int32)
    drawn = np.nonzero(status == 0)[0]
    for s in range(0, len(drawn), 4096):
        fi, px, py = _pairs(box, drawn[s:s + 4096])
        inside, z = fragments(x, y, A, Z3, fi, px, py)
        fi, px, py, z = fi[inside], px[inside], py[inside], z[inside]
        pix = py * W + px
        np.add.at(hits, pix, 1)
        keep = (z.astype(np.float64) >= near) & (z.astype(np.float64) <= far)
        k = (z[keep].view(np.uint32).astype(np.uint64) << np.uint64(32)) | fi[keep].astype(np.uint64)
        np.minimum.at(keys, pix[keep], k)
    hit = keys != EMPTY
    z = np.where(hit, (keys >> np.uint64(32)).astype(np.uint32), 0).astype(np.uint32).view(F32)
    face = np.where(hit, (keys & np.uint64(0xFFFFFFFF)).astype(np.int64), -1).astype(np.int32)
    return dict(z=z.reshape(H, W), mask=(hit.astype(np.uint8) * 255).reshape(H, W), face=face.reshape(H, W),
                hits=hits.reshape(H, W), error=int((status == 1).any()), skipped=int((status == 2).sum()))


def rasterize(V, F, M, fx, fy, cx, cy, W, H, near=0.01, far=100.0):
    U, Vv, Z, ok = project(V, M, fx, fy, cx, cy, near)
    return raster_fixed(U, Vv, Z, ok, F, W, H, near, far)


def rasterize_pixels(V, F, M, fx, fy, cx, cy, W, H, px, py, near=0.01, far=100.0):
    """z, face and hits of the listed pixels only (for large meshes): each pixel against every face whose box holds it."""
    U, Vv, Z, ok = project(V, M, fx, fy, cx, cy, near)
    status, x, y, A, box = setup(U, Vv, ok, F, W, H)
    Fl = np.asarray(F, np.int64).reshape(-1, 3)
    drawn = np.nonzero(status == 0)[0]
    bd = box[drawn]
    Z3 = Z[Fl[drawn]]
    xd, yd, Ad = x[drawn], y[drawn], A[drawn]
    out_z, out_f, out_h = np.zeros(len(px), F32), np.full(len(px), -1, np.int32), np.zeros(len(px), np.int32)
    for i, (qx, qy) in enumerate(zip(px, py)):
        c = np.nonzero((bd[:, 0] <= qx) & (qx <= bd[:, 2]) & (bd[:, 1] <= qy) & (qy <= bd[:, 3]))[0]
        inside, z = fragments(xd, yd, Ad, Z3, c, np.full(len(c), qx), np.full(len(c), qy))
        out_h[i] = inside.sum()
        keep = inside & (z.astype(np.float64) >= near) & (z.astype(np.float64) <= far)
        if keep.any():
            k = (z[keep].view(np.uint32).astype(np.uint64) << np.uint64(32)) | drawn[c[keep]].astype(np.uint64)
            best = k.min()
            out_z[i] = np.uint32(best >> np.uint64(32)).view(F32)
            out_f[i] = int(best & np.uint64(0xFFFFFFFF))
    return out_z, out_f, out_h


def depth_scores(pred_z, pred_mask, ref_z, ref_mask, taus):
    """float64 restatement: (out [4], counts [5 + T], error); out NaN when B is empty or error."""
    pz, rz = np.asarray(pred_z, F32).reshape(-1), np.asarray(ref_z, F32).reshape(-1)
    pm, rm = np.asarray(pred_mask).reshape(-1) != 0, np.asarray(ref_mask).reshape(-1) != 0
    B = pm & rm
    with np.errstate(all="ignore"):
        good = (pz > 0) & np.isfinite(pz) & (rz > 0) & np.isfinite(rz)
    err = int((B & ~good).any())
    sel = B & good
    d = pz[sel].astype(np.float64) - rz[sel].astype(np.float64)
    ad = np.abs(d)
    n = int(B.sum())
    counts = [n, int(pm.sum()), int(rm.sum()), int(B.sum()), int((pm | rm).sum())] + [int((ad <= t).sum()) for t in taus]
    if err or n == 0:
        out = np.full(4, np.nan)
    else:
        out = np.array([d.sum() / n, ad.sum() / n, np.sqrt((d * d).sum() / n), (ad / rz[sel].astype(np.float64)).sum() / n])
    sums = [np.abs(d).sum(), ad.sum(), (d * d).sum(), (ad / rz[sel].astype(np.float64)).sum()] if sel.any() else [0.0] * 4
    return out, np.array(counts, np.int64), err, sums


# ------------------------------------------------------------------------------------------------------- test scenes
class Camera:
    """A CameraData-like camera."""

    def __init__(self, width, height, rotation_axisangle, translation, focal_length, principal_point, name=None):
        self.width, self.height = width, height
        self.rotation_axisangle = np.asarray(rotation_axisangle, np.float64)
        self.translation = np.asarray(translation, np.float64)
        self.focal_length = np.asarray(focal_length, np.float64)
        self.principal_point = np.asarray(principal_point, np.float64)
        self.name = name


def pixel_camera(W, H):
    """Identity pose, fxW = fyH = 1 and the principal point at the corner, for power-of-two W and H: a point (X, Y, 1)
    lands on u = X, v = Y exactly."""
    return Camera(W, H, (0, 0, 0), (0, 0, 0), (1.0 / W, 1.0 / H), (0.0, 0.0))


def look_at(W, H, pos, target=(0, 0, 0), f=1.2, seed=0):
    """A camera at `pos` looking at `target` (RDF), focal f (relative to the width) and a jittered principal point."""
    rng = np.random.default_rng(seed)
    pos, target = np.asarray(pos, np.float64), np.asarray(target, np.float64)
    fwd = target - pos
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0.0, -1.0, 0.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    from scipy.spatial.transform import Rotation

    aa = Rotation.from_matrix(np.stack([right, down, fwd], 1)).as_rotvec()
    return Camera(W, H, aa, pos, (f, f * W / H), (0.5 + rng.uniform(-0.05, 0.05), 0.5 + rng.uniform(-0.05, 0.05)))


def random_rotation(seed):
    q = np.random.default_rng(seed).normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def quad_grid(nx, ny, W, H, seed, split="both", centres=True):
    """A plane z = 1 seen by ``pixel_camera(W, H)``, tiled by nx x ny jittered quads, each split into two triangles
    along one diagonal (alternating with `split` = "both").  The outer boundary is the rectangle [1.3, W - 1.3] x
    [1.3, H - 1.3] (no pixel centre on it); with `centres`, a third of the interior vertices sit exactly on pixel
    centres and one interior grid line runs through a column of pixel centres.  Returns V f32 [n,3], F i32 [m,3]."""
    rng = np.random.default_rng(seed)
    xs = np.linspace(1.3, W - 1.3, nx + 1)
    ys = np.linspace(1.3, H - 1.3, ny + 1)
    X, Y = np.meshgrid(xs, ys)
    dx, dy = (xs[1] - xs[0]) * 0.2, (ys[1] - ys[0]) * 0.2
    inner = np.zeros_like(X, bool)
    inner[1:-1, 1:-1] = True
    X = np.where(inner, X + rng.uniform(-dx, dx, X.shape), X)
    Y = np.where(inner, Y + rng.uniform(-dy, dy, Y.shape), Y)
    if centres:
        on = inner & (rng.random(X.shape) < 1 / 3)
        X = np.where(on, np.floor(X) + 0.5, X)
        Y = np.where(on, np.floor(Y) + 0.5, Y)
        col = nx // 2
        X[1:-1, col] = np.floor(xs[col]) + 0.5                # a vertical line through pixel centres
    X, Y = np.round(X * 256) / 256, np.round(Y * 256) / 256  # on the fixed-point grid
    V = np.stack([X, Y, np.ones_like(X)], -1).reshape(-1, 3).astype(F32)
    idx = np.arange((nx + 1) * (ny + 1)).reshape(ny + 1, nx + 1)
    F = []
    for j in range(ny):
        for i in range(nx):
            a, b, c, d = idx[j, i], idx[j, i + 1], idx[j + 1, i + 1], idx[j + 1, i]
            if split == "main" or (split == "both" and (i + j) % 2 == 0):
                F += [(a, b, c), (a, c, d)]
            else:
                F += [(a, b, d), (b, c, d)]
    return V, np.array(F, np.int32)
