"""Numpy restatement of the visibility filter (nrw/reprojection.py, csrc/raster.cu), TEST INFRASTRUCTURE.

* `raster_depth`: the depth rasteriser of csrc/raster.cu operation for operation (camera coordinates, pixel rays,
  edge functions with the ascending-index tie rule, facing, z = D / sum(e), the clip range, float32 minimum).  With
  box=True every face tests the pixel box of csrc/raster.cu, with box=False every pixel of the image (brute force, to
  check that the box is conservative).
* `backproject`, `mark`: the back-projection from integer pixel coordinates and the nearest-point marking (through
  `eval_port.nn_brute`).
* `pipeline`: the whole `python -m nrw.reprojection` from already-read arrays.
* `load_reproj`: the unmodified reference modules utils.reproj_filter, tools.reproj_error and utils.colmap_utils.
"""
import numpy as np

from oracle import eval_port

_EPS = 2.0 ** -30


def camera_coords(v, V):
    """P = ((V[r,0]·x + V[r,1]·y) + V[r,2]·z) + V[r,3] per row"""
    v = np.asarray(v, np.float64)
    V = np.asarray(V, np.float64)
    return np.stack([((V[r, 0] * v[:, 0] + V[r, 1] * v[:, 1]) + V[r, 2] * v[:, 2]) + V[r, 3] for r in range(3)], 1)


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def _box_axis(lo, hi, n):
    l = np.ceil(lo - (0.5625 + np.abs(lo) * _EPS))
    h = np.floor(hi + (np.abs(hi) * _EPS - 0.4375))
    return np.fmin(np.fmax(l, 0.0), float(n)).astype(np.int64), np.fmax(np.fmin(h, float(n - 1)), -1.0).astype(np.int64)


def face_setup(P, f, H, W, fx, fy, cx, cy, znear, zfar, cull, box=True):
    """-> dict of the drawn faces: id, m [n,3,3] (σ-signed), tie [n,3], D [n], box c0 c1 r0 r1 [n]; and the bad flag"""
    f = np.asarray(f, np.int64).reshape(-1, 3)
    nv = P.shape[0]
    bad = ((f < 0) | (f >= nv)).any(1)
    fid = np.nonzero(~bad)[0]
    g = f[fid]
    p = [P[g[:, k]] for k in range(3)]
    z = np.stack([q[:, 2] for q in p], 1)
    zmin, zmax = np.fmin(np.fmin(z[:, 0], z[:, 1]), z[:, 2]), np.fmax(np.fmax(z[:, 0], z[:, 1]), z[:, 2])
    c = _cross(p[1], p[2])
    D = (p[0][:, 0] * c[:, 0] + p[0][:, 1] * c[:, 1]) + p[0][:, 2] * c[:, 2]
    keep = ~((zmax < znear) | (zmin > zfar)) & (D != 0)
    if cull:
        keep &= ~(D >= 0)
    m = np.empty((len(g), 3, 3))
    tie = np.empty((len(g), 3), bool)
    for k in range(3):
        a, b = g[:, k], g[:, (k + 1) % 3]
        asc = a < b
        lo = np.where(asc[:, None], p[k], p[(k + 1) % 3])
        hi = np.where(asc[:, None], p[(k + 1) % 3], p[k])
        m[:, k] = _cross(lo, hi) * np.where(asc, 1.0, -1.0)[:, None]
        tie[:, k] = asc
    c0, c1 = np.zeros(len(g), np.int64), np.full(len(g), W - 1, np.int64)
    r0, r1 = np.zeros(len(g), np.int64), np.full(len(g), H - 1, np.int64)
    if box:
        front = zmin > 0
        with np.errstate(all="ignore"):
            u = np.stack([(q[:, 0] / q[:, 2]) * fx + cx for q in p], 1)
            v = np.stack([(q[:, 1] / q[:, 2]) * fy + cy for q in p], 1)
        ua, ub = _box_axis(np.fmin(np.fmin(u[:, 0], u[:, 1]), u[:, 2]), np.fmax(np.fmax(u[:, 0], u[:, 1]), u[:, 2]), W)
        va, vb = _box_axis(np.fmin(np.fmin(v[:, 0], v[:, 1]), v[:, 2]), np.fmax(np.fmax(v[:, 0], v[:, 1]), v[:, 2]), H)
        c0, c1 = np.where(front, ua, c0), np.where(front, ub, c1)
        r0, r1 = np.where(front, va, r0), np.where(front, vb, r1)
    keep &= (c0 <= c1) & (r0 <= r1)
    s = np.nonzero(keep)[0]
    return {"id": fid[s], "m": m[s], "tie": tie[s], "D": D[s], "c0": c0[s], "c1": c1[s], "r0": r0[s], "r1": r1[s]}, bool(bad.any())


def raster_depth(v, f, V, fx, fy, cx, cy, H, W, znear=0.05, zfar=100.0, cull=True, box=True, chunk=1 << 22, counts=False):
    """-> (depth float32 [H, W], bad face index flag) and with counts=True the number of faces that cover each pixel
    inside the clip range, int64 [H, W]"""
    P = camera_coords(v, V)
    F, bad = face_setup(P, f, H, W, fx, fy, cx, cy, znear, zfar, cull, box)
    rx = ((np.arange(W, dtype=np.float64) + 0.5) - cx) / fx
    ry = ((np.arange(H, dtype=np.float64) + 0.5) - cy) / fy
    depth = np.full(H * W, np.inf, np.float32)
    cover = np.zeros(H * W, np.int64)
    w = F["c1"] - F["c0"] + 1
    area = w * (F["r1"] - F["r0"] + 1)
    start = 0
    while start < len(area):
        csum = np.cumsum(area[start:])
        stop = start + max(1, int(np.searchsorted(csum, chunk, side="right")))
        sl = slice(start, stop)
        a = area[sl]
        j = np.repeat(np.arange(start, stop), a)
        t = np.arange(int(a.sum())) - np.repeat(np.cumsum(a) - a, a)
        r = F["r0"][j] + t // w[j]
        c = F["c0"][j] + t % w[j]
        dx, dy = rx[c], ry[r]
        D = F["D"][j]
        e = []
        inside = np.ones(len(j), bool)
        for k in range(3):
            m = F["m"][j, k]
            ek = (m[:, 0] * dx + m[:, 1] * dy) + m[:, 2]
            inside &= np.where(D < 0, ek < 0, ek > 0) | ((ek == 0) & F["tie"][j, k])
            e.append(ek)
        with np.errstate(all="ignore"):
            z = D / ((e[0] + e[1]) + e[2])
        ok = inside & (z >= znear) & (z <= zfar)
        np.minimum.at(depth, (r * W + c)[ok], z[ok].astype(np.float32))
        if counts:
            np.add.at(cover, (r * W + c)[ok], 1)
        start = stop
    depth[np.isinf(depth)] = 0.0
    if counts:
        return depth.reshape(H, W), bad, cover.reshape(H, W)
    return depth.reshape(H, W), bad


def backproject(depth, fx, fy, cx, cy, pose):
    """world points [n,3] of the pixels with depth > 0 in raster order"""
    r, c = np.nonzero(depth > 0)
    z = depth[r, c].astype(np.float64)
    xc, yc = ((c - cx) / fx) * z, ((r - cy) / fy) * z
    p = np.asarray(pose, np.float64)
    return np.stack([((p[k, 0] * xc + p[k, 1] * yc) + p[k, 2] * z) + p[k, 3] for k in range(3)], 1)


def mark(visible, target, X, threshold):
    """visible[nearest target point] = True for every X closer than threshold"""
    if len(X):
        d, i = eval_port.nn_brute(target, X)
        visible[i[d < threshold]] = True
    return visible


def pipeline(verts, faces, points, colors, intrinsics, extrinsics, whs, voxel_size=0.01, znear=0.05, zfar=100.0):
    """the rows of reprojected.ply: np.unique([xyz, rgb], axis=0) of the visible target points"""
    visible = np.zeros(len(points), bool)
    thr = 2 * np.sqrt(2) * voxel_size
    for K, E, (w, h) in zip(intrinsics, extrinsics, whs):
        fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        depth, _ = raster_depth(verts, faces, E, fx, fy, cx, cy, h, w, znear, zfar, True)
        mark(visible, points, backproject(depth, fx, fy, cx, cy, np.linalg.inv(E)), thr)
    return np.unique(np.hstack([points[visible], colors[visible]]), axis=0)


def load_reproj(data_path="."):
    """the unmodified utils.reproj_filter (which parses sys.argv at import; it is patched to carry `--data_path`),
    tools.reproj_error and utils.colmap_utils of the reference.  Third-party packages that are not installed are inert
    stand-ins (oracle.ref_import)."""
    import sys
    import types
    import warnings
    from unittest import mock

    from oracle import ref_import

    if not ref_import.available():
        raise RuntimeError(f"reference tree not present at {ref_import.REF_ROOT}")
    ref_import._install_stubs()
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    with warnings.catch_warnings(), mock.patch.object(sys, "argv", ["reproj_filter.py", "--data_path", str(data_path)]):
        warnings.simplefilter("ignore")
        import utils.colmap_utils as colmap_utils  # type: ignore
        import tools.reproj_error as reproj_error  # type: ignore
        import utils.reproj_filter as reproj_filter  # type: ignore
    return types.SimpleNamespace(reproj_filter=reproj_filter, reproj_error=reproj_error, colmap_utils=colmap_utils)
