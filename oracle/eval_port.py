"""Numpy restatement of the evaluation (nrw/evaluation.py, csrc/nnsearch.cu), TEST INFRASTRUCTURE.

* `nn_brute`: exact 1-NN by brute force in chunks, d2 = (dx*dx + dy*dy) + dz*dz, dist = sqrt(d2), the smallest index
  among equally near points (np.argmin returns the first minimum).
* `sample_points`: the sampling rules of csrc/nnsearch.cu (splitmix64 uniforms, tiled prefix sums, upper-bound face pick,
  barycentric point), operation for operation.
* `bbx_crop`, `box_crop`, `mesh_crop`, `point_crop`, `compute`: the crops and metrics of utils/eval_utils.py.
* `load_eval`: the unmodified reference modules utils.eval_utils and utils.eval_mesh (see oracle/ref_import.py).
"""
import numpy as np

MS_TILE = 1024
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def nn_brute(ref, q, chunk=2048):
    """for every row of q the (dist, index) of its nearest row of ref"""
    ref = np.asarray(ref, np.float64)
    q = np.asarray(q, np.float64)
    dist = np.empty(len(q))
    idx = np.empty(len(q), np.int64)
    for a in range(0, len(q), chunk):
        d = q[a:a + chunk, None, :] - ref[None, :, :]
        d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]
        i = np.argmin(d2, axis=1)
        idx[a:a + chunk] = i
        dist[a:a + chunk] = np.sqrt(d2[np.arange(len(i)), i])
    return dist, idx


def uniforms(seed, ctr):
    """(splitmix64(seed + ctr * golden) >> 11) * 2^-53 for an array of counters"""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.asarray(ctr, np.uint64) * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def face_areas(v, f):
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return 0.5 * np.sqrt(cx * cx + cy * cy + cz * cz)


def area_prefix(areas):
    """tiled prefix sum: sequential inside tiles of MS_TILE, sequential exclusive sum of the tile totals"""
    n = len(areas)
    t = (n + MS_TILE - 1) // MS_TILE
    pad = np.zeros(t * MS_TILE)
    pad[:n] = areas
    local = np.cumsum(pad.reshape(t, MS_TILE), axis=1)
    tot = local[np.arange(t), np.minimum(MS_TILE, n - np.arange(t) * MS_TILE) - 1]
    off = np.concatenate([[0.0], np.cumsum(tot)[:-1]])
    out = local.copy()
    out[1:] = off[1:, None] + local[1:]
    return out.reshape(-1)[:n]


def sample_points(v, f, n, seed=0):
    """-> (points f64 [n,3], face ids int64 [n])"""
    v = np.asarray(v, np.float64)
    f = np.asarray(f, np.int64)
    prefix = area_prefix(face_areas(v, f))
    total = prefix[-1]
    s = np.arange(n, dtype=np.uint64)
    target = uniforms(seed, 3 * s + 1) * total
    target = np.where(target >= total, np.nextafter(total, 0.0), target)
    fid = np.searchsorted(prefix, target, side="right").astype(np.int64)
    return barycentric(v, f, fid, seed), fid


def barycentric(v, f, fid, seed=0):
    """positions of samples 0..len(fid)-1 given their faces"""
    s = np.arange(len(fid), dtype=np.uint64)
    r = np.sqrt(uniforms(seed, 3 * s + 2))
    u2 = uniforms(seed, 3 * s + 3)
    a, b, c = 1.0 - r, r * (1.0 - u2), r * u2
    p0, p1, p2 = v[f[fid, 0]], v[f[fid, 1]], v[f[fid, 2]]
    return (a[:, None] * p0 + b[:, None] * p1) + c[:, None] * p2


def bbx_crop(points, bbx):
    """utils/eval_utils.py::bbx_crop: strict inside of the box normalised to [-1, 1]"""
    bmin, bmax = np.array(bbx[0]), np.array(bbx[1])
    origin = bmin + (bmax - bmin) / 2
    pn = (points - origin) / ((bmax - bmin) / 2)
    return points[np.all(pn > -1, axis=-1) & np.all(pn < 1, axis=-1)]


def box_mask(points, bbx):
    """open3d AxisAlignedBoundingBox crop: min <= p <= max on every axis"""
    bmin, bmax = np.array(bbx[0], np.float64)[:3], np.array(bbx[1], np.float64)[:3]
    return np.all(points >= bmin, axis=-1) & np.all(points <= bmax, axis=-1)


def mesh_crop(v, f, bbx):
    """TriangleMesh.crop: the faces whose three vertices all lie in the inclusive box"""
    inside = box_mask(v, bbx)
    return f[inside[f].all(axis=1)]


def point_crop(src, sfm, voxel_size, bbx):
    """utils/eval_utils.py::point_crop with exact cell-triple membership (no int16 wrap)"""
    bmin, bmax = np.array(bbx[0]), np.array(bbx[1])
    scale = np.max(bmax - bmin) / 2
    origin = bmin + (bmax - bmin) / 2
    res = int(np.floor(2 * scale / voxel_size))

    def cells(p):
        return np.floor(res * ((p - origin) / scale + 1.0) / 2.0).astype(np.int64)

    keep = set(map(tuple, cells(sfm)))
    return src[np.array([tuple(c) in keep for c in cells(src)], dtype=bool).reshape(len(src))]


def compute(dist1, dist2, threshold):
    """utils/eval_utils.py::_compute without the printing"""
    precision = max(np.mean((dist2 < threshold).astype("float")), 1e-6)
    recal = max(np.mean((dist1 < threshold).astype("float")), 1e-6)
    fscore = 2 * precision * recal / (precision + recal)
    return {"dist1": np.mean(dist2), "dist2": np.mean(dist1), "prec": precision, "recal": recal, "fscore": fscore}


def morton16(pts):
    """stand-in for kaolin's spc_ops.points_to_morton on int16 [n,3]: 16 bits per axis interleaved (x high)"""
    import torch

    q = pts.to(torch.int64) & 0xFFFF
    out = torch.zeros(q.shape[0], dtype=torch.int64, device=q.device)
    for b in range(16):
        for a in range(3):
            out |= ((q[:, a] >> b) & 1) << (3 * b + 2 - a)
    return out


def load_eval():
    """the unmodified utils.eval_utils and utils.eval_mesh of the reference (from the reference root or oracle/_ref).
    Third-party packages that are not installed are inert stand-ins (oracle.ref_import); callers patch
    `eval_utils.trimesh` and `eval_utils.spc_ops.points_to_morton` with working ones where a test needs them."""
    import sys
    import types
    import warnings

    from oracle import ref_import

    if not ref_import.available():
        raise RuntimeError(f"reference tree not present at {ref_import.REF_ROOT}")
    ref_import._install_stubs()
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import utils.eval_utils as eval_utils  # type: ignore
        import utils.eval_mesh as eval_mesh  # type: ignore
    return types.SimpleNamespace(eval_utils=eval_utils, eval_mesh=eval_mesh)
