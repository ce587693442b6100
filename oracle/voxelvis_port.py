"""Numpy restatement of the point-cloud visibility filter (csrc/voxelvis.cu, nrw.reprojection.VoxelRenderer and
reproj_filter_points), TEST INFRASTRUCTURE.

* `gen_rays`: kaolin_renderer.gen_rays in the fp32 order written down in csrc/voxelvis.cu.
* `slab`, `raytrace`: octree_port.py's hit list with the NaN rule of fminf / fmaxf (a 0/0 slab term is ignored), which
  only matters for a direction component that the +1e-7 turns into 0.
* `first_hit` / `cast`: the first leaf of every ray (the nearest entry, the smallest hierarchy index on ties, a miss
  unless near > 1e-4, as octree_port.get_near_far), the depth near * scale / |d|.
* `lookup`: the point -> leaf map with the builder's clamped quantisation.
* `filter_points`, `pipeline`: the whole filter and the rows of `python -m nrw.reprojection --point_source`.
* `load_kaolin_renderer`: the unmodified utils/kaolin_renderer.py (and through it tools/prepare_data/generate_voxel.py)
  with functional Kaolin stand-ins built on octree_port: quantize_points, unbatched_points_to_octree, scan_octrees,
  generate_points, unbatched_raytrace and points_to_morton, and a real kornia create_meshgrid.
"""
import numpy as np

from oracle import octree_port as op

f32 = np.float32


def gen_rays(H, W, K, c2w):
    """-> (o [H*W,3], unit d [H*W,3], n [H*W]) fp32, pixels in raster order"""
    K = np.asarray(K)
    fx, fy, cx, cy = f32(K[0, 0]), f32(K[1, 1]), f32(K[0, 2]), f32(K[1, 2])
    M = np.asarray(c2w, np.float64)[:3].astype(f32)
    r, c = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    dx = ((c.reshape(-1).astype(f32) - cx) / fx).astype(f32)
    dy = ((r.reshape(-1).astype(f32) - cy) / fy).astype(f32)
    d = np.stack([((dx * M[k, 0]).astype(f32) + (dy * M[k, 1]).astype(f32)).astype(f32) + M[k, 2] for k in range(3)], 1)
    d = d.astype(f32)
    n = np.sqrt((((d[:, 0] * d[:, 0]).astype(f32) + (d[:, 1] * d[:, 1]).astype(f32)).astype(f32)
                 + (d[:, 2] * d[:, 2]).astype(f32)).astype(f32)).astype(f32)
    with np.errstate(all="ignore"):
        d = (d / n[:, None]).astype(f32)
    o = np.ascontiguousarray(np.broadcast_to(M[:, 3], d.shape), dtype=f32)
    return o, d, n


def slab(o, d, coords, l):
    """fp32 slab test of rays (o, d [R,3], normalised) against the voxels coords [V,3] of level l -> (hit [R,V], entry
    [R,V]), as octree_trace.cuh's `slab`: fminf / fmaxf ignore a NaN operand (np.fmin / np.fmax), tmin starts at -inf"""
    r = f32(1.0) / f32(2 ** l)
    c = (r * (2 * coords + 1).astype(f32) - f32(1.0)).astype(f32)
    tmin = np.full((len(o), len(coords)), -np.inf, f32)
    tmax = np.full((len(o), len(coords)), np.inf, f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for a in range(3):
            t1 = (((c[:, a] - r).astype(f32)[None] - o[:, a, None]).astype(f32) / d[:, a, None]).astype(f32)
            t2 = (((c[:, a] + r).astype(f32)[None] - o[:, a, None]).astype(f32) / d[:, a, None]).astype(f32)
            tmin = np.fmax(tmin, np.fmin(t1, t2))
            tmax = np.fmin(tmax, np.fmax(t1, t2))
    return (tmax >= tmin) & (tmax >= 0), np.fmax(tmin, f32(0.0)).astype(f32)


def raytrace(tree, level, o, d, chunk=1 << 24):
    """every leaf hit by the normalised rays (o, d) whose ancestors' slab tests pass too -> (ray, hierarchy index,
    entry), sorted by ray, then entry, then index (unbatched_raytrace with return_depth)"""
    leaves = tree["levels"][level]
    step = max(1, chunk // max(1, len(leaves)))
    base = int(tree["pyramid"][1, level])
    out = []
    for s in range(0, len(o), step):
        os_, ds_ = o[s:s + step], d[s:s + step]
        ok = np.ones((len(os_), len(leaves)), bool)
        for l in range(level):
            ok &= slab(os_, ds_, leaves >> (level - l), l)[0]
        h, dep = slab(os_, ds_, leaves, level)
        ok &= h
        ri, li = np.nonzero(ok)
        dp = dep[ri, li]
        order = np.lexsort((li, dp, ri))
        out.append((ri[order] + s, li[order] + base, dp[order]))
    if not out:
        return np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, f32)
    return (np.concatenate([x[0] for x in out]).astype(np.int32), np.concatenate([x[1] for x in out]).astype(np.int32),
            np.concatenate([x[2] for x in out]).astype(f32))


def first_hit(tree, level, rays_o, rays_d, origin, scale):
    """get_near_far's (near * scale, pid) of every ray: pid = hierarchy index of the first leaf, -1 on a miss"""
    o, d = op.normalise_rays(rays_o, rays_d, origin, scale)
    R = len(o)
    near = np.zeros(R, f32)
    pid = -np.ones(R, np.int32)
    ri, pi, dep = raytrace(tree, level, o, d)
    u, first = np.unique(ri, return_index=True)
    near[u], pid[u] = dep[first], pi[first]
    bad = ~(near > f32(1e-4))
    near[bad] = 0
    pid[bad] = -1
    return (near * f32(scale)).astype(f32), pid


def cast(tree, level, origin, scale, H, W, K, c2w):
    """one view -> (depth f32 [H, W], leaf i32 [H, W], -1 on a miss)"""
    o, d, n = gen_rays(H, W, K, c2w)
    near, pid = first_hit(tree, level, o, d, origin, scale)
    with np.errstate(all="ignore"):
        depth = (near / n).astype(f32)
    leaf = np.where(pid >= 0, pid - int(tree["pyramid"][1, level]), -1).astype(np.int32)
    return depth.reshape(H, W), leaf.reshape(H, W)


def lookup(tree, level, pn):
    """-> (leaf i32 [n]: -1 outside the open cube (-1, 1)^3 or in a cell that is not a leaf, not-a-leaf flag)"""
    pn = np.asarray(pn, np.float64).reshape(-1, 3)
    inside = np.all((pn > -1) & (pn < 1), axis=1)
    q = op.quantize_points(np.where(inside[:, None], pn, 0.0), level).astype(np.int64)
    keys = op._morton(q, level)
    leaves = op._morton(tree["levels"][level].astype(np.int64), level)       # Morton-sorted
    j = np.clip(np.searchsorted(leaves, keys), 0, max(len(leaves) - 1, 0))
    found = inside & (len(leaves) > 0) & (leaves[j] == keys if len(leaves) else False)
    return np.where(found, j, -1).astype(np.int32), bool((inside & ~found).any())


def views(Ks, Es, whs):
    for K, E, (w, h) in zip(Ks, Es, whs):
        yield K, np.linalg.inv(np.asarray(E, np.float64)), int(h), int(w)


def filter_points(points, scene_config, Ks, Es, whs, voxel_size=0.01):
    """-> (mask bool [n], hit pixel count, per-view (depth, leaf) list) of reproj_filter_points"""
    points = np.asarray(points, np.float64)
    tree, origin, scale, level, _ = op.gen_octree(scene_config, points, voxel_size, expand=0, in_sfm=False)
    visible = np.zeros(len(tree["levels"][level]), bool)
    n_hit, maps = 0, []
    for K, c2w, h, w in views(Ks, Es, whs):
        depth, leaf = cast(tree, level, origin, scale, h, w, K, c2w)
        visible[leaf[leaf >= 0]] = True
        n_hit += int((leaf >= 0).sum())
        maps.append((depth, leaf))
    lf, _ = lookup(tree, level, (points - origin) / scale)
    mask = (lf >= 0) & visible[np.maximum(lf, 0)]
    return mask, n_hit, maps


def pipeline(src, target, colors, scene_config, Ks, Es, whs, voxel_size=0.01):
    """the rows of reprojected.ply: np.unique([target xyz, rgb], axis=0) of the kept source indices"""
    mask, _, _ = filter_points(src, scene_config, Ks, Es, whs, voxel_size)
    return np.unique(np.hstack([target[mask], colors[mask]]), axis=0)


# ---- functional Kaolin stand-ins ------------------------------------------------------------------------------------
def _tree_from_octree(octree):
    """decode Kaolin's octree bytes into octree_port's tree dict (levels in Morton order)"""
    octree = np.asarray(octree, np.uint8)
    levels, i = [np.zeros((1, 3), np.int64)], 0
    while i < len(octree):
        parents = levels[-1]
        b = octree[i:i + len(parents)].astype(np.int64)
        i += len(parents)
        pi, jj = np.nonzero((b[:, None] >> np.arange(8)[None, :]) & 1)      # parent-major, digit-minor: Morton order
        bits = np.stack([(jj >> 2) & 1, (jj >> 1) & 1, jj & 1], 1)
        levels.append(2 * parents[pi] + bits)
    level = len(levels) - 1
    centres = (levels[level] + 0.5) * (2.0 / 2 ** level) - 1.0               # quantises back to the same cells
    tree = op.build_octree(centres, level)
    assert np.array_equal(tree["octree"], octree)
    return tree, level


class _Spc:
    """kaolin.ops.spc / kaolin.render.spc as the reference calls them"""

    def __init__(self):
        import types
        self.points = types.SimpleNamespace(quantize_points=self.quantize_points)

    @staticmethod
    def quantize_points(x, level):
        import torch
        res = 2 ** level
        return torch.floor(torch.clamp(res * (x + 1.0) / 2.0, 0, res - 1.0)).short()

    @staticmethod
    def unbatched_points_to_octree(qpts, level, sorted=False):
        import torch
        q = qpts.cpu().numpy().astype(np.int64)
        tree = op.build_octree((q + 0.5) * (2.0 / 2 ** level) - 1.0, level)
        return torch.from_numpy(tree["octree"]).to(qpts.device)

    @staticmethod
    def scan_octrees(octree, lengths):
        import torch
        tree, level = _tree_from_octree(octree.cpu().numpy())
        return level, torch.from_numpy(tree["pyramid"])[None].to(octree.device), torch.from_numpy(tree["prefix"]).to(octree.device)

    @staticmethod
    def generate_points(octree, pyramids, exsum):
        import torch
        tree, _ = _tree_from_octree(octree.cpu().numpy())
        return torch.from_numpy(tree["points"]).to(octree.device)

    @staticmethod
    def points_to_morton(points):
        import torch
        return torch.from_numpy(op._morton(points.cpu().numpy().astype(np.int64), 16)).to(points.device)

    @staticmethod
    def unbatched_raytrace(octree, points, pyramid, exsum, origin, direction, level, return_depth=True, with_exit=False):
        """hits of the already-normalised rays, grouped by ray, front to back (ties: hierarchy index)"""
        import torch
        assert return_depth and not with_exit
        tree, _ = _tree_from_octree(octree.cpu().numpy())
        ri, pi, dp = raytrace(tree, level, origin.cpu().numpy().astype(f32), direction.cpu().numpy().astype(f32))
        dev = origin.device
        return (torch.from_numpy(ri).to(dev), torch.from_numpy(pi).to(dev),
                torch.from_numpy(dp).reshape(-1, 1).to(dev))


def load_kaolin_renderer():
    """the unmodified utils/kaolin_renderer.py of the reference (module), its Kaolin and kornia names bound to the
    stand-ins above; third-party packages that are not installed are inert stand-ins (oracle.ref_import)"""
    import sys
    import warnings

    from oracle import cache_port, ref_import

    if not ref_import.available():
        raise RuntimeError(f"reference tree not present at {ref_import.REF_ROOT}")
    ref_import._install_stubs()
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import tools.prepare_data.generate_voxel as gv  # type: ignore
        import utils.kaolin_renderer as kr  # type: ignore
    spc = _Spc()
    gv.spc, gv.spc_render = spc, spc
    gv.logger = _Quiet()
    kr.spc_ops = spc
    kr.create_meshgrid = cache_port.create_meshgrid
    kr.tqdm = lambda x, *a, **k: x
    return kr


class _Quiet:
    def __getattr__(self, name):
        return lambda *a, **k: None
