"""numpy restatement of the training ray-cache pass (csrc/raygen.cu, rules in its header) in the same operation order:
rays, rgb, label, keypoint depth / weight, the near/far percentiles, the depth_percent padding count and the split
writer's padding.  Voxel near/far come from the octree tracer, which has its own port (octree_port.py).  load_cache_ref()
imports the unmodified reference functions the restatement is checked against."""
import numpy as np

f32 = np.float32


def rays(H, W, K, c2w):
    """get_ray_directions + get_rays: (rays_o [HW,3], rays_d [HW,3], |d| [HW]) in fp32, raster order"""
    c2w = np.asarray(c2w, f32)
    j, i = np.meshgrid(np.arange(H, dtype=f32), np.arange(W, dtype=f32), indexing="ij")
    i, j = i.reshape(-1), j.reshape(-1)
    dx = (i - f32(K[0, 2])) / f32(K[0, 0])
    ndy = -((j - f32(K[1, 2])) / f32(K[1, 1]))
    d = np.stack([(dx * c2w[k, 0] + ndy * c2w[k, 1]) + (-c2w[k, 2]) for k in range(3)], 1).astype(f32)
    nrm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(f32)
    o = np.broadcast_to(c2w[:, 3], d.shape).astype(f32)
    return o, (d / nrm[:, None]).astype(f32), nrm


def nearest_index(dst, src):
    """cv2 INTER_NEAREST source index of every destination index (OpenCV resizeNN, fp64)"""
    ifx = 1.0 / (float(dst) / float(src))
    return np.minimum(np.floor(np.arange(dst, dtype=np.float64) * ifx).astype(np.int64), src - 1)


def label(sem, H, W):
    sy, sx = nearest_index(H, sem.shape[0]), nearest_index(W, sem.shape[1])
    return np.asarray(sem, f32)[sy[:, None], sx[None, :]].reshape(-1)


def keypoint_winners(xys, ids, n_table, ds, H, W):
    """(pixel of every in-frame keypoint or -1, in-frame mask); the last keypoint of a pixel wins"""
    ids = np.asarray(ids, np.int64)
    u, v = np.rint(xys[:, 0] / float(ds)), np.rint(xys[:, 1] / float(ds))
    ok = (ids >= 0) & (ids < n_table) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    pix = np.where(ok, np.where(ok, v, 0).astype(np.int64) * W + np.where(ok, u, 0).astype(np.int64), -1)
    return pix, ok


def mean_error(err_kp, index):
    """the kernel's order: keypoint k (its index in the image's point list) is added to lane k % 32 in list order, in
    fp64, then the 32 lanes are combined by the xor butterfly 16, 8, 4, 2, 1"""
    lanes = np.zeros(32)
    for e, k in zip(err_kp, index):
        lanes[k % 32] += e
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return lanes[0] / float(len(err_kp))


def depth_weight(H, W, nrm, xys, ids, table_xyz, table_err, ds, w2c_z):
    """keypoint depth [HW] and weight [HW] (get_colmap_depth in the stated orders)"""
    depth, weight = np.zeros(H * W, f32), np.zeros(H * W, f32)
    pix, ok = keypoint_winners(xys, ids, len(table_err), ds, H, W)
    if not ok.any():
        return depth, weight, {}
    k_ok = np.nonzero(ok)[0]
    mean = mean_error(table_err[ids[k_ok]], k_ok)
    win = {}
    for k in k_ok:                      # sequential: the last keypoint of a pixel wins
        win[int(pix[k])] = int(k)
    for p, k in win.items():
        X = table_xyz[ids[k]]
        z = ((w2c_z[0] * X[0] + w2c_z[1] * X[1]) + w2c_z[2] * X[2]) + w2c_z[3]
        q = table_err[ids[k]] / mean
        depth[p] = f32(z) * nrm[p]
        weight[p] = f32(2.0 * np.exp(-(q * q)))
    return depth, weight, win


def image_rows(H, W, K, c2w, image_id, rgb8, near, far, xys=None, ids=None, table_xyz=None, table_err=None, ds=1,
               w2c_z=None, sem=None):
    """cache rows [HW, 12 or 11] and rgbs [HW, 3] without voxels (constant near/far, every pixel kept)"""
    o, d, nrm = rays(H, W, K, c2w)
    n = H * W
    if xys is not None and len(xys):
        depth, weight, _ = depth_weight(H, W, nrm, xys, ids, table_xyz, table_err, ds, w2c_z)
    else:
        depth, weight = np.zeros(n, f32), np.zeros(n, f32)
    cols = [o, d, np.full((n, 1), f32(near)), np.full((n, 1), f32(far)), np.full((n, 1), f32(image_id))]
    if sem is not None:
        cols.append(label(sem, H, W)[:, None])
    cols += [depth[:, None], weight[:, None]]
    rgb = (np.asarray(rgb8, f32).reshape(-1, 3) / f32(255)).astype(f32)
    return np.concatenate(cols, 1).astype(f32), rgb


def padding_count(n, v, p):
    """read_meta :664 in fp64; a negative count or no depth row gives none"""
    if not p > 0 or v == 0:
        return 0
    x = np.ceil((p * n - v) / (1 - p))
    return int(x) if x > 0 else 0


def percentile_linear(sorted_vals, q):
    """np.percentile(..., method='linear') of an ascending array, in numpy's operation order"""
    m = len(sorted_vals)
    qq = q / 100.0
    v = (m - 1) * qq
    if v >= m - 1:
        lo = hi = m - 1
        g = v + 1.0
    elif v < 0:
        lo = hi = 0
        g = v
    else:
        lo = int(np.floor(v))
        hi = lo + 1
        g = v - lo
    a, b = sorted_vals[lo], sorted_vals[hi]
    diff = b - a
    return b - diff * (1.0 - g) if g >= 0.5 else a + diff * g


def camera_z(xyz, w2c):
    """camera z of every point in the stated fp64 order"""
    return ((w2c[2, 0] * xyz[:, 0] + w2c[2, 1] * xyz[:, 1]) + w2c[2, 2] * xyz[:, 2]) + w2c[2, 3]


def depth_bounds(xyz, w2c_all, q=(0.1, 99.9)):
    out = []
    for w in w2c_all:
        z = camera_z(xyz, w)
        z = np.sort(z[z > 0])
        out.append((percentile_linear(z, q[0]), percentile_linear(z, q[1])))
    return np.array(out)


def split_chunks(rows, n_chunks, padding_index):
    """split_to_chunks on one array: the list of chunk arrays"""
    full = np.concatenate([rows, rows[np.asarray(padding_index, np.int64)]], 0)
    L = full.shape[0] // n_chunks
    return [full[i * L:(i + 1) * L] for i in range(n_chunks)]


# ---- the unmodified reference functions ----------------------------------------------------------------------------------
def create_meshgrid(height, width, normalized_coordinates=True, device=None, dtype=None):
    """kornia.create_meshgrid: [1, H, W, 2] of (x, y) = (column, row), optionally mapped to [-1, 1]"""
    import torch

    dtype = dtype or torch.float32
    xs = torch.linspace(0, width - 1, width, device=device, dtype=dtype)
    ys = torch.linspace(0, height - 1, height, device=device, dtype=dtype)
    if normalized_coordinates:
        xs = (xs / (width - 1) - 0.5) * 2
        ys = (ys / (height - 1) - 0.5) * 2
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([gx, gy], -1).unsqueeze(0)


def load_cache_ref():
    """The unmodified datasets/ray_utils.py, datasets/phototourism.py, datasets/colmap_utils.py and
    tools/prepare_data/prepare_data_cache.py of the reference, through oracle.ref_import's stand-ins for the packages that
    are not installed (pandas is stood in as well: only read_meta uses it).  kornia's create_meshgrid is replaced by a
    real one.  Returns a namespace with get_ray_directions, get_rays, get_colmap_depth (call it unbound, self=None),
    read_images_binary and split_to_chunks."""
    import importlib.util
    import sys
    import types
    import warnings
    from unittest import mock

    from oracle import ref_import

    if not ref_import.available():
        raise RuntimeError(f"reference tree not present at {ref_import.REF_ROOT}")
    ref_import._install_yacs()
    ref_import._install_stubs()
    try:
        import pandas  # noqa: F401
    except Exception:
        sys.modules.setdefault("pandas", mock.MagicMock(name="pandas"))
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import datasets.colmap_utils as colmap_utils  # type: ignore
        import datasets.phototourism as phototourism  # type: ignore
        import datasets.ray_utils as ray_utils  # type: ignore

        ray_utils.create_meshgrid = create_meshgrid
        phototourism.create_meshgrid = create_meshgrid
        path = f"{ref_import.REF_ROOT}/tools/prepare_data/prepare_data_cache.py"
        spec = importlib.util.spec_from_file_location("ref_prepare_data_cache", path)
        pdc = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(pdc)
    return types.SimpleNamespace(get_ray_directions=ray_utils.get_ray_directions, get_rays=ray_utils.get_rays,
                                 get_colmap_depth=phototourism.PhototourismDataset.get_colmap_depth,
                                 read_images_binary=colmap_utils.read_images_binary, split_to_chunks=pdc.split_to_chunks)


def ref_colmap_depth(R, table_xyz, table_err, xys, ids, pose_c2w, K, img_w, img_h, ds, device="cpu"):
    """read_meta :564-580 around the reference's get_colmap_depth: (depth [H*W], weight [H*W]) as numpy fp32"""
    import torch

    pts3d_array = torch.ones(len(table_err), 4)
    pts3d_array[:, :3] = torch.from_numpy(table_xyz)
    error_array = torch.from_numpy(table_err).float().reshape(-1, 1)
    pose = torch.FloatTensor(pose_c2w).to(device)
    pose[..., 1:3] *= -1
    valid = ids != -1
    pid = torch.from_numpy(ids[valid])
    img_2d = torch.from_numpy(xys)[torch.from_numpy(valid)] / ds
    d, w = R.get_colmap_depth(None, pts3d_array[pid].to(device), img_2d.to(device), error_array[pid].to(device), pose,
                              torch.FloatTensor(K).to(device), img_w, img_h, device=device)
    return d.reshape(-1).numpy(), w.reshape(-1).numpy()
