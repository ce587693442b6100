"""numpy restatement of the ROI rule of the scene split (csrc/viewsel.cu, rules in its header) in the same fp32 operation
order, and loaders for the unmodified tools/prepare_data/dataset_filter_utils.py / prepare_data_split.py of the reference.
The ray is cache_port.rays' rule, computed here a band of rows at a time so views above 2^24 pixels fit in memory."""
import os

import numpy as np

from oracle import cache_port

f32 = np.float32

# Largest |ROI share (this rule) - ROI share (the reference's matmul + torch.norm rays)| the tests accept per view (on the
# synthetic scenes no pixel differs); the end-to-end test keeps every share at least this far from the threshold.
ROI_TOLERANCE = 2e-3


def rays_rows(r0, r1, W, K, c2w):
    """cache_port.rays for rows r0 .. r1-1 of a W-wide view: (o [n, 3], unit d [n, 3]) in fp32, raster order"""
    c2w = np.asarray(c2w, f32)
    j, i = np.meshgrid(np.arange(r0, r1, dtype=f32), np.arange(W, dtype=f32), indexing="ij")
    i, j = i.reshape(-1), j.reshape(-1)
    dx = (i - f32(K[0, 2])) / f32(K[0, 0])
    ndy = -((j - f32(K[1, 2])) / f32(K[1, 1]))
    d = np.stack([(dx * c2w[k, 0] + ndy * c2w[k, 1]) + (-c2w[k, 2]) for k in range(3)], 1).astype(f32)
    nrm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(f32)
    o = np.broadcast_to(c2w[:, 3], d.shape).astype(f32)
    return o, (d / nrm[:, None]).astype(f32)


def inside(o, d, origin, radius):
    """the per-pixel ROI test in the kernel's fp32 order"""
    s = np.asarray(origin, f32)
    R = f32(radius)
    c = (s[None, :] - o).astype(f32)
    dot = ((c[:, 0] * d[:, 0] + c[:, 1] * d[:, 1]) + c[:, 2] * d[:, 2]).astype(f32)
    e = (c - dot[:, None] * d).astype(f32)
    dist_ray = np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]).astype(f32)
    dist_cam = np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]).astype(f32)
    return ((R > dist_cam) | (dot > 0)) & (dist_ray < R)


def roi_count(H, W, K, c2w, origin, radius, band_pixels=1 << 22):
    rows = max(1, band_pixels // W)
    n = 0
    for r0 in range(0, H, rows):
        o, d = rays_rows(r0, min(H, r0 + rows), W, K, c2w)
        n += int(inside(o, d, origin, radius).sum())
    return n


def roi_counts(views, hw, origin, radius):
    """roi_count of every row of the kernel's view table (f32 [n, 16] = fx, fy, cx, cy, c2w[12]; hw [n, 2])"""
    out = []
    for v, (H, W) in zip(np.asarray(views, f32), np.asarray(hw)):
        K = np.array([[v[0], 0, v[2]], [0, v[1], v[3]], [0, 0, 1]], f32)
        out.append(roi_count(int(H), int(W), K, v[4:].reshape(3, 4), origin, radius))
    return np.array(out, np.int64)


def static_count(sem, ids):
    """pixels of a semantic map whose label is none of ids (the reference's static_mask, counted)"""
    sem = np.asarray(sem)
    return int((~np.isin(sem, np.asarray(ids, sem.dtype))).sum())


# ---- the unmodified reference ----------------------------------------------------------------------------------------
def load_split_ref():
    """The unmodified tools/prepare_data/dataset_filter_utils.py, imported through oracle.ref_import's stand-ins with
    cache_port's real create_meshgrid, and registered as the module ``dataset_filter_utils`` so that the unmodified
    prepare_data_split.py (``script``) imports it.  view_selection calls .cuda(): bind torch.Tensor.cuda to the identity
    to run it on the CPU.  Returns a namespace with the module, view_selection, filter_image_based_on_transient_percent,
    get_label_id_mapping, get_ray_directions, get_rays and the script's path."""
    import importlib.util
    import sys
    import types
    import warnings

    from oracle import ref_import

    if not ref_import.available():
        raise RuntimeError(f"reference tree not present at {ref_import.REF_ROOT}")
    ref_import._install_yacs()
    ref_import._install_stubs()
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import datasets.ray_utils as ray_utils  # type: ignore

        ray_utils.create_meshgrid = cache_port.create_meshgrid
        base = os.path.join(ref_import.REF_ROOT, "tools", "prepare_data")
        mod = sys.modules.get("dataset_filter_utils")
        if mod is None:
            spec = importlib.util.spec_from_file_location("dataset_filter_utils", os.path.join(base, "dataset_filter_utils.py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules["dataset_filter_utils"] = mod
            spec.loader.exec_module(mod)
    return types.SimpleNamespace(module=mod, view_selection=mod.view_selection,
                                 filter_image_based_on_transient_percent=mod.filter_image_based_on_transient_percent,
                                 get_label_id_mapping=mod.get_label_id_mapping, get_ray_directions=ray_utils.get_ray_directions,
                                 get_rays=ray_utils.get_rays, script=os.path.join(base, "prepare_data_split.py"))


def ref_roi_count(R, H, W, K, c2w, origin, radius, device="cpu"):
    """the ROI count of view_selection's own torch expressions (dataset_filter_utils.py, the loop body of the ROI pass)
    on the reference's get_ray_directions / get_rays"""
    import torch

    scene_origin = torch.tensor(origin).to(device)
    rays_o, rays_d = R.get_rays(R.get_ray_directions(H, W, K).to(device), torch.FloatTensor(np.asarray(c2w)).to(device))
    camera2origin = scene_origin - rays_o
    dot_product = torch.sum((scene_origin - rays_o) * rays_d, -1, keepdim=True)
    camera2origin_project = dot_product * rays_d
    dist_ray_origin = torch.linalg.norm((camera2origin - camera2origin_project), ord=2, dim=-1)
    dist_camera2origin = torch.linalg.norm(camera2origin, ord=2, dim=-1)
    if_ROI = torch.logical_and(torch.logical_or((radius > dist_camera2origin), dot_product.squeeze(-1) > 0),
                               (dist_ray_origin < radius))
    return int(torch.count_nonzero(if_ROI))
