"""Reconstruction evaluation on the GPU: a drop-in for utils/eval_utils.py and utils/eval_mesh.py (same names and
signatures) that needs neither open3d, Kaolin nor trimesh.

* Nearest neighbours: exact fp64 search on the device (csrc/nnsearch.cu): for every query the nearest point, the
  smallest index among equally near ones, with numpy's distance arithmetic.
* Surface sampling (`--mesh`): area-weighted uniform samples, reproducible from (seed, sample index).
* SfM crop: exact match of the integer voxel cells of the SfM points.  The reference casts cells to int16 (`.short()`),
  so cells more than 32767 cells from the box's corner wrap around there; here they do not.

`eval_mesh` follows the open3d branch of the reference (`o3d_load`), the configuration the authors ran:
  - point-cloud predictions are taken as they are (utils/reproj_filter.py already writes ground-truth-frame points;
    the reference's trimesh fallback applies `sfm2gt` a second time) and cropped with the inclusive box
    min <= p <= max, as AxisAlignedBoundingBox does;
  - mesh predictions get `sfm2gt` on their vertices, keep the faces whose three vertices lie in the inclusive box
    (TriangleMesh.crop) and are sampled to 10 x the number of cropped ground-truth points.
Distances stay on the device; precision and recall come from one device sort per direction and a strict `<` search,
so count / N equals numpy's mean(d < t) exactly.  Inputs that are non-finite, empty after cropping or have malformed
faces raise NrwError (the reference returns NaN metrics for empty sets).  The error-coloured visualize/*/error_*.ply files
are not written (they need matplotlib's jet colormap).

    python -m nrw.evaluation --file_pred P.ply --file_trgt GT.ply --scene_config_path config.yaml --threshold 0.01,0.2,0.01
"""
import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib
from ._lib import NrwError, check, ptr, stream_ptr
from .colmap import read_points3d
from .mesh import read_ply, write_ply


def _device(device):
    return torch.device(f"cuda:{device}" if isinstance(device, int) else device)


def _scratch(nbytes, dev):
    """256-byte aligned device scratch: (owner tensor, pointer)"""
    if nbytes < 0:
        check(int(nbytes), "scratch size")
    t = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=dev)
    return t, C.c_void_p((t.data_ptr() + 255) // 256 * 256)


def _points(x, what, dev=None):
    """[n,3] float64 contiguous CUDA tensor of finite points"""
    t = torch.as_tensor(x)
    dev = dev if dev is not None else (t.device if t.is_cuda else torch.device("cuda", torch.cuda.current_device()))
    t = t.to(device=dev, dtype=torch.float64).contiguous()
    if t.dim() != 2 or t.shape[1] != 3:
        raise NrwError(f"{what}: expected points of shape [n, 3], got {tuple(t.shape)}")
    if t.shape[0] and not bool(torch.isfinite(t).all()):
        raise NrwError(f"{what}: points are not all finite")
    return t


class NearestNeighbours:
    """Exact fp64 nearest-neighbour index of a point set [n,3] (1 <= n <= 2^31 - 1) on its CUDA device."""

    def __init__(self, ref):
        self.ref = _points(ref, "NearestNeighbours")
        n = self.ref.shape[0]
        if n == 0 or n > 0x7FFFFFFF:
            raise NrwError(f"NearestNeighbours: {n} reference points (need 1 .. 2^31 - 1)")
        L = _lib.lib()
        self.n = n
        self._index, self._ip = _scratch(L.nrw_nn_index_bytes(n), self.ref.device)
        with torch.cuda.device(self.ref.device):
            check(L.nrw_nn_build(ptr(self.ref), n, self._ip, stream_ptr()), "nrw_nn_build")

    def query(self, queries):
        """-> (dist float64 [m], idx int64 [m]) CUDA tensors: the nearest indexed point of every query"""
        q = _points(queries, "NearestNeighbours.query", self.ref.device)
        m = q.shape[0]
        dist = torch.empty(m, dtype=torch.float64, device=q.device)
        idx = torch.empty(m, dtype=torch.int64, device=q.device)
        if m == 0:
            return dist, idx
        L = _lib.lib()
        _, sp = _scratch(L.nrw_nn_query_scratch_bytes(m), q.device)
        with torch.cuda.device(q.device):
            check(L.nrw_nn_query(self._ip, self.n, ptr(q), m, ptr(dist), ptr(idx), sp, stream_ptr()), "nrw_nn_query")
        return dist, idx


def nn_correspondance_torch(verts1, verts2):
    """For every point of verts2 its nearest point of verts1: (indices int64 [m], distances float64 [m]) CUDA tensors."""
    dist, idx = NearestNeighbours(verts1).query(verts2)
    return idx, dist


def nn_correspondance(verts1, verts2, use_o3d=True):
    """utils/eval_utils.py::nn_correspondance: for each vertex in verts2 the nearest vertex in verts1 ->
    (indices, distances) numpy arrays; ([], []) when either set is empty.  `use_o3d` is accepted and ignored."""
    if len(verts1) == 0 or len(verts2) == 0:
        return [], []
    idx, dist = nn_correspondance_torch(verts1, verts2)
    return idx.cpu().numpy(), dist.cpu().numpy()


def sample_points_uniformly(verts, faces, n, seed=0, return_face_ids=False):
    """Area-weighted uniform samples of a triangle mesh (open3d's sample_points_uniformly, reproducible): float64 [n,3]
    CUDA tensor (and the int64 face id of every sample with return_face_ids).  Sample s depends only on (seed, s)."""
    v = _points(verts, "sample_points_uniformly")
    f = torch.as_tensor(faces)
    if f.dim() != 2 or f.shape[1] != 3 or f.shape[0] == 0 or f.dtype.is_floating_point or f.dtype == torch.bool:
        raise NrwError(f"sample_points_uniformly: faces must be a non-empty integer array [F, 3], got {tuple(f.shape)} {f.dtype}")
    f = f.to(device=v.device, dtype=torch.int64).contiguous()
    n = int(n)
    if n < 0:
        raise NrwError(f"sample_points_uniformly: n = {n}")
    L = _lib.lib()
    out = torch.empty(n, 3, dtype=torch.float64, device=v.device)
    fid = torch.empty(n, dtype=torch.int64, device=v.device) if return_face_ids else None
    status = torch.empty(1, dtype=torch.int32, device=v.device)
    _, sp = _scratch(L.nrw_mesh_sample_scratch_bytes(f.shape[0]), v.device)
    with torch.cuda.device(v.device):
        check(L.nrw_mesh_sample(ptr(v), v.shape[0], ptr(f), f.shape[0], n, int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(out), ptr(fid),
                                ptr(status), sp, stream_ptr()), "nrw_mesh_sample")
    st = int(status.item())
    if st & 1:
        raise NrwError(f"sample_points_uniformly: a face index lies outside [0, {v.shape[0]})")
    if st & 2:
        raise NrwError("sample_points_uniformly: the total face area is not positive and finite")
    return (out, fid) if return_face_ids else out


def _compute_from(n1, n2, c1, c2, s1, s2):
    """_compute's formulas from counts c = #(d < t), sizes n and distance sums s"""
    precision = max(c2 / n2, 1e-6)
    recal = max(c1 / n1, 1e-6)
    fscore = 2 * precision * recal / (precision + recal)
    return {"dist1": s2 / n2, "dist2": s1 / n1, "prec": precision, "recal": recal, "fscore": fscore}


def _compute(dist1, dist2, threshold):
    """utils/eval_utils.py::_compute (same formulas, including the 1e-6 floors and 'dist1': mean(dist2))"""
    precision = max(np.mean((dist2 < threshold).astype("float")), 1e-6)
    recal = max(np.mean((dist1 < threshold).astype("float")), 1e-6)
    fscore = 2 * precision * recal / (precision + recal)
    metrics = {"dist1": np.mean(dist2), "dist2": np.mean(dist1), "prec": precision, "recal": recal, "fscore": fscore}
    print(f"****metrics for threshold {threshold:.2f}****")
    print(metrics)
    print("******************************************")
    return metrics


def bbx_crop(points, bbx):
    """utils/eval_utils.py::bbx_crop: the points strictly inside the box normalised to [-1, 1] (numpy or tensor in,
    same kind out)."""
    is_t = torch.is_tensor(points)
    p = torch.as_tensor(points, dtype=torch.float64)
    bmin = torch.as_tensor(np.array(bbx[0]), dtype=torch.float64, device=p.device)
    bmax = torch.as_tensor(np.array(bbx[1]), dtype=torch.float64, device=p.device)
    pn = (p - (bmin + (bmax - bmin) / 2)) / ((bmax - bmin) / 2)
    mask = ((pn > -1).all(-1) & (pn < 1).all(-1))
    return points[mask] if is_t else points[mask.cpu().numpy()]


def _box_mask(p, bbx):
    """inclusive axis-aligned box min <= p <= max (open3d's AxisAlignedBoundingBox crop)"""
    bmin = torch.as_tensor(np.array(bbx[0], np.float64)[:3], device=p.device)
    bmax = torch.as_tensor(np.array(bbx[1], np.float64)[:3], device=p.device)
    return (p >= bmin).all(-1) & (p <= bmax).all(-1)


def filtered_sfm(data_dir, sfm_to_gt, track_length=200, reproj_error=0.5, save_path=None):
    """utils/eval_utils.py::filtered_sfm: SfM points of data_dir/points3D.bin with track length > track_length and
    error < reproj_error, mapped by sfm_to_gt[:3] @ [xyz, 1] in float64 -> numpy [n,3]."""
    pts = read_points3d(os.path.join(data_dir, "points3D.bin"))
    keep = (pts["track_length"] > track_length) & (pts["error"] < reproj_error)
    xyz = pts["xyz"][keep]
    if len(xyz) == 0:
        raise NrwError(f"filtered_sfm: no SfM point has track length > {track_length} and error < {reproj_error}")
    xyz = np.concatenate((xyz, np.ones((xyz.shape[0], 1))), axis=-1)
    out = (np.array(sfm_to_gt)[:3] @ xyz.T).T
    if save_path is not None:
        write_ply(save_path, out)
    return out


def point_crop(src_pts, tsr_pts, voxel_size, bbx, batch_size=8, save_path=None, device=0):
    """utils/eval_utils.py::point_crop: the source points whose voxel cell holds an SfM point, in source order.  Cells
    are floor(res * ((p - origin) / scale + 1) / 2) in float64 with scale = max extent / 2 and
    res = floor(2 scale / voxel_size), matched exactly as integer triples (no int16 wrap).  Numpy in -> numpy out,
    tensor in -> tensor out; `batch_size` is accepted and ignored."""
    is_t = torch.is_tensor(src_pts)
    dev = src_pts.device if is_t and src_pts.is_cuda else _device(device)
    src = _points(src_pts, "point_crop", dev)
    sfm = _points(tsr_pts, "point_crop", dev)
    bmin, bmax = np.array(bbx[0]), np.array(bbx[1])
    scale = np.max(bmax - bmin) / 2
    origin = torch.as_tensor(bmin + (bmax - bmin) / 2, dtype=torch.float64, device=dev)
    res = int(np.floor(2 * scale / voxel_size))

    def cells(p):
        c = torch.floor(res * ((p - origin) / float(scale) + 1.0) / 2.0)
        if c.numel() and float(c.abs().max()) >= 2.0 ** 62:
            raise NrwError("point_crop: voxel cells exceed the int64 range")
        return c.to(torch.int64)

    cs, ct = cells(src), cells(sfm)
    _, inv = torch.unique(torch.cat([ct, cs]), dim=0, return_inverse=True)
    hit = torch.zeros(int(inv.max()) + 1 if inv.numel() else 0, dtype=torch.bool, device=dev)
    hit[inv[:ct.shape[0]]] = True
    mask = hit[inv[ct.shape[0]:]]
    out = src[mask]
    if save_path is not None:
        write_ply(save_path, out.cpu().numpy())
    if is_t:
        return out
    return np.asarray(src_pts)[mask.cpu().numpy()]


def _load(file_pred, file_trgt, scene_config, is_mesh, bbx_name, dev, seed):
    """o3d_load of the reference: -> (pred, trgt) float64 CUDA tensors in the ground-truth frame, cropped"""
    bbx = scene_config[bbx_name]
    trgt = _points(read_ply(file_trgt)["vertices"], f"eval_mesh: {file_trgt}", dev)
    trgt = trgt[_box_mask(trgt, bbx)]
    m = read_ply(file_pred)
    if is_mesh:
        sfm_to_gt = np.array(scene_config["sfm2gt"])
        v = np.asarray(m["vertices"], np.float64)
        v = np.concatenate((v, np.ones((v.shape[0], 1))), axis=-1)
        v = _points((sfm_to_gt[:3] @ v.T).T, f"eval_mesh: {file_pred}", dev)
        f = torch.as_tensor(m["faces"], device=dev)
        if f.shape[0] == 0:
            raise NrwError(f"eval_mesh: {file_pred} has no faces (drop --mesh for point clouds)")
        if bool(((f < 0) | (f >= v.shape[0])).any()):
            raise NrwError(f"eval_mesh: {file_pred} has face indices outside [0, {v.shape[0]})")
        f = f[_box_mask(v, bbx)[f].all(1)]
        if f.shape[0] == 0:
            raise NrwError(f"eval_mesh: no face of {file_pred} lies inside {bbx_name}")
        pred = sample_points_uniformly(v, f, int(trgt.shape[0]) * 10, seed=seed)
    else:
        pred = _points(m["vertices"], f"eval_mesh: {file_pred}", dev)
        pred = pred[_box_mask(pred, bbx)]
    return pred, trgt


def _nonempty(t, what):
    if t.shape[0] == 0:
        raise NrwError(f"eval_mesh: no {what} point is left after cropping")
    return t


def eval_mesh(file_pred, file_trgt, scene_config, is_mesh, threshold=.1, bbx_name='eval_bbx', use_o3d=True, save_name="eval",
              device=0, seed=0):
    """utils/eval_mesh.py::eval_mesh: precision, recall and F-score of a predicted point cloud or mesh against a
    ground-truth point cloud for one threshold or a list of them.  Writes <dir of file_pred>/eval_<save_name>/metrics.json
    (thresholds, fscores, precs, recals), visualize/<t:.2f>/metrics.json per threshold and the point clouds down_gt.ply,
    down_pred_in_gt.ply (and, with scene_config['sfm_path'], sfm_points.ply, pred_filtered.ply, target_filtered.ply).
    Returns the last threshold's metrics.  `use_o3d` is accepted and ignored."""
    dev = _device(device)
    save_dir = '/'.join(file_pred.split('/')[:-1])
    save_dir = os.path.join(save_dir, "eval_" + save_name)
    os.makedirs(save_dir, exist_ok=True)
    print(f"results will save in {save_dir}")
    pred, trgt = _load(file_pred, file_trgt, scene_config, is_mesh, bbx_name, dev, seed)
    _nonempty(trgt, "ground-truth")
    _nonempty(pred, "predicted")
    write_ply(f"{save_dir}/down_gt.ply", trgt.cpu().numpy())
    write_ply(f"{save_dir}/down_pred_in_gt.ply", pred.cpu().numpy())
    if "sfm_path" in scene_config.keys():
        sfm = filtered_sfm(scene_config["sfm_path"], sfm_to_gt=np.array(scene_config['sfm2gt']), track_length=scene_config['eval_tl'],
                           reproj_error=scene_config['eval_error'], save_path=f"{save_dir}/sfm_points.ply")
        print(f"filtered points: {sfm.shape[0]}")
        pred = point_crop(pred, sfm, scene_config['eval_voxel'], scene_config[bbx_name], save_path=f"{save_dir}/pred_filtered.ply")
        trgt = point_crop(trgt, sfm, scene_config['eval_voxel'], scene_config[bbx_name], save_path=f"{save_dir}/target_filtered.ply")
        _nonempty(trgt, "ground-truth")
        _nonempty(pred, "predicted")

    dist1, _ = NearestNeighbours(pred).query(trgt)       # recall side: ground truth -> prediction
    dist2, _ = NearestNeighbours(trgt).query(pred)       # precision side: prediction -> ground truth
    if not isinstance(threshold, list):
        threshold = [threshold]
    thr = torch.tensor([float(t) for t in threshold], dtype=torch.float64, device=dev)
    s1, s2 = torch.sort(dist1).values, torch.sort(dist2).values
    c1 = torch.searchsorted(s1, thr, side="left")          # #(d < t)
    c2 = torch.searchsorted(s2, thr, side="left")
    host = torch.stack([c1.double(), c2.double(), dist1.sum().expand_as(thr), dist2.sum().expand_as(thr)]).cpu().numpy()
    n1, n2 = int(dist1.shape[0]), int(dist2.shape[0])

    fscores, precs, recals = [], [], []
    metrics = None
    for i, t in enumerate(threshold):
        save_path = os.path.join(save_dir, "visualize", f"{threshold[i]:.2f}")
        os.makedirs(save_path, exist_ok=True)
        metrics = _compute_from(n1, n2, int(host[0, i]), int(host[1, i]), float(host[2, i]), float(host[3, i]))
        print(f"****metrics for threshold {t:.2f}****")
        print(metrics)
        with open(os.path.join(save_path, 'metrics.json'), 'w') as fh:
            json.dump(metrics, fh)
        fscores.append(metrics["fscore"])
        precs.append(metrics["prec"])
        recals.append(metrics["recal"])
    all_metrics = {"thresholds": [float(t) for t in threshold], "fscores": fscores, "precs": precs, "recals": recals}
    with open(os.path.join(save_dir, 'metrics.json'), 'w') as fh:
        json.dump(all_metrics, fh)
    print(f"fscores: {fscores}")
    print(f"precs: {precs}")
    print(f"recals: {recals}")
    return metrics


def get_opts(argv=None):
    """utils/eval_mesh.py::get_opts (same flags and spelling)"""
    from argparse import ArgumentParser

    parser = ArgumentParser(prog="python -m nrw.evaluation")
    parser.add_argument('--file_pred', type=str, required=True, help='ply file path for prediction')
    parser.add_argument('--file_trgt', type=str, required=True, help='ply file path for ground truth')
    parser.add_argument('--scene_config_path', type=str, required=True, help='scene config path')
    parser.add_argument('--mesh', default=False, action="store_true", help='whether prediction is mesh')
    parser.add_argument('--threshold', type=str, default="0.1",
                        help='threshold for precision and recall in cm, in order of [start,end,interval]')
    parser.add_argument('--bbx_name', type=str, default='eval_bbx', help='area to eval')
    parser.add_argument('--sfm_path', type=str, help='if set, eval will use sfm points to crop both gt and prediction')
    parser.add_argument('--track_lenth', type=float, help='track length threshold for sfm points')
    parser.add_argument('--reproj_error', type=float, help='mean reprojection error threshold for sfm points')
    parser.add_argument('--voxel_size', type=float, help='voxel size for sfm points to crop point clouds')
    parser.add_argument('--save_name', type=str, default='eval', help='visualization save path')
    return parser.parse_args(argv)


def main(argv=None):
    import yaml

    args = get_opts(argv)
    t = [float(num.strip()) for num in args.threshold.split(',')]
    thresholds = list(np.arange(t[0], t[1], t[2])) if len(t) == 3 else t     # [start, end, interval] or explicit values
    print(f"thresholds to eval: {thresholds}")
    with open(args.scene_config_path, "r") as yamlfile:
        scene_config = yaml.load(yamlfile, Loader=yaml.FullLoader)
    if args.sfm_path:
        print(f"crop with sfm in {args.sfm_path}")
        scene_config["sfm_path"] = args.sfm_path
        scene_config['eval_tl'] = args.track_lenth
        scene_config['eval_error'] = args.reproj_error
        scene_config['eval_voxel'] = args.voxel_size
    eval_mesh(args.file_pred, args.file_trgt, scene_config, args.mesh, threshold=thresholds, bbx_name=args.bbx_name,
              save_name=args.save_name)


if __name__ == "__main__":
    main()
