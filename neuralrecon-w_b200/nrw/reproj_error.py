"""Ground-truth alignment check of a scene on the GPU: a drop-in for tools/reproj_error.py (same names, flags, printed
lines and output files but `reproj_error.png`) that needs neither open3d, matplotlib, imageio nor pandas.

It tells whether the `sfm2gt` of a scene's config.yaml maps the COLMAP model onto the ground-truth scan.  Views whose
mean keypoint error is below --img_reproj_error are tested; every SfM point with a track longer than --track_length and an
error below --reproj_error is a track, with its observations in the tested views.  The ground-truth point of a track is
the nearest GT point (in camera depth) that lands on the pixel of its first observation (csrc/gtproj.cu: every GT point
is splatted once per pass into up to 16 views, and only queried pixels take an atomic); the error of the track is the
pixel distance of that point's projection to each of its observations, and the result is the mean over all of them.

    python -m nrw.reproj_error --data_dir SCENE --gt_pcd_path GT.ply [--reconstuct_path dense/sparse]

Writes samples/reproject/colmap_sfm.ply, samples/reproject/gt.ply and reprojects/<image name>.png under the working
directory.  Deviations from the reference are listed in INTEGRATION.md.
"""
import argparse
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import NrwError, check, ptr, stream_ptr
from .colmap import read_cameras, read_images, read_points3d
from .evaluation import _device, _scratch
from .mesh import read_ply, write_ply
from .reprojection import get_entrinsics, get_intrinsic  # noqa: F401  (the reference's names, re-exported)

# map entries (4 bytes each) one pass of first_hits may use beyond its largest view: more fit more views into a pass
MAP_PIXELS = 1 << 26


def get_image_id(imdata, data_dir):
    """tools/reproj_error.py::get_image_id: the ids of sorted(os.listdir(data_dir/dense/images))[2:] (the first two
    names are skipped, as in the reference) and {id: name}.  imdata: {id: Image} or read_images(with_points=True)."""
    files = sorted(os.listdir(os.path.join(data_dir, "dense", "images")))[2:]
    img_path_to_id, img_id_to_name = {}, {}
    for v in imdata.values():
        im = v[0] if isinstance(v, tuple) else v
        img_path_to_id[im.name] = im.id
        img_id_to_name[im.id] = im.name
    return [img_path_to_id[f] for f in files], img_id_to_name


def _view_row(K, E):
    K = np.asarray(K, np.float32).astype(np.float64)
    return np.concatenate([np.asarray(E, np.float64)[:3].reshape(-1), [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]])


def _projection(K, E):
    return (np.asarray(K, np.float32).astype(np.float64) @ np.asarray(E, np.float64)[:3]).reshape(-1)


def first_hits(points, intrinsics, world_to_cams, query_view, query_xy, device=0, map_pixels=None):
    """For each query (view index into intrinsics / world_to_cams, observation xy rounded to f32) the index of the point
    (f32 [N, 3]) nearest in camera depth whose projection rounds to the query's pixel, or -1 (rules in
    csrc/gtproj.cu).  Returns an int64 CUDA tensor [n_queries]; nothing is read back.  map_pixels bounds the map
    entries of one pass (default: every view in one pass, or MAP_PIXELS when that is larger)."""
    dev = _device(device)
    pts = torch.as_tensor(points)
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise NrwError(f"first_hits: expected points of shape [n, 3], got {tuple(pts.shape)}")
    if pts.shape[0] >= 1 << 32:
        raise NrwError(f"first_hits: {pts.shape[0]} points (need < 2^32)")
    pts = pts.to(device=dev, dtype=torch.float32).contiguous()
    if pts.shape[0] and not bool(torch.isfinite(pts).all()):
        raise NrwError("first_hits: points are not all finite")
    n_views = len(world_to_cams)
    if len(intrinsics) != n_views:
        raise NrwError(f"first_hits: {len(intrinsics)} intrinsics for {n_views} views")
    qv = np.asarray(query_view, np.int64).reshape(-1)
    qxy = np.asarray(query_xy, np.float32).reshape(-1, 2)
    if len(qxy) != len(qv):
        raise NrwError(f"first_hits: {len(qv)} query views and {len(qxy)} query xy")
    if len(qv) and (qv.min() < 0 or qv.max() >= n_views):
        raise NrwError(f"first_hits: a query view index is outside [0, {n_views})")
    pix = np.rint(qxy)
    if not (np.isfinite(pix).all() and (np.abs(pix) < 2 ** 30).all()):
        raise NrwError("first_hits: query xy must be finite and below 2^30 in magnitude")
    pix = pix.astype(np.int64)
    boxes = np.zeros((n_views, 4), np.int64)
    for v in np.unique(qv):
        p = pix[qv == v]
        lo, hi = p.min(0), p.max(0)
        boxes[v] = lo[0], lo[1], hi[0] - lo[0] + 1, hi[1] - lo[1] + 1
    views = np.stack([_view_row(K, E) for K, E in zip(intrinsics, world_to_cams)]) if n_views else np.zeros((0, 16))
    if not np.isfinite(views).all():
        raise NrwError("first_hits: a pose or intrinsic is not finite")
    area = boxes[:, 2] * boxes[:, 3]
    if map_pixels is None:
        map_pixels = min(int(area.sum()), max(int(area.max(initial=0)), MAP_PIXELS))
    L = _lib.lib()
    hit = torch.empty(len(qv), dtype=torch.int64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        nbytes = L.nrw_first_hit_scratch_bytes(len(qv), int(map_pixels))
        owner, scratch = _scratch(nbytes, dev)
        q_view = torch.as_tensor(qv.astype(np.int32), device=dev)
        q_xy = torch.as_tensor(qxy, device=dev)
        check(L.nrw_first_hit(ptr(pts), pts.shape[0], (C.c_double * views.size)(*views.reshape(-1).tolist()),
                              (C.c_int * boxes.size)(*boxes.reshape(-1).tolist()), n_views, ptr(q_view), ptr(q_xy),
                              len(qv), ptr(hit), ptr(status), scratch, int(nbytes), stream_ptr()), "nrw_first_hit")
    return hit


def obs_errors(X, view, xy, projections, device=0, with_uv=False):
    """Pixel distance (f64 CUDA tensor [n]) of the projection of X [n, 3] by projections[view] (P = K [R|t], [V, 3, 4])
    to xy [n, 2]; with_uv also returns the projections [n, 2]."""
    dev = _device(device)
    X = torch.as_tensor(np.asarray(X, np.float64).reshape(-1, 3), device=dev)
    xy = torch.as_tensor(np.asarray(xy, np.float64).reshape(-1, 2), device=dev)
    v = torch.as_tensor(np.asarray(view, np.int32).reshape(-1), device=dev)
    P = torch.as_tensor(np.asarray(projections, np.float64).reshape(-1, 12), device=dev)
    err = torch.empty(X.shape[0], dtype=torch.float64, device=dev)
    uv = torch.empty(X.shape[0], 2, dtype=torch.float64, device=dev) if with_uv else None
    with torch.cuda.device(dev):
        check(_lib.lib().nrw_obs_reproj_error(ptr(X), ptr(v), ptr(xy), X.shape[0], ptr(P), P.shape[0], ptr(err), ptr(uv),
                                              stream_ptr()), "nrw_obs_reproj_error")
    return (err, uv) if with_uv else err


def _keypoint_rows(pts3d, ids):
    """row of each point3D id in pts3d, -1 when it is -1 or not in the table"""
    ids = np.asarray(ids, np.int64)
    table = pts3d["id"].astype(np.int64)
    if len(table) == 0:
        return np.full(len(ids), -1, np.int64)
    order = np.argsort(table, kind="stable")
    pos = np.clip(np.searchsorted(table[order], ids), 0, len(table) - 1)
    return np.where((table[order][pos] == ids) & (ids >= 0), order[pos], -1)


def image_reproj_error(imdata, pts3d, img_ids, entrinsics_dict, intrinsics_dict, device=0):
    """tools/reproj_error.py::image_reproj_error: the mean pixel distance of each view's keypoints (imdata of
    read_images(with_points=True)) to the projections of their 3-D points (pts3d of read_points3d), float64
    [len(img_ids)].  Keypoints whose point3D id is -1 or not in the table are left out; a view without any gets NaN."""
    X, V, XY = [], [], []
    for k, id_ in enumerate(img_ids):
        _, xys, pids = imdata[id_]
        rows = _keypoint_rows(pts3d, pids)
        ok = rows >= 0
        X.append(pts3d["xyz"][rows[ok]])
        XY.append(xys[ok])
        V.append(np.full(int(ok.sum()), k, np.int32))
    P = [_projection(intrinsics_dict[i], entrinsics_dict[i]) for i in img_ids]
    n = sum(len(v) for v in V)
    err = obs_errors(np.concatenate(X) if n else np.zeros((0, 3)), np.concatenate(V) if n else np.zeros(0, np.int32),
                     np.concatenate(XY) if n else np.zeros((0, 2)), np.array(P).reshape(-1, 12), device).cpu().numpy()
    view = np.concatenate(V) if n else np.zeros(0, np.int64)
    sums = np.bincount(view, weights=err, minlength=len(img_ids))
    cnt = np.bincount(view, minlength=len(img_ids))
    with np.errstate(invalid="ignore", divide="ignore"):
        return sums / cnt


def _read_gt(gt_pcd_path):
    if not os.path.isfile(gt_pcd_path):
        raise NrwError(f"reproj_error: ground-truth cloud {gt_pcd_path} not found")
    gt = np.asarray(read_ply(gt_pcd_path)["vertices"]).astype(np.float32)
    if not np.isfinite(gt).all():
        raise NrwError(f"reproj_error: {gt_pcd_path} has non-finite points")
    return gt


def track_errors(data_dir, gt_pcd_path, sfm_to_gt, reconstuct_path="dense/sparse", track_length=200, reproj_error=0.4,
                 img_reproj_error=300, device=0, gt=None):
    """The check without files or prints.  Returns a dict: kept_views (image ids), track_point_ids (point3D id of each
    track), gt_index (GT index per track's reference observation, -1 = none), errors (f64 per observation of the
    tracks with a GT point) and obs_track (their track index), loss (their mean, summed in observation order),
    n_obs (all observations of the tracks), ref_view / ref_xy (each track's reference observation: index into
    kept_views, xy), and for the output files track_xyz, gt_points, obs_image_id, obs_xy, uv, image_errors, names and
    whs."""
    base = os.path.join(data_dir, reconstuct_path)
    imdata = read_images(os.path.join(base, "images.bin"), with_points=True)
    camdata = read_cameras(os.path.join(base, "cameras.bin"))
    pts3d = read_points3d(os.path.join(base, "points3D.bin"), with_tracks=True)
    gt = _read_gt(gt_pcd_path) if gt is None else gt
    sfm_to_gt = np.asarray(sfm_to_gt, np.float64)
    img_ids, img_id_to_name = get_image_id(imdata, data_dir)
    ims = {k: v[0] for k, v in imdata.items()}
    entrinsics = get_entrinsics(ims, img_ids)
    E = {id_: entrinsics[i] for i, id_ in enumerate(img_ids)}
    K, whs = get_intrinsic(camdata, img_ids, ims)
    img_err = image_reproj_error(imdata, pts3d, img_ids, E, K, device)
    kept = [id_ for id_, e in zip(img_ids, img_err) if e < img_reproj_error]
    print(f"selected {len(kept)} view for testing.")
    if not kept:
        raise NrwError(f"reproj_error: no view has a mean keypoint error below {img_reproj_error}")

    # observations of the kept tracks in the kept views, in points3D order, then track order
    tl = pts3d["track_length"]
    pt_of_obs = np.repeat(np.arange(len(tl)), tl)
    img = pts3d["track_image_id"].astype(np.int64)
    ks = np.sort(np.array(kept, np.int64))
    in_kept = ks[np.clip(np.searchsorted(ks, img), 0, len(ks) - 1)] == img
    keep_pt = (tl > track_length) & (pts3d["error"] < reproj_error)
    sel = np.nonzero(keep_pt[pt_of_obs] & in_kept)[0]
    tracks = np.unique(pt_of_obs[sel])
    if len(tracks) == 0:
        raise NrwError("reproj_error: no track passes --track_length and --reproj_error with an observation in a kept view")
    obs_track = np.searchsorted(tracks, pt_of_obs[sel])
    obs_view = _kept_index(kept, img[sel])
    p2 = pts3d["track_point2d_idx"][sel].astype(np.int64)
    obs_xy = np.empty((len(sel), 2))
    for k, id_ in enumerate(kept):
        m = obs_view == k
        xys = imdata[id_][1]
        if m.any() and (p2[m].min() < 0 or p2[m].max() >= len(xys)):
            raise NrwError(f"reproj_error: a track refers to a keypoint image {id_} does not have")
        obs_xy[m] = xys[p2[m]]
    first = np.searchsorted(obs_track, np.arange(len(tracks)))
    inv_s = np.linalg.inv(sfm_to_gt)
    Ks = [K[i] for i in kept]
    Egt = [E[i] @ inv_s for i in kept]
    hit = first_hits(gt, Ks, Egt, obs_view[first], obs_xy[first], device).cpu().numpy()
    use = hit[obs_track] >= 0
    if not use.any():
        raise NrwError("reproj_error: no track's reference pixel receives a ground-truth point")
    X = gt[hit[obs_track[use]]].astype(np.float64)
    P = np.array([_projection(k, e) for k, e in zip(Ks, Egt)])
    err, uv = obs_errors(X, obs_view[use], obs_xy[use], P, device, with_uv=True)
    err, uv = err.cpu().numpy(), uv.cpu().numpy()
    return {"kept_views": np.array(kept, np.int64), "track_point_ids": pts3d["id"][tracks].astype(np.int64),
            "gt_index": hit, "errors": err, "obs_track": obs_track[use], "loss": float(np.sum(err) / len(err)),
            "n_obs": len(sel), "track_xyz": pts3d["xyz"][tracks], "gt_points": gt[hit[hit >= 0]].astype(np.float64),
            "obs_image_id": np.array(kept, np.int64)[obs_view[use]], "obs_xy": obs_xy[use], "uv": uv,
            "ref_view": obs_view[first], "ref_xy": obs_xy[first],
            "image_errors": img_err, "names": img_id_to_name, "whs": whs}


def _kept_index(kept, img):
    """position in `kept` of each image id of img (all in kept)"""
    order = np.argsort(np.array(kept, np.int64), kind="stable")
    return order[np.searchsorted(np.array(kept, np.int64)[order], img)]


def reproject_vis(r, out_dir="reprojects"):
    """tools/reproj_error.py::reproject_vis: per observed image a black image with the GT projections in green, then
    the SfM observations in red, at truncated coordinates clamped into the image"""
    from PIL import Image

    print("visualize imgs...")
    os.makedirs(out_dir, exist_ok=True)
    for id_ in np.unique(r["obs_image_id"]):
        w, h = (int(a) for a in r["whs"][int(id_)])
        img = np.zeros((h, w, 3), np.uint8)
        m = r["obs_image_id"] == id_
        wh = np.array([w - 1, h - 1], np.float64)
        gt = np.clip(np.trunc(r["uv"][m]), 0, wh).astype(np.int64)
        sfm = np.clip(np.trunc(r["obs_xy"][m]), 0, wh).astype(np.int64)
        img[gt[:, 1], gt[:, 0]] = (0, 255, 0)
        img[sfm[:, 1], sfm[:, 0]] = (255, 0, 0)
        Image.fromarray(img).save(os.path.join(out_dir, f"{r['names'][int(id_)]}.png"))


def gt_reproject_error(data_dir, gt_pcd_path, sfm_to_gt, reconstuct_path, track_length=200, reproj_error=0.4,
                       batch_size=2, img_reproj_error=300):
    """tools/reproj_error.py::gt_reproject_error: prints and returns the mean re-projection error of the GT points of
    the tracks and writes samples/reproject/{colmap_sfm,gt}.ply and reprojects/<name>.png.  batch_size is accepted and
    ignored (the result does not depend on it)."""
    r = track_errors(data_dir, gt_pcd_path, sfm_to_gt, reconstuct_path, track_length, reproj_error, img_reproj_error)
    os.makedirs("samples/reproject", exist_ok=True)
    write_ply("samples/reproject/colmap_sfm.ply", r["track_xyz"], double=True)
    inv_s = np.linalg.inv(np.asarray(sfm_to_gt, np.float64))
    g = r["gt_points"]
    write_ply("samples/reproject/gt.ply", (inv_s[:3, :3] @ g.T).T + inv_s[:3, 3], double=True)
    n_miss = int((r["gt_index"] < 0).sum())
    print(f"avg re-projection error {r['loss']}, {len(r['errors'])}/{r['n_obs']}, "
          f"{n_miss} tracks without a ground-truth point")
    reproject_vis(r)
    return r["loss"]


def get_opts(argv=None):
    """tools/reproj_error.py::get_opts (same flags and defaults)"""
    parser = argparse.ArgumentParser(prog="python -m nrw.reproj_error")
    parser.add_argument('--data_dir', type=str, default='/nas/datasets/IMC/phototourism/training_set/brandenburg_gate',
                        help='path to data folder')
    parser.add_argument('--gt_pcd_path', type=str,
                        default="/nas/datasets/OpenHeritage3D/pro/brandenburg_gate/bg_sampled_0.01_cropped.ply",
                        help='target point cloud')
    parser.add_argument('--reconstuct_path', type=str, default="dense/sparse", help='reconstruction work space')
    parser.add_argument('--track_length', type=int, default='200', help='track length threshold')
    parser.add_argument('--reproj_error', type=float, default='0.4', help='reproj error threshold')
    parser.add_argument('--batch_size', type=int, default='2', help='accepted and ignored')
    parser.add_argument('--img_reproj_error', type=float, default='300',
                        help='filter out image with reproj error above this threshold')
    return parser.parse_args(argv)


def main(argv=None):
    import yaml

    args = get_opts(argv)
    cfg = os.path.join(args.data_dir, "config.yaml")
    if not os.path.isfile(cfg):
        raise NrwError(f"reproj_error: {cfg} not found")
    with open(cfg, "r") as fh:
        scene_config = yaml.load(fh, Loader=yaml.FullLoader)
    return gt_reproject_error(args.data_dir, args.gt_pcd_path, np.array(scene_config["sfm2gt"]), args.reconstuct_path,
                              args.track_length, args.reproj_error, args.batch_size, args.img_reproj_error)


if __name__ == "__main__":
    main()
