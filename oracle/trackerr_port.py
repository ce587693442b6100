"""Numpy restatement of the ground-truth alignment check (nrw/reproj_error.py, csrc/gtproj.cu), TEST INFRASTRUCTURE.

Rules, as csrc/gtproj.cu states them:
* `first_hit`: a ground-truth point (fp32) is taken to a view's camera in fp64, c_r = ((E[r,0]·x + E[r,1]·y) +
  E[r,2]·z) + E[r,3], and projected as u = (fx·xc + cx·zc) / zc, v = (fy·yc + cy·zc) / zc.  Its pixel is (rint(u),
  rint(v)) and it needs zc > 0.  A query's pixel is rint of its fp32 xy.  The winner on a query's pixel has the smallest
  fp32 depth (zc rounded to nearest), equal depths going to the smaller index; -1 when no point lands there.
* `obs_error`: p = P·[X, 1] row by row in the same order, (u, v) = p[:2] / p[2], the distance to the observation.
* `gt_reproject_error`: the whole pipeline from already-read arrays, with the deviations of INTEGRATION.md (a track whose
  reference pixel gets no point is dropped; keypoints without a valid 3-D point are left out of a view's mean).

Also: a seeded scene for exact comparisons with the reference (`make_scene`), COLMAP writers for it, and the unmodified
tools/reproj_error.py with functional stand-ins for open3d's point-cloud I/O (`load_reference`).
"""
import os
import struct

import numpy as np


def _row(M, x, y, z):
    return ((M[0] * x + M[1] * y) + M[2] * z) + M[3]


def pixels(points, view):
    """(pixel x, pixel y, fp32 depth, in front) of points f32 [n, 3] in one view f64 [16] (E[3,4], fx, fy, cx, cy)"""
    p = np.asarray(points, np.float32).astype(np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    E = np.asarray(view[:12], np.float64).reshape(3, 4)
    fx, fy, cx, cy = (float(a) for a in view[12:16])
    xc, yc, zc = _row(E[0], x, y, z), _row(E[1], x, y, z), _row(E[2], x, y, z)
    with np.errstate(all="ignore"):
        u = (fx * xc + cx * zc) / zc
        v = (fy * yc + cy * zc) / zc
    return np.rint(u), np.rint(v), zc.astype(np.float32), zc > 0


def first_hit(points, views, q_view, q_xy):
    """hit int64 [n_q] (see the module docstring); views f64 [n_views, 16]"""
    points = np.asarray(points, np.float32)
    q_view = np.asarray(q_view, np.int64)
    q_xy = np.asarray(q_xy, np.float32)
    hit = np.full(len(q_view), -1, np.int64)
    idx = np.arange(len(points), dtype=np.uint64)
    for v in np.unique(q_view):
        qs = np.nonzero(q_view == v)[0]
        pu, pv, z32, front = pixels(points, views[v])
        key = (z32.view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx
        for q in qs:
            qx, qy = np.rint(q_xy[q].astype(np.float64))
            m = front & (pu == qx) & (pv == qy)
            if m.any():
                hit[q] = int(key[m].min() & np.uint64(0xFFFFFFFF))
    return hit


def obs_error(X, view, xy, P):
    """(err f64 [n], uv f64 [n, 2]) of points X [n, 3] in views P f64 [n_views, 3, 4]"""
    X = np.asarray(X, np.float64)
    P = np.asarray(P, np.float64)[np.asarray(view)]
    p = [_row(P[:, r].T, X[:, 0], X[:, 1], X[:, 2]) for r in range(3)]
    u, v = p[0] / p[2], p[1] / p[2]
    du, dv = u - xy[:, 0], v - xy[:, 1]
    return np.sqrt(du * du + dv * dv), np.stack([u, v], 1)


def projection(K, E):
    """P = K·E[:3] in fp64 from the float32 K"""
    return np.asarray(K, np.float32).astype(np.float64) @ np.asarray(E, np.float64)[:3]


def view_row(K, E):
    """the f64 [16] view of first_hit: E[:3] row-major, fx, fy, cx, cy"""
    K = np.asarray(K, np.float32).astype(np.float64)
    return np.concatenate([np.asarray(E, np.float64)[:3].reshape(-1), [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]])


def image_errors(views, Ks, Es, pt_index, pt_xyz):
    """per-view mean keypoint error; views: [(xys f64 [k, 2], point3D ids [k])]; pt_index: {point3D id: row}.  Keypoints
    without a valid point are left out; a view without any gets NaN."""
    out = np.empty(len(views))
    for i, ((xys, ids), K, E) in enumerate(zip(views, Ks, Es)):
        rows = np.array([pt_index.get(int(j), -1) for j in ids], np.int64)
        ok = rows >= 0
        if not ok.any():
            out[i] = np.nan
            continue
        e, _ = obs_error(pt_xyz[rows[ok]], np.zeros(int(ok.sum()), np.int64), xys[ok], projection(K, E)[None])
        out[i] = np.sum(e) / len(e)
    return out


def gt_reproject_error(img_ids, views, Ks, Es, pts, gt, sfm_to_gt, track_length, reproj_error, img_reproj_error):
    """The check from read arrays.  img_ids: the tested view ids (get_image_id's order); views {id: (xys, point3D ids)};
    Ks, Es {id: K [3,3], E [4,4]}; pts: dict of nrw.colmap.read_points3d(with_tracks=True); gt f32 [N, 3].
    Returns the dict of nrw.reproj_error.track_errors plus `loss`, `uv` and `gt_index`."""
    ids = pts["id"].astype(np.int64)
    pt_index = {int(j): r for r, j in enumerate(ids)}
    img_err = image_errors([views[i] for i in img_ids], [Ks[i] for i in img_ids], [Es[i] for i in img_ids], pt_index,
                           pts["xyz"])
    kept = [i for i, e in zip(img_ids, img_err) if e < img_reproj_error]
    vpos = {i: k for k, i in enumerate(kept)}
    inv_s = np.linalg.inv(sfm_to_gt)
    track_ids, obs_view, obs_xy, obs_track = [], [], [], []
    off = pts["track_offsets"]
    for r in range(len(ids)):
        if not (pts["track_length"][r] > track_length and pts["error"][r] < reproj_error):
            continue
        n0 = len(obs_view)
        for j in range(off[r], off[r + 1]):
            im, p2 = int(pts["track_image_id"][j]), int(pts["track_point2d_idx"][j])
            if im not in vpos:
                continue
            obs_view.append(vpos[im])
            obs_xy.append(views[im][0][p2])
            obs_track.append(len(track_ids))
        if len(obs_view) > n0:
            track_ids.append(r)
    obs_view = np.array(obs_view, np.int64)
    obs_xy = np.array(obs_xy, np.float64).reshape(-1, 2)
    obs_track = np.array(obs_track, np.int64)
    first = np.searchsorted(obs_track, np.arange(len(track_ids)))
    gt_views = np.stack([view_row(Ks[i], Es[i] @ inv_s) for i in kept]) if kept else np.zeros((0, 16))
    gt_index = first_hit(gt, gt_views, obs_view[first], obs_xy[first].astype(np.float32))
    use = gt_index[obs_track] >= 0
    X = np.asarray(gt, np.float32)[gt_index[obs_track[use]]].astype(np.float64)
    P = np.stack([projection(Ks[i], Es[i] @ inv_s) for i in kept]) if kept else np.zeros((0, 3, 4))
    err, uv = obs_error(X, obs_view[use], obs_xy[use], P)
    return {"image_errors": img_err, "kept_views": np.array(kept, np.int64), "track_point_ids": ids[track_ids],
            "gt_index": gt_index, "obs_view": obs_view, "obs_xy": obs_xy, "obs_track": obs_track, "obs_used": use,
            "errors": err, "uv": uv, "loss": float(np.sum(err) / len(err)) if len(err) else float("nan")}


# ---- seeded scene -------------------------------------------------------------------------------------------------

def write_cameras(path, cams):
    """cameras.bin; cams: [(id, model id, width, height, params)]"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(cams)))
        for cid, mid, w, h, params in cams:
            fh.write(struct.pack("<iiQQ", cid, mid, w, h))
            fh.write(struct.pack("<" + "d" * len(params), *[float(p) for p in params]))


def write_images(path, images):
    """images.bin; images: [(id, qvec, tvec, camera id, name, xys [k, 2], point3D ids [k])]"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(images)))
        for iid, q, t, cid, name, xys, pids in images:
            fh.write(struct.pack("<idddddddi", iid, *[float(x) for x in q], *[float(x) for x in t], cid))
            fh.write(name.encode("utf-8") + b"\x00")
            fh.write(struct.pack("<Q", len(pids)))
            rec = np.empty(len(pids), dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
            rec["x"], rec["y"], rec["id"] = xys[:, 0], xys[:, 1], pids
            fh.write(rec.tobytes())


def write_points3d(path, ids, xyz, error, tracks):
    """points3D.bin; tracks: per point a list of (image id, point2D index)"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(ids)))
        for i, p, e, tr in zip(ids, xyz, error, tracks):
            fh.write(struct.pack("<QdddBBBd", int(i), *[float(x) for x in p], 10, 20, 30, float(e)))
            fh.write(struct.pack("<Q", len(tr)))
            fh.write(np.asarray(tr, "<i4").reshape(-1).tobytes())


def _qvec(R):
    """unit quaternion (w, x, y, z) of a rotation matrix (Shepperd: from the largest component)"""
    t = np.trace(R)
    k = int(np.argmax([t, R[0, 0], R[1, 1], R[2, 2]]))
    if k == 0:
        s = 2 * np.sqrt(1 + t)
        q = [s / 4, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    elif k == 1:
        s = 2 * np.sqrt(1 + R[0, 0] - R[1, 1] - R[2, 2])
        q = [(R[2, 1] - R[1, 2]) / s, s / 4, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s]
    elif k == 2:
        s = 2 * np.sqrt(1 + R[1, 1] - R[0, 0] - R[2, 2])
        q = [(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, s / 4, (R[1, 2] + R[2, 1]) / s]
    else:
        s = 2 * np.sqrt(1 + R[2, 2] - R[0, 0] - R[1, 1])
        q = [(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, s / 4]
    q = np.array(q)
    return q / np.linalg.norm(q)


def _qrot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def similarity(rng, scale):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    S = np.eye(4)
    S[:3, :3], S[:3, 3] = scale * _qrot(q), rng.normal(size=3)
    return S


def make_scene(seed=0, n_views=6, width=64, height=48, n_gt=60000, n_tracks=60, scale=1.7, margin=1e-3, tie=1e-5):
    """A seeded scene on which the reference and the restatement must agree exactly: a sim(3) sfm2gt with scale, GT
    points on two wavy sheets (many per pixel), mirrored copies behind the cameras that land on the same pixels, exact
    duplicates, no GT projection within `margin` px of a rounding edge in any view, no observation near one either, no
    depth tie within `tie` relative except exact duplicates at the winning pixel, every reference pixel hit, one view
    with a bad keypoint error, tracks that fail the length or error threshold, and no -1 keypoints.

    Returns a dict of arrays: names, ids, qvec, K (f32 [V,3,3]), E [V,4,4], wh, gt (f32 [N,3]), sfm2gt,
    xys / pids per view (object arrays), pt_id, pt_xyz, pt_err, track (object array of [(image id, idx)]), n_listed
    (views named in dense/images, the first two of which are skipped), thresholds."""
    rng = np.random.default_rng(seed)
    S = similarity(rng, scale)
    S_inv = np.linalg.inv(S)
    ids = [7 + 5 * k for k in range(n_views + 2)]      # two extra views that get_image_id skips
    Ks, Es, qs = [], [], []
    for k in range(n_views + 2):
        th, ph = np.deg2rad(rng.uniform(0, 12)), rng.uniform(0, 2 * np.pi)
        eye = 5.0 * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        z = -eye / np.linalg.norm(eye)
        x = np.cross(z, [rng.normal() * 0.1, 1.0, 0.0])
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        q = _qvec(R)
        R = _qrot(q)                                      # what qvec2rotmat gives back
        qs.append(q)
        E = np.eye(4)
        E[:3, :3], E[:3, 3] = R, -R @ eye
        Es.append(E)
        f = rng.uniform(55, 65)
        Ks.append(np.array([[f, 0, width / 2 + rng.uniform(-2, 2)], [0, f * 1.01, height / 2 + rng.uniform(-2, 2)],
                            [0, 0, 1]], np.float32))
    # GT points in the SfM frame: two sheets z = 0.6 sin.. and z = -0.4 + .., then into the GT frame
    xy = rng.uniform(-2.2, 2.2, (n_gt, 2))
    zs = np.where(rng.random(n_gt) < 0.5, 0.15 * np.sin(2 * xy[:, 0]) * np.cos(xy[:, 1]), -0.5 + 0.1 * xy[:, 0])
    sfm = np.concatenate([xy, zs[:, None]], 1)
    gt = (S[:3, :3] @ sfm.T).T + S[:3, 3]
    gt = gt.astype(np.float32)
    views_gt = [view_row(K, E @ S_inv) for K, E in zip(Ks, Es)]

    def edge_free(points):
        ok = np.ones(len(points), bool)
        for v in views_gt:
            u, w, _, _ = _raw_uv(points, v)
            ok &= (np.abs(u - np.floor(u) - 0.5) > margin) & (np.abs(w - np.floor(w) - 0.5) > margin)
        return ok

    gt = gt[edge_free(gt)]
    # mirrored copies behind view 2 of the tested views (same pixel, negative depth)
    v = views_gt[4]
    E = v[:12].reshape(3, 4)
    cam = (E[:, :3] @ gt[:4000].astype(np.float64).T).T + E[:, 3]
    mir = (np.linalg.inv(E[:, :3]) @ (-cam - E[:, 3]).T).T.astype(np.float32)
    gt = np.concatenate([gt, mir[edge_free(mir)]])
    dup = rng.choice(len(gt), 200, replace=False)
    gt = np.concatenate([gt, gt[dup]])                   # exact duplicates (later indices)
    n_tested = n_views                                    # ids[2:] are tested
    # tracks: an SfM point near a GT point, observed in 3..n_views tested views (and sometimes a skipped view)
    pix = [pixels(gt, v) for v in views_gt]
    pt_xyz, pt_err, tracks, xys, pids = [], [], [], [[] for _ in ids], [[] for _ in ids]
    bad_view = 3                                          # index into ids: a tested view with large keypoint errors
    tries = 0
    while len(pt_xyz) < n_tracks and tries < 100 * n_tracks:
        tries += 1
        g = int(rng.integers(len(gt)))
        X = (S_inv[:3, :3] @ gt[g].astype(np.float64)) + S_inv[:3, 3] + rng.normal(0, 0.004, 3)
        obs_views = list(rng.permutation(np.arange(2, n_views + 2))[:int(rng.integers(3, n_views + 1))])
        if rng.random() < 0.3:
            obs_views.insert(int(rng.integers(len(obs_views) + 1)), int(rng.integers(0, 2)))
        obs = []
        for k in obs_views:
            P = projection(Ks[k], Es[k])
            p = P @ np.append(X, 1.0)
            o = p[:2] / p[2] + rng.normal(0, 0.3, 2) + (25.0 if k == bad_view else 0.0)
            o32 = o.astype(np.float32).astype(np.float64)
            if np.any(np.abs(o32 - np.floor(o32) - 0.5) < 0.01):
                break
            obs.append((k, o))
        else:
            ref = next((k for k, _ in obs if 2 <= k and k != bad_view), None)
            if ref is None:
                continue
            # the reference observation is the first in a kept view: move it to the front of the kept ones
            kx, ky = np.rint(dict(obs)[ref].astype(np.float32).astype(np.float64))
            pu, pv, z32, front = pix[ref]
            m = front & (pu == kx) & (pv == ky)
            if not m.any():
                continue
            zs_ = np.sort(np.unique(z32[m]).astype(np.float64))
            if len(zs_) > 1 and (zs_[1] - zs_[0]) <= tie * zs_[0]:
                continue
            obs = [o for o in obs if o[0] == ref] + [o for o in obs if o[0] != ref]
            tr = []
            for k, o in obs:
                tr.append((ids[k], len(xys[k])))
                xys[k].append(o)
                pids[k].append(0)          # filled below
            tracks.append(tr)
            pt_xyz.append(X)
            pt_err.append(rng.uniform(0, 0.3))
    n = len(pt_xyz)
    pt_id = 1000 + 3 * np.arange(n + 6)
    # six extra points: three with short tracks, three with a large error, observed in the tested views
    for e in range(6):
        X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 0.0])
        tr = []
        for k in range(2, 2 + (2 if e < 3 else 4)):
            p = projection(Ks[k], Es[k]) @ np.append(X, 1.0)
            tr.append((ids[k], len(xys[k])))
            xys[k].append(p[:2] / p[2] + rng.normal(0, 0.3, 2))
            pids[k].append(0)
        tracks.append(tr)
        pt_xyz.append(X)
        pt_err.append(0.2 if e < 3 else 2.0)
    for r, tr in enumerate(tracks):
        for im, j in tr:
            pids[ids.index(im)][j] = int(pt_id[r])
    obj = lambda xs: np.array([np.asarray(x) for x in xs] + [None], dtype=object)[:-1]
    return {"names": np.array([f"view_{k:02d}.jpg" for k in range(len(ids))]), "ids": np.array(ids, np.int64),
            "qvec": np.stack(qs), "K": np.stack(Ks), "E": np.stack(Es), "wh": np.array([[width, height]] * len(ids), np.int64), "gt": gt,
            "sfm2gt": S, "xys": obj([np.array(x, np.float64).reshape(-1, 2) for x in xys]),
            "pids": obj([np.array(p, np.int64) for p in pids]), "pt_id": pt_id.astype(np.int64),
            "pt_xyz": np.array(pt_xyz, np.float64), "pt_err": np.array(pt_err, np.float64),
            "track": obj([np.array(t, np.int64).reshape(-1, 2) for t in tracks]),
            "track_length": 2, "reproj_error": 1.0, "img_reproj_error": 5.0}


def _raw_uv(points, view):
    p = np.asarray(points, np.float32).astype(np.float64)
    E = np.asarray(view[:12], np.float64).reshape(3, 4)
    fx, fy, cx, cy = (float(a) for a in view[12:16])
    xc, yc, zc = (_row(E[r], p[:, 0], p[:, 1], p[:, 2]) for r in range(3))
    with np.errstate(all="ignore"):
        return (fx * xc + cx * zc) / zc, (fy * yc + cy * zc) / zc, zc, zc > 0


def write_scene(d, sc, gt_path=None):
    """data_dir layout of the reference: dense/images/<names>, dense/sparse/{cameras,images,points3D}.bin, config.yaml;
    the GT cloud as a float32 PLY at gt_path (default d/gt.ply).  Returns gt_path."""
    import yaml

    from nrw.mesh import write_ply

    os.makedirs(os.path.join(d, "dense", "sparse"), exist_ok=True)
    os.makedirs(os.path.join(d, "dense", "images"), exist_ok=True)
    for name in sc["names"]:
        open(os.path.join(d, "dense", "images", str(name)), "wb").close()
    cams = [(k + 1, 1, int(w), int(h), (K[0, 0], K[1, 1], K[0, 2], K[1, 2])) for k, (K, (w, h)) in enumerate(zip(sc["K"], sc["wh"]))]
    write_cameras(os.path.join(d, "dense", "sparse", "cameras.bin"), cams)
    images = [(int(i), q, E[:3, 3], k + 1, str(n), x, p)
              for k, (i, q, E, n, x, p) in enumerate(zip(sc["ids"], sc["qvec"], sc["E"], sc["names"], sc["xys"], sc["pids"]))]
    write_images(os.path.join(d, "dense", "sparse", "images.bin"), images)
    write_points3d(os.path.join(d, "dense", "sparse", "points3D.bin"), sc["pt_id"], sc["pt_xyz"], sc["pt_err"],
                   [t.tolist() for t in sc["track"]])
    with open(os.path.join(d, "config.yaml"), "w") as fh:
        yaml.safe_dump({"sfm2gt": np.asarray(sc["sfm2gt"]).tolist()}, fh)
    gt_path = gt_path or os.path.join(d, "gt.ply")
    write_ply(gt_path, np.asarray(sc["gt"], np.float32))
    return gt_path


# ---- the unmodified reference -------------------------------------------------------------------------------------

def load_reference():
    """tools/reproj_error.py with open3d's read_point_cloud reading our PLY files and write_point_cloud recording rows
    (into `mod.written`); imageio.imwrite records images (into `mod.images`), plt is inert.  Needs `.cuda()` to be the
    identity on a machine without a GPU."""
    from unittest import mock

    from oracle import reproj_port

    mod = reproj_port.load_reproj().reproj_error
    mod.written, mod.images = {}, {}

    def read_point_cloud(path):
        from nrw.mesh import read_ply

        return mock.Mock(points=np.asarray(read_ply(path)["vertices"], np.float64))

    def write_point_cloud(path, pcd):
        mod.written[path] = np.asarray(pcd.points, np.float64)

    o3d = mock.MagicMock()
    o3d.io.read_point_cloud = read_point_cloud
    o3d.io.write_point_cloud = write_point_cloud
    o3d.utility.Vector3dVector = lambda a: np.asarray(a)
    o3d.geometry.PointCloud = lambda: mock.Mock(spec=["points"])
    imageio = mock.MagicMock()
    imageio.imwrite = lambda path, img: mod.images.__setitem__(path, np.asarray(img))
    mod.o3d, mod.imageio, mod.plt = o3d, imageio, mock.MagicMock()
    return mod
