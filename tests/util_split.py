"""Seeded synthetic scene for the scene-split tests: PINHOLE cameras only, lossless PNG images of odd sizes (one >= 1000 px
wide), int64 semantic maps (savez_compressed), COLMAP binaries with keypoints (so nrw.prepare_data_cache can run on the
result), config.yaml with origin and radius, and a dense/sparse_filtered_3 model.  Besides cameras on a ring that look at
the scene sphere with different focal lengths, it holds a camera inside the sphere, one looking away from it, one whose
rays graze it, two cameras missing from sparse_filtered_3 (one rescued by the fx, fy > 2000 rule) and one image whose
semantic map is all "person"."""
import os
import struct

import numpy as np

from util_cache import look_at, qvec2rotmat

ORIGIN = [0.1, -0.2, 0.3]
RADIUS = 1.0
# (kind, width, height, focal / width)
CAMERAS = [("ring", 1001, 67, 0.9), ("ring", 81, 61, 0.5), ("ring", 95, 73, 1.3), ("ring", 63, 49, 2.1), ("ring", 77, 59, 0.7),
           ("ring", 91, 65, 3.0), ("ring", 69, 55, 1.7), ("ring", 85, 63, 1.1), ("inside", 73, 51, 0.8), ("away", 99, 71, 0.9),
           ("graze", 65, 45, 1.0), ("covis_rescued", 87, 57, None), ("covis_dropped", 79, 53, 1.2), ("transient", 83, 61, 1.5)]
FULLY_TRANSIENT = "img_013.png"
COVIS_RESCUED, COVIS_DROPPED = "img_011.png", "img_012.png"


def _pose(kind, i, n, rng):
    s = np.asarray(ORIGIN)
    ang = 2 * np.pi * i / n
    C = s + np.array([4 * np.cos(ang), 4 * np.sin(ang), 0.5 + 0.2 * rng.standard_normal()])
    if kind == "inside":
        C = s + np.array([0.2, -0.1, 0.15])
        target = C + np.array([1.0, 0.3, -0.2])
    elif kind == "away":
        target = C + (C - s)
    elif kind == "graze":
        f = (s - C) / np.linalg.norm(s - C)
        side = np.cross(f, [0, 0, 1.0])
        target = s + side / np.linalg.norm(side) * RADIUS       # the silhouette runs through the image centre
    else:
        target = s
    q = look_at(C - target, rng)                                 # look_at looks at the world origin from its argument
    R = qvec2rotmat(q)
    return q / np.linalg.norm(q), -R @ C


def write_scene(root, seed=0, n_points=2000, cameras=None, ext="png"):
    """Writes the scene under root (its basename is the scene name); returns a dict describing it.  cameras (default
    CAMERAS) and the image format can be replaced, e.g. by many ring cameras and "jpg" for a benchmark."""
    cameras = CAMERAS if cameras is None else cameras
    from PIL import Image

    rng = np.random.default_rng(seed)
    dense = os.path.join(root, "dense")
    for d in ("sparse", "sparse_filtered_3", "images"):
        os.makedirs(os.path.join(dense, d), exist_ok=True)
    os.makedirs(os.path.join(root, "semantic_maps"), exist_ok=True)
    xyz = np.asarray(ORIGIN) + rng.uniform(-1, 1, (n_points, 3)) * 0.9
    ids = np.arange(n_points, dtype=np.int64) * 2 + 1
    err = rng.uniform(0.2, 2.0, n_points)
    track = rng.integers(1, 6, n_points)
    n = len(cameras)
    cams, images = [], []
    for i, (kind, W, H, fw) in enumerate(cameras):
        fx = 2500.0 if kind == "covis_rescued" else fw * W
        fy = fx * 1.01
        cams.append((i + 1, 1, W, H, [fx, fy, W / 2 + 0.3, H / 2 - 0.2]))
        q, t = _pose(kind, i, n, rng)
        R = qvec2rotmat(q)
        Xc = xyz @ R.T + t
        u = fx * Xc[:, 0] / np.where(Xc[:, 2] > 0, Xc[:, 2], 1) + W / 2
        v = fy * Xc[:, 1] / np.where(Xc[:, 2] > 0, Xc[:, 2], 1) + H / 2
        sel = np.nonzero((Xc[:, 2] > 0) & (u > 0) & (u < W - 1) & (v > 0) & (v < H - 1))[0]
        sel = rng.choice(sel, min(len(sel), 300), replace=False) if len(sel) else sel
        xy = np.stack([u[sel], v[sel]], 1) + rng.normal(0, 0.3, (len(sel), 2))
        pid = ids[sel]
        name = f"img_{i:03d}.{ext}"
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(dense, "images", name))
        if name == FULLY_TRANSIENT:
            sem = np.full((H, W), 12, np.int64)
        else:                     # a per-image share of transient labels (person, car, tree, bicycle, minibike) among others
            p = rng.uniform(0.05, 0.6)
            h4, w4 = (H + 3) // 4, (W + 3) // 4               # labels in 4 x 4 pixel blocks
            sem = np.where(rng.random((h4, w4)) < p, rng.choice([12, 20, 4, 127, 116], (h4, w4)),
                           rng.choice([0, 1, 2, 6, 9, 25], (h4, w4))).astype(np.int64)
            sem = np.repeat(np.repeat(sem, 4, 0), 4, 1)[:H, :W]
        np.savez_compressed(os.path.join(root, "semantic_maps", f"img_{i:03d}.npz"), sem)
        images.append((i + 10, q, t, i + 1, name, xy, pid))
    _write_cameras(os.path.join(dense, "sparse", "cameras.bin"), cams)
    _write_images(os.path.join(dense, "sparse", "images.bin"), images)
    _write_images(os.path.join(dense, "sparse_filtered_3", "images.bin"),
                  [im for im in images if im[4] not in (COVIS_RESCUED, COVIS_DROPPED)])
    with open(os.path.join(dense, "sparse", "points3D.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", n_points))
        for k in range(n_points):
            fh.write(struct.pack("<QdddBBBdQ", int(ids[k]), *xyz[k], 1, 2, 3, err[k], int(track[k])))
            for _ in range(int(track[k])):
                fh.write(struct.pack("<ii", 1, 0))
    with open(os.path.join(root, "config.yaml"), "w") as fh:
        fh.write(f"origin: [{ORIGIN[0]}, {ORIGIN[1]}, {ORIGIN[2]}]\nradius: {RADIUS}\n")
        fh.write("sfm2gt: [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]\n")
        fh.write("eval_bbx: [[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]]\n")
        fh.write("voxel_size: 0.1\nmin_track_length: 1\n")
    return {"root": root, "images": images, "cameras": cams, "names": [im[4] for im in images]}


def _write_cameras(path, cams):
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(cams)))
        for cid, mid, W, H, params in cams:
            fh.write(struct.pack("<iiQQ", cid, mid, W, H))
            fh.write(struct.pack("<" + "d" * len(params), *params))


def _write_images(path, images):
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(images)))
        for iid, q, t, cid, name, xy, pid in images:
            fh.write(struct.pack("<idddddddi", iid, *q, *t, cid))
            fh.write(name.encode() + b"\x00")
            fh.write(struct.pack("<Q", len(pid)))
            for (x, y), p in zip(xy, pid):
                fh.write(struct.pack("<ddq", x, y, int(p)))


def set_camera_model(root, model_id):
    """rewrite dense/sparse/cameras.bin with every camera's model id replaced (e.g. 2 = SIMPLE_RADIAL, 4 parameters)"""
    from nrw import colmap

    path = os.path.join(root, "dense", "sparse", "cameras.bin")
    cams = colmap.read_cameras(path)
    _write_cameras(path, [(c.id, model_id, c.width, c.height, list(c.params)) for c in cams.values()])

