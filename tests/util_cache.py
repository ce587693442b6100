"""Seeded synthetic Phototourism scene for the ray-cache tests: COLMAP binaries (PINHOLE and SIMPLE_RADIAL cameras,
keypoints that are noisy projections of points3D plus duplicates on one pixel, out-of-frame points and -1 ids), lossless
PNG images of odd sizes (one >= 1000 px wide), semantic maps, config.yaml and a tsv with one row missing from images.bin."""
import os
import struct

import numpy as np


def rot_to_qvec(R):
    w = np.sqrt(max(1e-12, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])


def qvec2rotmat(q):
    return np.array([
        [1 - 2 * q[2]**2 - 2 * q[3]**2, 2 * q[1] * q[2] - 2 * q[0] * q[3], 2 * q[3] * q[1] + 2 * q[0] * q[2]],
        [2 * q[1] * q[2] + 2 * q[0] * q[3], 1 - 2 * q[1]**2 - 2 * q[3]**2, 2 * q[2] * q[3] - 2 * q[0] * q[1]],
        [2 * q[3] * q[1] - 2 * q[0] * q[2], 2 * q[2] * q[3] + 2 * q[0] * q[1], 1 - 2 * q[1]**2 - 2 * q[2]**2]])


def look_at(C, rng):
    f = -C / np.linalg.norm(C)
    up = np.array([0, 0, 1.0]) + 0.1 * rng.standard_normal(3)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    R = np.stack([r, d, f], 0)                 # world -> camera rows: x right, y down, z forward
    q = rot_to_qvec(R)
    return q / np.linalg.norm(q)


SIZES = [(1001, 67), (81, 61), (95, 73), (63, 49), (77, 59), (91, 65), (69, 55), (85, 63), (73, 51), (99, 71), (65, 45),
         (87, 57)]


def write_scene(root, n_train=10, n_test=2, n_points=3000, seed=0, semantics=True):
    """Writes the scene under root (its basename is the scene name) and returns a dict describing it."""
    from PIL import Image

    rng = np.random.default_rng(seed)
    dense = os.path.join(root, "dense")
    sparse = os.path.join(dense, "sparse")
    os.makedirs(sparse, exist_ok=True)
    os.makedirs(os.path.join(dense, "images"), exist_ok=True)
    if semantics:
        os.makedirs(os.path.join(root, "semantic_maps"), exist_ok=True)
    n_img = n_train + n_test
    # points in a ball, ids with gaps
    xyz = rng.uniform(-1, 1, (n_points, 3)) * 0.9
    ids = np.arange(n_points, dtype=np.int64) * 2 + 1
    err = rng.uniform(0.2, 2.0, n_points)
    track = rng.integers(0, 6, n_points)
    cams, images = [], []
    for i in range(n_img):
        W, H = SIZES[i % len(SIZES)]
        f = 0.9 * W
        cid = i + 1
        if i % 2 == 0:
            cams.append((cid, 1, W, H, [f, f * 1.01, W / 2, H / 2]))      # PINHOLE
        else:
            cams.append((cid, 2, W, H, [f, W / 2, H / 2, 0.01]))          # SIMPLE_RADIAL
        ang = 2 * np.pi * i / n_img
        C = np.array([4 * np.cos(ang), 4 * np.sin(ang), 1.0 + 0.2 * rng.standard_normal()])
        q = look_at(C, rng)
        R = qvec2rotmat(q)
        t = -R @ C
        Xc = xyz @ R.T + t
        fx, fy = (f, f * 1.01) if i % 2 == 0 else (f, f)
        u = fx * Xc[:, 0] / Xc[:, 2] + W / 2
        v = fy * Xc[:, 1] / Xc[:, 2] + H / 2
        sel = np.nonzero((Xc[:, 2] > 0) & (u > -3) & (u < W + 3) & (v > -3) & (v < H + 3))[0]
        sel = rng.choice(sel, min(len(sel), 400), replace=False)
        xy = np.stack([u[sel], v[sel]], 1) + rng.normal(0, 0.3, (len(sel), 2))
        pid = ids[sel]
        # duplicates on one pixel, an out-of-frame keypoint, -1 ids
        dup = np.array([[xy[0, 0] + 0.1, xy[0, 1] - 0.1], [xy[1, 0], xy[1, 1]]])
        xy = np.concatenate([xy, dup, [[-50.0, 10.0], [W + 40.0, 5.0]], rng.uniform(0, W, (5, 2))], 0)
        pid = np.concatenate([pid, [ids[sel[5]], ids[sel[6]]], [ids[0], ids[1]], [-1] * 5])
        name = f"img_{i:03d}.png"
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        Image.fromarray(img).save(os.path.join(dense, "images", name))
        if semantics:
            sem = rng.integers(0, 20, (H, W)).astype(np.int32)
            np.savez(os.path.join(root, "semantic_maps", f"img_{i:03d}.npz"), sem)
        images.append((i + 10, q, t, cid, name, xy, pid))
    with open(os.path.join(sparse, "cameras.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", len(cams)))
        for cid, mid, W, H, params in cams:
            fh.write(struct.pack("<iiQQ", cid, mid, W, H))
            fh.write(struct.pack("<" + "d" * len(params), *params))
    with open(os.path.join(sparse, "images.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", len(images)))
        for iid, q, t, cid, name, xy, pid in images:
            fh.write(struct.pack("<idddddddi", iid, *q, *t, cid))
            fh.write(name.encode() + b"\x00")
            fh.write(struct.pack("<Q", len(pid)))
            for (x, y), p in zip(xy, pid):
                fh.write(struct.pack("<ddq", x, y, int(p)))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", n_points))
        for k in range(n_points):
            fh.write(struct.pack("<QdddBBBdQ", int(ids[k]), *xyz[k], 1, 2, 3, err[k], int(track[k])))
            for _ in range(int(track[k])):
                fh.write(struct.pack("<ii", 1, 0))
    with open(os.path.join(root, "config.yaml"), "w") as fh:
        fh.write("sfm2gt: [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]\n")
        fh.write("eval_bbx: [[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]]\n")
        fh.write("voxel_size: 0.1\nmin_track_length: 1\n")
    with open(os.path.join(root, os.path.basename(root) + ".tsv"), "w") as fh:
        fh.write("filename\tid\tsplit\tdataset\n")
        fh.write("missing.png\t-1\ttrain\tsynth\n")            # not in images.bin: must not shift the splits
        for k, (iid, _, _, _, name, _, _) in enumerate(images):
            fh.write(f"{name}\t{k}\t{'train' if k < n_train else 'test'}\tsynth\n")
    return {"root": root, "images": images, "n_train": n_train, "xyz": xyz, "ids": ids}
