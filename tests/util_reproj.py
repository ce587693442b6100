"""Fixture writers and seeded scenes for the visibility-filter tests: COLMAP cameras.bin / images.bin, the scene *.tsv,
look-at cameras, triangle soups and the two-sphere scene."""
import os
import struct

import numpy as np


def write_cameras(path, cams):
    """cameras.bin (utils/colmap_utils.py::read_cameras_binary layout); cams: [(id, model id, width, height, params)]"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(cams)))
        for cid, mid, w, h, params in cams:
            fh.write(struct.pack("<iiQQ", cid, mid, w, h))
            fh.write(struct.pack("<" + "d" * len(params), *[float(p) for p in params]))


def write_images(path, images, seed=0):
    """images.bin (read_images_binary layout); images: [(id, qvec, tvec, camera id, name)], each with a few random
    2-D points"""
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(images)))
        for iid, q, t, cid, name in images:
            fh.write(struct.pack("<idddddddi", iid, *[float(x) for x in q], *[float(x) for x in t], cid))
            fh.write(name.encode("utf-8") + b"\x00")
            n = int(rng.integers(0, 4))
            fh.write(struct.pack("<Q", n))
            for _ in range(n):
                fh.write(struct.pack("<ddq", *rng.random(2) * 100, int(rng.integers(-1, 1000))))


def write_tsv(path, rows):
    """the scene's *.tsv: rows of (filename, id or '' for a missing id, split)"""
    with open(path, "w") as fh:
        fh.write("filename\tid\tsplit\tdataset\n")
        for name, id_, split in rows:
            fh.write(f"{name}\t{id_}\t{split}\tsynthetic\n")


def rotmat2qvec(R):
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


def look_at(eye, target, up=(0.0, 1.0, 0.0)):
    """world->camera rotation and translation (COLMAP axes: z forward, y down) of a camera at eye looking at target"""
    eye, target = np.asarray(eye, float), np.asarray(target, float)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, np.asarray(up, float))
    if np.linalg.norm(x) < 1e-9:
        x = np.cross(z, [1.0, 0.0, 0.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ eye


def view_matrix(R, t):
    V = np.eye(4)
    V[:3, :3], V[:3, 3] = R, t
    return V


def soup(rng, n, spread=1.0, depth=(0.5, 6.0)):
    """n independent triangles in front of, across and behind a camera at the origin looking down +z"""
    c = np.stack([rng.uniform(-spread, spread, n), rng.uniform(-spread, spread, n), rng.uniform(*depth, n)], 1)
    v = c[:, None, :] + rng.normal(0, 0.4, (n, 3, 3))
    return v.reshape(-1, 3), np.arange(3 * n).reshape(n, 3)


def sdf_spheres(centres, radii, lo, hi, h):
    """SDF volume (float32) of a union of spheres on the lattice lo + h * (i, j, k), and the lattice origin/spacing"""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    n = np.floor((hi - lo) / h).astype(int) + 1
    g = [lo[a] + h * np.arange(n[a]) for a in range(3)]
    X, Y, Z = np.meshgrid(*g, indexing="ij")
    d = np.full(X.shape, np.inf)
    for c, r in zip(centres, radii):
        d = np.minimum(d, np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r)
    return d.astype(np.float32), lo, h


# the end-to-end scene: sphere A (visible) at the origin, sphere B (hidden) behind it on the -z axis; the cameras sit
# within 3 degrees of the +z axis at distance 6, so A always covers B and every visible point of A has z > 0.1
SPHERE_A, RADIUS_A = (0.0, 0.0, 0.0), 1.0
SPHERE_B, RADIUS_B = (0.0, 0.0, -3.0), 0.4


def two_sphere_mesh(h=0.06):
    """marching_cubes (oracle/mc_port.py) of the two spheres: (vertices float64 [V,3] in the SfM frame, faces int64,
    sphere id of every vertex: 0 = A, 1 = B)"""
    from oracle import mc_port

    vol, lo, h = sdf_spheres([SPHERE_A, SPHERE_B], [RADIUS_A, RADIUS_B], (-1.3, -1.3, -3.6), (1.3, 1.3, 1.3), h)
    v, f, _ = mc_port.marching_cubes(vol)
    verts = lo + h * v.astype(np.float64)
    which = (verts[:, 2] < -1.5).astype(np.int64)
    return verts, f.astype(np.int64), which


def similarity(seed=0, scale=2.0):
    """a seeded 4x4 similarity sfm2gt = [s R | t]"""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    S = np.eye(4)
    S[:3, :3], S[:3, 3] = scale * R, rng.normal(size=3)
    return S


def write_scene(d, n_train=6, n_test=2, width=81, height=61, seed=0, scale=2.0):
    """data_path layout of the reference: dense/sparse/{cameras,images}.bin, scene.tsv (train and test rows and one
    row without id), config.yaml with a similarity sfm2gt.  Returns sfm2gt."""
    import yaml

    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(d, "dense", "sparse"), exist_ok=True)
    cams = [(1, 1, width, height, (100.3, 99.7, width / 2 - 0.35, height / 2 + 0.2)),
            (2, 1, width + 10, height - 6, (110.1, 110.1, (width + 10) / 2 + 0.4, (height - 6) / 2 - 0.3))]
    write_cameras(os.path.join(d, "dense", "sparse", "cameras.bin"), cams)
    images, rows = [], []
    for k in range(n_train + n_test + 1):
        th, ph = np.deg2rad(rng.uniform(0, 3)), rng.uniform(0, 2 * np.pi)
        eye = 6.0 * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        R, t = look_at(eye, SPHERE_A, up=(rng.normal(), 1.0, rng.normal() * 0.1))
        name = f"img_{k:03d}.jpg"
        images.append((10 + 3 * k, rotmat2qvec(R), t, 1 + k % 2, name))
        split = "train" if k < n_train or k == n_train + n_test else "test"     # the last row has no id
        rows.append((name, "" if k == n_train + n_test else 10 + 3 * k, split))
    write_images(os.path.join(d, "dense", "sparse", "images.bin"), images, seed)
    write_tsv(os.path.join(d, "scene.tsv"), rows)
    S = similarity(seed, scale)
    with open(os.path.join(d, "config.yaml"), "w") as fh:
        yaml.safe_dump({"sfm2gt": S.tolist(), "eval_bbx": [[-10.0, -10.0, -10.0], [10.0, 10.0, 10.0]]}, fh)
    return S
