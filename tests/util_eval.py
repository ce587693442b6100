"""Fixture writers shared by the evaluation tests: COLMAP points3D.bin and seeded scenes."""
import struct

import numpy as np


def write_points3d(path, xyz, error, track_length, seed=0):
    """points3D.bin in COLMAP's binary layout (utils/colmap_utils.py::read_points3d_binary)"""
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<Q", len(xyz)))
        for i, (p, e, t) in enumerate(zip(xyz, error, track_length)):
            fh.write(struct.pack("<QdddBBBd", 1000 + 3 * i, *[float(x) for x in p], *[int(c) for c in rng.integers(0, 256, 3)],
                                 float(e)))
            fh.write(struct.pack("<Q", int(t)))
            fh.write(rng.integers(0, 5000, 2 * int(t)).astype("<i4").tobytes())


def sfm_points(rng, n, lo, hi, margin=0.2):
    """n SfM points, some outside [lo, hi], with errors in [0, 3) and track lengths in [0, 30)"""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    ext = hi - lo
    xyz = lo - margin * ext + rng.random((n, 3)) * (1 + 2 * margin) * ext
    return xyz, rng.random(n) * 3.0, rng.integers(0, 30, n)


def surface_scene(rng, n_gt, n_pred, lo, hi, noise=0.01, outliers=0.01):
    """ground truth on a wavy surface z = f(x, y) inside [lo, hi], a noisy prediction of it with a share of outliers;
    float32-representable float64 coordinates (so float32 PLY files hold them exactly)"""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)

    def surf(n):
        xy = lo[:2] + rng.random((n, 2)) * (hi[:2] - lo[:2])
        z = (lo[2] + hi[2]) / 2 + 0.2 * (hi[2] - lo[2]) * np.sin(xy[:, 0] * 3) * np.cos(xy[:, 1] * 2)
        return np.concatenate([xy, z[:, None]], 1)

    gt = surf(n_gt)
    pred = surf(n_pred) + rng.normal(0, noise, (n_pred, 3))
    k = int(outliers * n_pred)
    pred[:k] = lo + rng.random((k, 3)) * 1.4 * (hi - lo) - 0.2 * (hi - lo)
    return gt.astype(np.float32).astype(np.float64), pred.astype(np.float32).astype(np.float64)
