"""COLMAP sparse-model reader (the slice of utils/colmap_utils.py the evaluation needs)."""
import struct

import numpy as np

from ._lib import NrwError


def read_points3d(path):
    """points3D.bin (utils/colmap_utils.py::read_points3d_binary layout, little endian): per point u64 id, 3 f64 xyz,
    3 u8 rgb, f64 error, u64 track length, then track length (i32 image id, i32 point2D index) pairs.  Returns a dict of
    numpy arrays in file order: id uint64 [n], xyz float64 [n,3], rgb uint8 [n,3], error float64 [n], track_length
    int64 [n]."""
    with open(path, "rb") as fh:
        data = fh.read()
    if len(data) < 8:
        raise NrwError(f"read_points3d: {path} is shorter than its header")
    n = struct.unpack_from("<Q", data, 0)[0]
    rec = struct.Struct("<QdddBBBdQ")
    ids = np.empty(n, np.uint64)
    xyz = np.empty((n, 3), np.float64)
    rgb = np.empty((n, 3), np.uint8)
    err = np.empty(n, np.float64)
    tl = np.empty(n, np.int64)
    off = 8
    try:
        for i in range(n):
            r = rec.unpack_from(data, off)
            ids[i], xyz[i], rgb[i], err[i], tl[i] = r[0], r[1:4], r[4:7], r[7], r[8]
            off += rec.size + 8 * r[8]
    except struct.error as e:
        raise NrwError(f"read_points3d: {path} is truncated") from e
    if off > len(data):
        raise NrwError(f"read_points3d: {path} is truncated")
    return {"id": ids, "xyz": xyz, "rgb": rgb, "error": err, "track_length": tl}
