"""COLMAP sparse-model readers (the slice of utils/colmap_utils.py the evaluation and the visibility filter need)."""
import collections
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


# model id -> (name, number of parameters), COLMAP's camera models
CAMERA_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}

Camera = collections.namedtuple("Camera", ["id", "model", "width", "height", "params"])


class Image(collections.namedtuple("Image", ["id", "qvec", "tvec", "camera_id", "name"])):
    """utils/colmap_utils.py::Image without the 2-D points (xys, point3D_ids)"""

    def qvec2rotmat(self):
        return qvec2rotmat(self.qvec)


def qvec2rotmat(qvec):
    """utils/colmap_utils.py::qvec2rotmat: rotation matrix of the quaternion (w, x, y, z), same expressions"""
    return np.array([
        [1 - 2 * qvec[2]**2 - 2 * qvec[3]**2,
         2 * qvec[1] * qvec[2] - 2 * qvec[0] * qvec[3],
         2 * qvec[3] * qvec[1] + 2 * qvec[0] * qvec[2]],
        [2 * qvec[1] * qvec[2] + 2 * qvec[0] * qvec[3],
         1 - 2 * qvec[1]**2 - 2 * qvec[3]**2,
         2 * qvec[2] * qvec[3] - 2 * qvec[0] * qvec[1]],
        [2 * qvec[3] * qvec[1] - 2 * qvec[0] * qvec[2],
         2 * qvec[2] * qvec[3] + 2 * qvec[0] * qvec[1],
         1 - 2 * qvec[1]**2 - 2 * qvec[2]**2]])


def read_cameras(path):
    """cameras.bin (utils/colmap_utils.py::read_cameras_binary layout, little endian): u64 count, then per camera i32 id,
    i32 model id, u64 width, u64 height and the model's f64 parameters.  Returns {id: Camera} in file order, params a
    float64 array."""
    with open(path, "rb") as fh:
        data = fh.read()
    try:
        n = struct.unpack_from("<Q", data, 0)[0]
        off, out = 8, {}
        for _ in range(n):
            cid, mid, w, h = struct.unpack_from("<iiQQ", data, off)
            off += 24
            if mid not in CAMERA_MODELS:
                raise NrwError(f"read_cameras: {path}: unknown camera model id {mid}")
            name, k = CAMERA_MODELS[mid]
            params = np.array(struct.unpack_from("<" + "d" * k, data, off))
            off += 8 * k
            out[cid] = Camera(id=cid, model=name, width=w, height=h, params=params)
    except struct.error as e:
        raise NrwError(f"read_cameras: {path} is truncated") from e
    return out


def read_images(path):
    """images.bin (utils/colmap_utils.py::read_images_binary layout, little endian): u64 count, then per image i32 id,
    4 f64 qvec, 3 f64 tvec, i32 camera id, a NUL-terminated UTF-8 name, u64 point count and that many (f64 x, f64 y,
    i64 point3D id) records, which are skipped.  Returns {id: Image} in file order."""
    with open(path, "rb") as fh:
        data = fh.read()
    try:
        n = struct.unpack_from("<Q", data, 0)[0]
        off, out = 8, {}
        for _ in range(n):
            r = struct.unpack_from("<idddddddi", data, off)
            off += 64
            end = data.index(b"\x00", off)
            name = data[off:end].decode("utf-8")
            off = end + 1
            npts = struct.unpack_from("<Q", data, off)[0]
            off += 8 + 24 * npts
            out[r[0]] = Image(id=r[0], qvec=np.array(r[1:5]), tvec=np.array(r[5:8]), camera_id=r[8], name=name)
    except (struct.error, ValueError) as e:
        raise NrwError(f"read_images: {path} is truncated") from e
    if off > len(data):
        raise NrwError(f"read_images: {path} is truncated")
    return out
