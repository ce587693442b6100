"""Visibility filtering of a reconstruction by the training cameras on the GPU: a drop-in for the mesh branch of
utils/reproj_filter.py (same names, flags and output file) that needs neither pyrender, an EGL context, trimesh, open3d
nor ray.

For every training view the source mesh is rasterised into a depth map (csrc/raster.cu: watertight fp64 edge
functions, pyrender's pixel-centre convention, back faces culled as pyrender's single-sided material does), every
covered pixel is back-projected from its integer pixel coordinate as the reference's `reproject` does, and the target
point nearest to it (exact fp64 search, csrc/nnsearch.cu) is kept when it lies closer than 2·√2·voxel_size.  The output
is the union over the views: the kept target points as rows [x, y, z, r, g, b] (colours in [0, 1]), unique and sorted as
np.unique(axis=0) returns them, written to <output_path>/reprojected.ply with double coordinates.

Deviations from the reference, by design: depth is fp64 (OpenGL has fp32 and a 24-bit depth buffer), nearest neighbours
are exact with the smallest index on ties, --visualize raises NrwError, and --n_cpus / --n_gpus are accepted and ignored
(one process; the union over views does not depend on the split).

With --point_source the source is a point cloud (its faces, if any, are ignored): the reference's Kaolin branch
(utils/kaolin_renderer.py).  The source points are voxelised into an octree (nrw.octree.gen_octree, expand 0, in the
frame of the points), every pixel of every training view casts one ray to the first leaf it hits (csrc/voxelvis.cu), and
a source point is kept when its leaf was hit by some view; the output rows are the target points of the kept source
indices, as for meshes.  Deviations of this branch are listed in INTEGRATION.md.

    python -m nrw.reprojection --src_file M.ply --target_file M.ply --data_path SCENE --output_path OUT [--point_source]
"""
import csv
import ctypes as C
import glob
import os

import numpy as np
import torch

from . import _lib
from ._lib import NrwError, check, ptr, stream_ptr
from .colmap import read_cameras, read_images
from .evaluation import NearestNeighbours, _device, _points, _scratch
from .mesh import read_ply, write_ply
from .octree import gen_octree, scene_bbox

# pyrender.constants DEFAULT_Z_NEAR / DEFAULT_Z_FAR, the clip range of its IntrinsicsCamera
Z_NEAR = 0.05
Z_FAR = 100.0

# pandas.read_csv's default missing-value strings (the reference drops rows whose `id` is missing)
_NA = {"", "#N/A", "#N/A N/A", "#NA", "-1.#IND", "-1.#QNAN", "-NaN", "-nan", "1.#IND", "1.#QNAN", "<NA>", "N/A", "NA", "NULL",
       "NaN", "None", "n/a", "nan", "null"}


def _host12(m, what):
    m = np.asarray(m, np.float64)
    if m.shape not in ((3, 4), (4, 4)):
        raise NrwError(f"{what}: expected a 3x4 or 4x4 matrix, got shape {m.shape}")
    return (C.c_double * 12)(*m[:3].reshape(-1).tolist())


def _pinhole(intrinsic):
    K = np.asarray(intrinsic)
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def get_image_id(imdata, data_dir):
    """utils/reproj_filter.py::get_image_id: (image ids, {id: name}, {name: id}) in images.bin order"""
    img_path_to_id = {}
    img_id_to_name = {}
    img_ids = []
    for v in imdata.values():
        img_path_to_id[v.name] = v.id
        img_id_to_name[v.id] = v.name
        img_ids += [v.id]
    return img_ids, img_id_to_name, img_path_to_id


def get_train_ids(data_path, img_ids_all, img_path_to_id):
    """utils/reproj_filter.py::get_train_ids: the ids of the rows of the scene's *.tsv (the first in sorted order) whose
    `split` is `train`, in file order, rows with a missing `id` dropped."""
    tsvs = sorted(glob.glob(os.path.join(data_path, "*.tsv")))
    if not tsvs:
        raise NrwError(f"get_train_ids: no *.tsv in {data_path}")
    with open(tsvs[0], newline="") as fh:
        rows = list(csv.DictReader(fh, delimiter="\t"))
    if rows and not all(k in rows[0] for k in ("filename", "id", "split")):
        raise NrwError(f"get_train_ids: {tsvs[0]} lacks one of the columns filename, id, split")
    img_ids = []
    for row in rows:
        if row["id"] is None or row["id"] in _NA:
            continue
        if row["filename"] not in img_path_to_id:
            raise NrwError(f"get_train_ids: {row['filename']} of {tsvs[0]} is not in images.bin")
        if row["split"] == "train":
            img_ids.append(img_path_to_id[row["filename"]])
    return img_ids


def get_entrinsics(imdata, img_ids):
    """tools/reproj_error.py::get_entrinsics: world->camera [N,4,4] float64 from qvec2rotmat and tvec"""
    entrinsics = np.zeros([len(img_ids), 4, 4])
    entrinsics[:, 3, 3] = 1
    for i, img_id in enumerate(img_ids):
        im = imdata[img_id]
        entrinsics[i, :3, :3] = im.qvec2rotmat()
        entrinsics[i, :3, 3] = im.tvec
    return entrinsics


def get_intrinsic(camdata, img_ids, imdata):
    """tools/reproj_error.py::get_intrinsic: ({id: K float32 [3,3]}, {id: (width, height)}).  Only PINHOLE cameras
    (params fx, fy, cx, cy) are accepted; the reference reads the first four parameters of any model."""
    Ks, whs = {}, {}
    for id_ in img_ids:
        cam = camdata[imdata[id_].camera_id]
        if cam.model != "PINHOLE":
            raise NrwError(f"get_intrinsic: camera {cam.id} of image {id_} is {cam.model}; only PINHOLE is supported")
        Ks[id_] = np.array([[cam.params[0], 0, cam.params[2]], [0, cam.params[1], cam.params[3]], [0, 0, 1]], dtype=np.float32)
        whs[id_] = cam.width, cam.height
    return Ks, whs


def reproject(height, width, depth, intrinsic, pose, valid_mask):
    """utils/reproj_filter.py::reproject with the device's arithmetic: the world points [n,3] float64 of the pixels of
    valid_mask in raster order, X = pose[:3] @ [((c - cx)/fx)·z, ((r - cy)/fy)·z, z, 1] from the integer pixel
    coordinate, each step rounded in this order (the reference inverts K in float32)."""
    depth = np.asarray(depth)
    r, c = np.nonzero(np.asarray(valid_mask).reshape(height, width))
    z = depth[r, c].astype(np.float64)
    fx, fy, cx, cy = _pinhole(intrinsic)
    xc, yc = ((c - cx) / fx) * z, ((r - cy) / fy) * z
    p = np.asarray(pose, np.float64)
    return np.stack([((p[k, 0] * xc + p[k, 1] * yc) + p[k, 2] * z) + p[k, 3] for k in range(3)], 1)


class DepthRenderer:
    """Depth maps of a triangle mesh (vertices [V,3], faces [F,3]) on its CUDA device; the mesh is uploaded once.
    __call__(height, width, intrinsic, world_to_cam) -> float32 [height, width] CUDA tensor: the camera z of the nearest
    front face (every face with cull_back=False) with znear <= z <= zfar, 0 elsewhere (rules in csrc/raster.cu).
    world_to_cam is a 3x4 or 4x4 COLMAP-convention matrix (z forward, y down) and may include a scale."""

    def __init__(self, vertices, faces, znear=Z_NEAR, zfar=Z_FAR, cull_back=True, device=None):
        self.v = _points(vertices, "DepthRenderer", None if device is None else _device(device))
        f = torch.as_tensor(faces)
        if f.dim() != 2 or f.shape[1] != 3 or f.dtype.is_floating_point or f.dtype == torch.bool:
            raise NrwError(f"DepthRenderer: faces must be an integer array [F, 3], got {tuple(f.shape)} {f.dtype}")
        if f.shape[0] == 0:
            raise NrwError("DepthRenderer: the source has no faces (point-cloud sources are not supported)")
        nv = self.v.shape[0]
        if nv == 0 or nv > 0x7FFFFFFF or f.shape[0] > 0x7FFFFFFF:
            raise NrwError(f"DepthRenderer: {nv} vertices, {f.shape[0]} faces (need 1 .. 2^31 - 1)")
        self.f = f.to(device=self.v.device, dtype=torch.int64).contiguous()
        if bool(((self.f < 0) | (self.f >= nv)).any()):
            raise NrwError(f"DepthRenderer: a face index lies outside [0, {nv})")
        self.znear, self.zfar, self.cull_back = float(znear), float(zfar), bool(cull_back)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.v.device)

    def __call__(self, height, width, intrinsic, world_to_cam):
        L = _lib.lib()
        height, width = int(height), int(width)
        fx, fy, cx, cy = _pinhole(intrinsic)
        depth = torch.empty(height, width, dtype=torch.float32, device=self.v.device)
        nb = L.nrw_raster_scratch_bytes(self.v.shape[0], self.f.shape[0], height, width)
        _, sp = _scratch(nb, self.v.device)
        with torch.cuda.device(self.v.device):
            check(L.nrw_raster_depth(ptr(self.v), self.v.shape[0], ptr(self.f), self.f.shape[0],
                                     _host12(world_to_cam, "DepthRenderer"), fx, fy, cx, cy, height, width, self.znear,
                                     self.zfar, int(self.cull_back), ptr(depth), ptr(self.status), sp, stream_ptr()),
                  "nrw_raster_depth")
        return depth


class VisibilityMarker:
    """The target points [n,3] indexed once; mark(depth, intrinsic, cam_to_world, threshold) sets `visible[i]` for the
    nearest target point i of every back-projected pixel closer than threshold.  Nothing is read back until
    `valid_pixels()` or `mask()`."""

    def __init__(self, target):
        self.nn = NearestNeighbours(target)
        self.visible = torch.zeros(self.nn.n, dtype=torch.uint8, device=self.nn.ref.device)
        self.n_valid = torch.zeros(1, dtype=torch.int64, device=self.nn.ref.device)

    def mark(self, depth, intrinsic, cam_to_world, threshold):
        L = _lib.lib()
        if depth.dim() != 2 or depth.dtype != torch.float32 or depth.device != self.nn.ref.device:
            raise NrwError("VisibilityMarker.mark: depth must be a float32 [H, W] tensor on the target's device")
        depth = depth.contiguous()
        h, w = depth.shape
        fx, fy, cx, cy = _pinhole(intrinsic)
        _, sp = _scratch(L.nrw_reproject_scratch_bytes(h, w), depth.device)
        with torch.cuda.device(depth.device):
            check(L.nrw_reproject_mark(ptr(depth), h, w, fx, fy, cx, cy, _host12(cam_to_world, "VisibilityMarker"),
                                       self.nn._ip, self.nn.n, float(threshold), ptr(self.visible), ptr(self.n_valid), sp,
                                       stream_ptr()), "nrw_reproject_mark")

    def valid_pixels(self):
        return int(self.n_valid.item())

    def mask(self):
        return self.visible.bool().cpu().numpy()


def reproj_filter(vertices, faces, target, intrinsics, extrinsics, whs, voxel_size=0.01, znear=Z_NEAR, zfar=Z_FAR,
                  cull_back=True, device=0):
    """The visibility mask (numpy bool [n_target]) of the target points: True where some view's back-projected depth
    pixel has the point as its nearest target point closer than 2·√2·voxel_size.  extrinsics [N,4,4] map the frame of
    `vertices` and `target` to each camera (reproj_filter.py's `extrinsics @ inv(sfm2gt)`), intrinsics [N,3,3], whs [N]
    (width, height).  Raises NrwError when no view has a covered pixel."""
    dev = _device(device)
    renderer = DepthRenderer(vertices, faces, znear, zfar, cull_back, device=dev)
    marker = VisibilityMarker(_points(target, "reproj_filter", dev))
    thr = 2 * np.sqrt(2) * voxel_size
    for K, E, (width, height) in zip(intrinsics, extrinsics, whs):
        pose = np.linalg.inv(E)
        depth = renderer(height, width, K, E)
        marker.mark(depth, K, pose, thr)
    if marker.valid_pixels() == 0:
        raise NrwError("reproj_filter: no view sees any face of the source mesh")
    return marker.mask()


class VoxelRenderer:
    """First-hit voxel renders of a point cloud [N,3] (utils/kaolin_renderer.py): the points are voxelised once with
    nrw.octree.gen_octree(scene_config, points, voxel_size, expand=0, in_sfm=False) on the CUDA device.
    __call__(height, width, intrinsic, world_to_cam) -> (depth float32 [H, W], leaf int32 [H, W]) CUDA tensors: per
    pixel the first leaf its ray hits (-1 on a miss) and the entry distance divided by the length of the ray's camera
    direction ((c - cx)/fx, (r - cy)/fy, 1), i.e. the camera z of a rigid camera (0 on a miss); every hit leaf is
    marked in `visible`, which accumulates over calls.  point_leaves() -> int32 [N] CUDA tensor: each input point's leaf, or -1
    for a point outside the octree's cube.  Rules in csrc/voxelvis.cu."""

    def __init__(self, points, scene_config, voxel_size, device=0):
        self.dev = _device(device)
        self.points = _points(points, "VoxelRenderer", self.dev)
        voxel_size = float(voxel_size)
        if not (np.isfinite(voxel_size) and voxel_size > 0):
            raise NrwError(f"VoxelRenderer: voxel_size = {voxel_size} (need finite, > 0)")
        bbx_min, bbx_max = scene_bbox(scene_config, in_sfm=False)
        scale = float(np.max(bbx_max - bbx_min)) / 2
        if not (np.isfinite(scale) and scale > 0):
            raise NrwError(f"VoxelRenderer: the scene's eval_bbx gives scale {scale} (need finite, > 0)")
        level = int(np.floor(np.log2(2 * scale / voxel_size)))       # gen_octree's rule
        if not 1 <= level <= 16:
            raise NrwError(f"VoxelRenderer: voxel_size {voxel_size} in a cube of half-size {scale} gives octree level "
                           f"{level} (need 1 .. 16)")
        self.tree, origin, self.scale, self.level = gen_octree(scene_config, self.points, voxel_size, device=self.dev,
                                                               expand=0, in_sfm=False)
        self.origin = np.asarray(origin, np.float64)
        pyr = self.tree["pyramid"].to(torch.int32).contiguous()
        self.n_leaf = int(pyr[0, self.level])
        if self.n_leaf == 0:
            raise NrwError("VoxelRenderer: no source point lies inside the scene's cube (eval_bbx)")
        self._pyr = (C.c_int * pyr.numel())(*pyr.reshape(-1).tolist())
        self._origin = (C.c_float * 3)(*self.origin.tolist())
        self.visible = torch.zeros(self.n_leaf, dtype=torch.uint8, device=self.dev)
        self.n_hit = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.dev)

    def cast(self, height, width, intrinsic, world_to_cam, depth=None, leaf=None):
        """one view into the given outputs (each may be None); marks `visible` and counts hit pixels in `n_hit`"""
        L = _lib.lib()
        E = np.asarray(world_to_cam, np.float64)
        if E.shape == (3, 4):
            E = np.concatenate([E, [[0.0, 0.0, 0.0, 1.0]]])
        c2w = np.linalg.inv(E)
        fx, fy, cx, cy = _pinhole(intrinsic)
        with torch.cuda.device(self.dev):
            check(L.nrw_voxel_cast(ptr(self.tree["octree"]), ptr(self.tree["prefix"]), self._pyr, self.level, self._origin,
                                   self.scale, _host12(c2w, "VoxelRenderer"), fx, fy, cx, cy, int(height), int(width),
                                   ptr(self.visible), ptr(depth), ptr(leaf), ptr(self.n_hit), stream_ptr()),
                  "nrw_voxel_cast")

    def __call__(self, height, width, intrinsic, world_to_cam):
        height, width = int(height), int(width)
        if height < 1 or width < 1:
            raise NrwError(f"VoxelRenderer: image {height} x {width}")
        depth = torch.empty(height, width, dtype=torch.float32, device=self.dev)
        leaf = torch.empty(height, width, dtype=torch.int32, device=self.dev)
        self.cast(height, width, intrinsic, world_to_cam, depth, leaf)
        return depth, leaf

    def point_leaves(self):
        """each input point's leaf index (int32 CUDA tensor), -1 outside the open cube; points normalised by the
        expression of gen_octree"""
        L = _lib.lib()
        pn = ((self.points - torch.as_tensor(self.origin, device=self.dev)) / self.scale).contiguous()
        leaf = torch.empty(pn.shape[0], dtype=torch.int32, device=self.dev)
        with torch.cuda.device(self.dev):
            check(L.nrw_voxel_lookup(ptr(self.tree["octree"]), ptr(self.tree["prefix"]), self._pyr, self.level, ptr(pn),
                                     pn.shape[0], ptr(leaf), ptr(self.status), stream_ptr()), "nrw_voxel_lookup")
        return leaf


def reproj_filter_points(points, scene_config, intrinsics, extrinsics, whs, voxel_size=0.01, device=0):
    """The visibility mask (numpy bool [n_points]) of a point cloud: True where the point's leaf voxel (octree of the
    points themselves, gen_octree with expand 0 in their own frame) is the first leaf hit by some pixel's ray of some
    view.  extrinsics [N,4,4] map the frame of `points` to each camera, intrinsics [N,3,3], whs [N] (width, height).
    Reads back once, at the end.  Raises NrwError when no view hits any voxel."""
    r = VoxelRenderer(points, scene_config, voxel_size, device=device)
    for K, E, (width, height) in zip(intrinsics, extrinsics, whs):
        r.cast(int(height), int(width), K, E)
    leaf = r.point_leaves().long()
    keep = (leaf >= 0) & (r.visible[leaf.clamp(min=0)] != 0)
    host = torch.cat([r.n_hit, r.status.long(), keep.long()]).cpu().numpy()
    if host[1]:
        raise NrwError("reproj_filter_points: a source point's cell is not a leaf of its own octree")
    if host[0] == 0:
        raise NrwError("reproj_filter_points: no view hits any voxel of the source points")
    return host[2:].astype(bool)


def _scene_config(data_path):
    import yaml

    with open(os.path.join(data_path, "config.yaml"), "r") as fh:
        return yaml.load(fh, Loader=yaml.FullLoader)


def _sfm2gt(data_path):
    return np.array(_scene_config(data_path)["sfm2gt"])


def _to_gt(pts, sfm_to_gt):
    """utils/reproj_filter.py::sfm2gt"""
    homo = np.concatenate((pts, np.ones((pts.shape[0], 1))), axis=-1).T
    return (sfm_to_gt[:3] @ homo).T


def get_opts(argv=None):
    """utils/reproj_filter.py::parse_args (same flags and defaults)"""
    import argparse

    parser = argparse.ArgumentParser(prog="python -m nrw.reprojection")
    parser.add_argument('--src_file', type=str, required=True, help='mesh file path')
    parser.add_argument('--target_file', type=str, required=True, help='point cloud to be filtered')
    parser.add_argument('--data_path', type=str, required=True, help='camera poses in colmap format')
    parser.add_argument('--output_path', type=str, required=True, help='output path')
    parser.add_argument('--gt', default=False, action="store_true", help='whether target pc/mesh is in gt coordinates system')
    parser.add_argument('--visualize', default=False, action="store_true", help='whether to store render results')
    parser.add_argument('--voxel_size', type=float, default=0.01, help='voxel size in world coordinate system')
    parser.add_argument('--n_cpus', type=int, default=1, help='accepted and ignored (one process)')
    parser.add_argument('--n_gpus', type=int, default=4, help='accepted and ignored (every view on one device)')
    parser.add_argument('--point_source', default=False, action="store_true",
                        help='the source is a point cloud: filter it through its voxel octree (faces are ignored)')
    return parser.parse_args(argv)


def main(argv=None):
    args = get_opts(argv)
    if args.visualize:
        raise NrwError("--visualize is not supported (its images need matplotlib's colormap and cv2)")
    print(f"result will be saved to {args.output_path}")
    os.makedirs(args.output_path, exist_ok=True)
    sparse = os.path.join(args.data_path, "dense", "sparse")
    imdata = read_images(os.path.join(sparse, "images.bin"))
    camdata = read_cameras(os.path.join(sparse, "cameras.bin"))
    _, _, img_path_to_id = get_image_id(imdata, args.data_path)
    img_ids = get_train_ids(args.data_path, None, img_path_to_id)
    print(f"views to process: {len(img_ids)}")
    if not img_ids:
        raise NrwError(f"reproj_filter: no training view in the *.tsv of {args.data_path}")
    intrinsics, whs = get_intrinsic(camdata, img_ids, imdata)
    sfm_to_gt = _sfm2gt(args.data_path)
    extrinsics = get_entrinsics(imdata, img_ids) @ np.linalg.inv(sfm_to_gt)

    src = read_ply(args.src_file)
    if src["faces"].shape[0] == 0 and not args.point_source:
        raise NrwError(f"{args.src_file} has no faces: point-cloud sources need --point_source")
    verts = np.asarray(src["vertices"], np.float64)
    tgt = read_ply(args.target_file)
    points = np.asarray(tgt["vertices"], np.float64)
    colors = np.zeros_like(points) if tgt["colors"] is None else tgt["colors"].astype(np.float64) / 255.0
    if args.point_source and points.shape[0] != verts.shape[0]:
        raise NrwError(f"--point_source: the target has {points.shape[0]} points and the source {verts.shape[0]}; the "
                       "kept source indices select target points, so the counts must be equal")
    if not args.gt:
        verts, points = _to_gt(verts, sfm_to_gt), _to_gt(points, sfm_to_gt)
    if not np.isfinite(verts).all():
        raise NrwError(f"{args.src_file}: vertices are not all finite")

    Ks, Ws = [intrinsics[k] for k in img_ids], [whs[k] for k in img_ids]
    if args.point_source:
        mask = reproj_filter_points(verts, _scene_config(args.data_path), Ks, extrinsics, Ws, voxel_size=args.voxel_size)
    else:
        mask = reproj_filter(verts, src["faces"], points, Ks, extrinsics, Ws, voxel_size=args.voxel_size)
    rows = np.unique(np.hstack([points[mask], colors[mask]]), axis=0)
    out = os.path.join(args.output_path, "reprojected.ply")
    write_ply(out, rows[:, :3], colors=np.round(rows[:, 3:] * 255.0).astype(np.uint8), double=True)
    print(f"kept {rows.shape[0]} of {points.shape[0]} points -> {out}")
    return rows


if __name__ == "__main__":
    main()
