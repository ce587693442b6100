"""Training ray-cache generation on the GPU: the scene reader, the per-image driver and a drop-in PhototourismDataset
(datasets/phototourism.py) that needs neither Kaolin, open3d, kornia, h5py nor cv2.

    read_scene        read_meta steps 1-4: tsv, images.bin / cameras.bin / points3D.bin, K, c2w, near/far bounds
    RayGenerator      one image -> the reference's cache rows and rgbs (csrc/raygen.cu, rules in its header)
    PhototourismDataset  the reference's constructor, __len__ and __getitem__ for "train" and "val" / "test_train"

Images are decoded and LANCZOS-downscaled by PIL on the host (as the reference does) by a small thread pool that runs
ahead of the device.  Deviations from the reference are listed in INTEGRATION.md.
"""
import collections
import concurrent.futures
import csv
import ctypes
import glob
import os
import warnings

import numpy as np
import torch

from . import _lib, colmap
from ._lib import NrwError, check, ptr, stream_ptr

# scene name -> (sfm_path, depth_percent), datasets/phototourism.py:82-90; other scenes use ("sparse", 0)
SCENE_DEFAULTS = {"brandenburg_gate": ("../neuralsfm", 0.2), "palacio_de_bellas_artes": ("../neuralsfm", 0.4),
                  "lincoln_memorial": ("sparse", 0.0), "pantheon_exterior": ("sparse", 0.0)}


def scene_defaults(root_dir):
    return SCENE_DEFAULTS.get(os.path.basename(os.path.normpath(root_dir)), ("sparse", 0.0))


def _scratch(nbytes, device, what):
    if nbytes < 0:
        check(int(nbytes), what)
    buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
    return buf, ctypes.c_void_p((buf.data_ptr() + 255) // 256 * 256)


def read_config(root_dir):
    import yaml

    path = os.path.join(root_dir, "config.yaml")
    if not os.path.isfile(path):
        raise NrwError(f"read_scene: {path} not found")
    with open(path, "r") as f:
        return yaml.load(f, Loader=yaml.FullLoader)


def read_tsv(root_dir):
    """[(filename, split)] in file order of the scene's *.tsv (datasets/phototourism.py:319-321)."""
    tsvs = sorted(glob.glob(os.path.join(root_dir, "*.tsv")))
    if not tsvs:
        raise NrwError(f"read_scene: no *.tsv in {root_dir}")
    with open(tsvs[0], newline="") as f:
        rows = list(csv.DictReader(f, delimiter="\t"))
    if rows and ("filename" not in rows[0] or "split" not in rows[0]):
        raise NrwError(f"read_scene: {tsvs[0]} has no filename / split columns")
    return [(r["filename"], r["split"]) for r in rows]


def intrinsics(cam, img_downscale):
    """read_meta step 2: fp32 K of the downscaled image (PINHOLE and SIMPLE_RADIAL only)."""
    K = np.zeros((3, 3), dtype=np.float32)
    p = cam.params
    if cam.model == "PINHOLE":
        fx, fy, cx, cy = p[0], p[1], p[2], p[3]
    elif cam.model == "SIMPLE_RADIAL":
        fx, fy, cx, cy = p[0], p[0], p[1], p[2]
    else:
        raise NrwError(f"read_scene: camera model {cam.model} is not supported (PINHOLE, SIMPLE_RADIAL)")
    img_w, img_h = int(cx * 2), int(cy * 2)
    w_, h_ = img_w // img_downscale, img_h // img_downscale
    K[0, 0] = fx * w_ / img_w
    K[1, 1] = fy * h_ / img_h
    K[0, 2] = cx * w_ / img_w
    K[1, 2] = cy * h_ / img_h
    K[2, 2] = 1
    return K


def camera_poses(images, who):
    """read_meta step 3: (w2c f64 [n, 4, 4], c2w f64 [n, 3, 4]) of COLMAP images, c2w = inv(w2c)[:, :3] in fp64 with
    columns 1:2 negated ("right down front" -> "right up back"); the kernels take its fp32 rounding."""
    bottom = np.array([0, 0, 0, 1.0]).reshape(1, 4)
    w2c = np.stack([np.concatenate([np.concatenate([im.qvec2rotmat(), im.tvec.reshape(3, 1)], 1), bottom], 0) for im in images], 0)
    if not np.isfinite(w2c).all():
        raise NrwError(f"{who}: non-finite camera pose in images.bin")
    poses = np.linalg.inv(w2c)[:, :3]
    poses[..., 1:3] *= -1
    if not np.isfinite(poses).all():
        raise NrwError(f"{who}: singular camera pose in images.bin")
    return w2c, poses


Scene = collections.namedtuple("Scene", ["root_dir", "sfm_path", "img_downscale", "img_ids", "image_paths", "splits", "Ks",
                                         "w2c", "poses", "imdata", "xyz_world", "table_xyz", "table_err", "config"])


def read_scene(root_dir, img_downscale=1, sfm_path="sparse"):
    """read_meta steps 1-3 and the point table of the keypoint depth.  Each image's split is read from its own tsv row."""
    if img_downscale < 1:
        raise NrwError("read_scene: img_downscale must be >= 1")
    rows = read_tsv(root_dir)
    base = os.path.join(root_dir, "dense", sfm_path)
    for f in ("images.bin", "cameras.bin", "points3D.bin"):
        if not os.path.isfile(os.path.join(base, f)):
            raise NrwError(f"read_scene: {os.path.join(base, f)} not found")
    imdata = colmap.read_images(os.path.join(base, "images.bin"), with_points=True)
    cams = colmap.read_cameras(os.path.join(base, "cameras.bin"))
    by_name = {v[0].name: k for k, v in imdata.items()}
    img_ids, image_paths, splits = [], {}, {}
    for filename, split in rows:
        if filename not in by_name:
            warnings.warn(f"image {filename} not found in the SfM result")
            continue
        id_ = by_name[filename]
        image_paths[id_] = filename
        splits[id_] = split
        img_ids.append(id_)
    if not img_ids:
        raise NrwError("read_scene: no tsv image is in images.bin")
    Ks = {id_: intrinsics(cams[imdata[id_][0].camera_id], img_downscale) for id_ in img_ids}
    w2c, poses = camera_poses([imdata[i][0] for i in img_ids], "read_scene")
    pts = colmap.read_points3d(os.path.join(base, "points3D.bin"))
    n_table = int(pts["id"].max()) + 1 if len(pts["id"]) else 1
    table_xyz = np.ones((n_table, 3), np.float64)      # ids absent from points3D.bin read as the reference's ones
    table_err = np.ones(n_table, np.float64)
    table_xyz[pts["id"].astype(np.int64)] = pts["xyz"]
    table_err[pts["id"].astype(np.int64)] = pts["error"]
    return Scene(root_dir, sfm_path, img_downscale, img_ids, image_paths, splits, Ks, w2c, poses,
                 {i: imdata[i] for i in img_ids}, pts["xyz"], table_xyz, table_err, read_config(root_dir))


def depth_bounds(xyz, w2c, device, scene_origin=None, scene_radius=None, q=(0.1, 99.9)):
    """read_meta step 4: per-image (near, far) as float64 [n_img, 2].  np.percentile of the camera z of the points in
    front (linear method) on the device, or origin_z -/+ 1.5 * radius with a scene origin.  Raises when an image sees no
    point in front of it."""
    w2c = np.asarray(w2c, np.float64)
    if scene_origin is not None:
        oh = np.concatenate([np.asarray(scene_origin, np.float64), np.ones(1)], -1)[np.newaxis, :]
        z = np.array([(oh @ w.T)[0, 2] for w in w2c])
        return np.stack([z - scene_radius * 1.5, z + scene_radius * 1.5], 1)
    n = len(xyz)
    if n == 0:
        raise NrwError("depth_bounds: no SfM points")
    L = _lib.lib()
    X = torch.from_numpy(np.ascontiguousarray(xyz, np.float64)).to(device)
    out = torch.empty((len(w2c), 2), dtype=torch.float64, device=device)
    status = torch.zeros(1, dtype=torch.int32, device=device)
    per = max(1, min(len(w2c), (1 << 26) // n))          # images per call: keeps the sort under ~1 GB of keys
    for i0 in range(0, len(w2c), per):
        m = min(per, len(w2c) - i0)
        W = torch.from_numpy(np.ascontiguousarray(w2c[i0:i0 + m, :3, :])).to(device)
        _buf, sp = _scratch(L.nrw_depth_range_scratch_bytes(n, m), device, "nrw_depth_range_scratch_bytes")
        check(L.nrw_depth_range(ptr(X), n, ptr(W), m, q[0], q[1], ptr(out[i0:]), None, ptr(status), sp, stream_ptr()),
              "nrw_depth_range")
        if int(status.item()) & 1:
            raise NrwError("depth_bounds: an image has no SfM point in front of it")
    return out.cpu().numpy()


def build_octrees(root_dir, config, device):
    """The two octrees of PhototourismDataset.get_octree (expand 1 radius 1, expand 2 radius 1.5) from
    dense/sparse/points3D.bin points with track_length > min_track_length (gen_octree_from_sfm keeps its own "sparse")."""
    from .octree import gen_octree

    path = os.path.join(root_dir, "dense", "sparse", "points3D.bin")
    if not os.path.isfile(path):
        raise NrwError(f"build_octrees: {path} not found")
    pts = colmap.read_points3d(path)
    sel = pts["xyz"][pts["track_length"] > config["min_track_length"]]
    out = []
    for expand, radius in ((1, 1.0), (2, 1.5)):
        tree, origin, scale, level = gen_octree(config, sel, config["voxel_size"], device=device, expand=expand, radius=radius)
        out.append((tree, np.asarray(origin, np.float64).astype(np.float32), float(scale), int(level)))
    return out


def load_image(path, img_downscale):
    """PIL decode + LANCZOS downscale (read_meta :542-551) -> uint8 [h, w, 3]."""
    from PIL import Image

    img = Image.open(path).convert("RGB")
    w, h = img.size
    if img_downscale > 1:
        img = img.resize((w // img_downscale, h // img_downscale), Image.LANCZOS)
    return np.array(img, dtype=np.uint8)


def load_semantics(root_dir, semantic_map_path, image_name):
    path = os.path.join(root_dir, f"{semantic_map_path}/{image_name}.npz")
    if not os.path.isfile(path):
        raise NrwError(f"semantic map {path} not found")
    return np.ascontiguousarray(np.load(path)["arr_0"], dtype=np.float32)


class RayGenerator:
    """One image -> (rows f32 [T, 12 or 11], rgbs f32 [T, 3]) on the device through nrw_raygen_image."""

    def __init__(self, scene, device, with_semantics, semantic_map_path=None, use_voxel=True, depth_percent=0.0, seed=0,
                 bounds=None, octrees=None):
        self.scene, self.device = scene, torch.device(device)
        self.with_semantics, self.semantic_map_path = with_semantics, semantic_map_path
        self.use_voxel, self.depth_percent, self.seed = use_voxel, float(depth_percent), int(seed)
        if not 0.0 <= self.depth_percent < 1.0:
            raise NrwError(f"depth_percent must lie in [0, 1) (got {depth_percent})")
        self.bounds = bounds
        self.octrees = octrees if octrees is not None or not use_voxel else build_octrees(scene.root_dir, scene.config, self.device)
        self.table_xyz = torch.from_numpy(scene.table_xyz).to(self.device)
        self.table_err = torch.from_numpy(scene.table_err).to(self.device)
        self.counts = torch.zeros(4, dtype=torch.int64, device=self.device)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)

    def decode(self, id_):
        """host half: the image (and semantic map) of id_ as pinned tensors"""
        s = self.scene
        img = load_image(os.path.join(s.root_dir, "dense/images", s.image_paths[id_]), s.img_downscale)
        sem = None
        if self.with_semantics:
            sem = load_semantics(s.root_dir, self.semantic_map_path, s.image_paths[id_].split(".")[0])
            sem = torch.from_numpy(sem).pin_memory()
        return torch.from_numpy(img).pin_memory(), sem

    def cfg(self, id_, h, w, sem_shape):
        s = self.scene
        g = _lib.RaygenCfg()
        g.height, g.width, g.img_downscale = h, w, s.img_downscale
        K = s.Ks[id_]
        g.fx, g.fy, g.cx, g.cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        i = s.img_ids.index(id_)
        g.c2w[:] = [float(v) for v in s.poses[i].astype(np.float32).reshape(-1)]
        g.w2c_z[:] = [float(v) for v in s.w2c[i, 2, :4]]
        g.image_id = int(id_)
        g.with_label = 1 if sem_shape is not None else 0
        if sem_shape is not None:
            g.sem_height, g.sem_width = sem_shape
        g.use_voxel = 1 if self.use_voxel else 0
        if self.bounds is not None:
            g.near, g.far = float(np.float32(self.bounds[i, 0])), float(np.float32(self.bounds[i, 1]))
        g.voxel_size = float(s.config.get("voxel_size", 0.0)) if self.use_voxel else 0.0
        if self.use_voxel:
            for ref, (tree, origin, scale, level) in zip((g.sfm, g.expanded), self.octrees):
                ref.octree, ref.prefix, ref.level = tree["octree"].data_ptr(), tree["prefix"].data_ptr(), level
                ref.scene_origin[:] = [float(v) for v in origin]
                ref.scale = scale
        g.depth_percent = self.depth_percent
        g.seed = self.seed
        return g

    def run(self, id_, img, sem):
        """device half: (rows, rgbs) CUDA tensors of image id_ from its decoded uint8 image and semantic map"""
        L, dev, s = _lib.lib(), self.device, self.scene
        h, w = int(img.shape[0]), int(img.shape[1])
        im, xys, ids = s.imdata[id_]
        g = self.cfg(id_, h, w, None if sem is None else tuple(sem.shape))
        cap = int(L.nrw_raygen_capacity(h, w, self.depth_percent))
        if cap < 0:
            check(cap, "nrw_raygen_capacity")
        C = 12 if sem is not None else 11
        nk = len(ids)
        _buf, sp = _scratch(L.nrw_raygen_scratch_bytes(h, w, g.with_label, nk, cap), dev, "nrw_raygen_scratch_bytes")
        rgb8 = img.to(dev, non_blocking=True)
        semd = None if sem is None else sem.to(dev, non_blocking=True)
        xy = torch.from_numpy(np.ascontiguousarray(xys)).to(dev) if nk else None
        pid = torch.from_numpy(np.ascontiguousarray(ids)).to(dev) if nk else None
        rows = torch.empty((cap, C), dtype=torch.float32, device=dev)
        rgbs = torch.empty((cap, 3), dtype=torch.float32, device=dev)
        check(L.nrw_raygen_image(ctypes.byref(g), ptr(rgb8), ptr(semd), ptr(xy), ptr(pid), nk, ptr(self.table_xyz), ptr(self.table_err),
                                 len(s.table_err), ptr(rows), ptr(rgbs), cap, ptr(self.counts), ptr(self.status), sp,
                                 stream_ptr()), "nrw_raygen_image")
        counts = self.counts.cpu()                    # the one read-back: sizes the copy-out
        st = int(self.status.item())
        if st & 1:
            raise NrwError(f"image {id_}: a keypoint's point3D id is past the points3D table")
        if st & 2:
            raise NrwError(f"image {id_}: padding rows exceed the output capacity")
        t = int(counts[0])
        return rows[:t], rgbs[:t], [int(v) for v in counts]

    def images(self, img_ids, workers=4, ahead=4):
        """yields (id_, rows, rgbs, counts) in order; PIL decodes up to `ahead` images while the device works"""
        with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
            futs = collections.deque()
            it = iter(img_ids)
            for id_ in it:
                futs.append((id_, pool.submit(self.decode, id_)))
                if len(futs) >= ahead:
                    break
            while futs:
                id_, f = futs.popleft()
                nxt = next(it, None)
                if nxt is not None:
                    futs.append((nxt, pool.submit(self.decode, nxt)))
                img, sem = f.result()
                yield (id_,) + self.run(id_, img, sem)


class PhototourismDataset(torch.utils.data.Dataset):
    """datasets/phototourism.py::PhototourismDataset for split "train" (use_cache or in-memory generation) and
    "val" / "test_train" (one image generated on the fly).  "eval", "test" and shared_cache raise NrwError."""

    def __init__(self, root_dir, split="train", img_downscale=1, val_num=1, use_cache=False, cache_paths=["cache"],
                 split_path="", semantic_map_path=None, with_semantics=True, use_voxel=True, scene_origin=None,
                 scene_radius=None, shared_cache=False, shared_rays_base=None, shared_rgbs_base=None, all_rays_shape=None,
                 all_rgbs_shape=None, device=0, sfm_path=None, depth_percent=None, seed=0):
        if split not in ("train", "val", "test_train"):
            raise NrwError(f"PhototourismDataset: split {split!r} is not supported (train, val, test_train)")
        if shared_cache:
            raise NrwError("PhototourismDataset: shared_cache is not supported")
        if img_downscale < 1:
            raise NrwError("image can only be downsampled, please set img_downscale>=1!")
        if use_cache and split != "train":
            raise NrwError("only can use cache during training")
        self.root_dir, self.split, self.split_path = root_dir, split, split_path
        self.img_downscale = max(8, img_downscale) if split == "val" else img_downscale
        self.val_num = max(1, val_num)
        self.semantic_map_path, self.with_semantics = semantic_map_path, with_semantics
        self.scene_origin, self.scene_radius = scene_origin, scene_radius
        d_sfm, d_pct = scene_defaults(root_dir)
        self.sfm_path = d_sfm if sfm_path is None else sfm_path
        self.depth_percent = d_pct if depth_percent is None else depth_percent
        self.use_cache, self.use_voxel, self.cache_paths = use_cache, use_voxel, cache_paths
        self.white_back = False
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if use_cache:
            from .raycache import load_split_arrays

            rays, rgbs = load_split_arrays(root_dir, split_path, list(cache_paths), self.img_downscale)
            self.all_rays, self.all_rgbs = torch.from_numpy(rays), torch.from_numpy(rgbs)
            return
        s = read_scene(root_dir, self.img_downscale, self.sfm_path)
        self.scene = s
        self.img_ids, self.image_paths, self.Ks = s.img_ids, s.image_paths, s.Ks
        self.poses_dict = {id_: s.poses[i] for i, id_ in enumerate(s.img_ids)}
        b = depth_bounds(s.xyz_world, s.w2c, self.device, scene_origin, scene_radius)
        self.nears = {id_: b[i, 0] for i, id_ in enumerate(s.img_ids)}
        self.fars = {id_: b[i, 1] for i, id_ in enumerate(s.img_ids)}
        self.img_ids_train = [i for i in s.img_ids if s.splits[i] != "test"]
        self.img_ids_test = [i for i in s.img_ids if s.splits[i] == "test"]
        self.N_images_train, self.N_images_test = len(self.img_ids_train), len(self.img_ids_test)
        voxel = split == "train" and use_voxel
        self.gen = RayGenerator(s, self.device, with_semantics, semantic_map_path, use_voxel=voxel,
                                depth_percent=self.depth_percent if split == "train" else 0.0, seed=seed, bounds=b)
        if split == "train":
            self.all_rays, self.all_rgbs, n_miss = [], [], 0
            for id_, rows, rgbs, counts in self.gen.images(self.img_ids_train):
                n_miss += counts[1] == 0
                self.all_rays.append(rows.cpu())
                self.all_rgbs.append(rgbs.cpu())
            check_voxel_misses(n_miss, len(self.img_ids_train))
        else:
            self.val_id = self.img_ids_train[0]

    def __len__(self):
        if self.split == "train":
            return len(self.all_rays)
        if self.split == "test_train":
            return self.N_images_train
        return self.val_num

    def __getitem__(self, idx):
        if self.split == "train":
            sample = {"rays": self.all_rays[idx, :8], "ts": self.all_rays[idx, 8].long(), "rgbs": self.all_rgbs[idx]}
            if self.with_semantics:
                sample["semantics"] = self.all_rays[idx, 9]
                sample["rays"] = torch.cat((self.all_rays[idx, :8], self.all_rays[idx, 10:13]), dim=-1)
            else:
                sample["rays"] = torch.cat((self.all_rays[idx, :8], self.all_rays[idx, 9:12]), dim=-1)
            return sample
        id_ = self.val_id if self.split == "val" else self.img_ids_train[idx]
        sample = {"c2w": torch.FloatTensor(self.poses_dict[id_])}
        img, sem = self.gen.decode(id_)
        rows, rgbs, _ = self.gen.run(id_, img, sem)
        h, w = int(img.shape[0]), int(img.shape[1])
        sample["rgbs"] = rgbs.cpu()
        sample["rays"] = rows[:, :8].cpu()
        sample["ts"] = id_ * torch.ones(h * w, dtype=torch.long)
        if self.with_semantics:                        # in the semantic map's own dtype, as cv2.resize returns it
            name = self.image_paths[id_].split(".")[0]
            dtype = np.load(os.path.join(self.root_dir, f"{self.semantic_map_path}/{name}.npz"))["arr_0"].dtype
            sample["semantics"] = torch.from_numpy(rows[:, 9:10].cpu().numpy().astype(dtype))
        sample["img_wh"] = torch.LongTensor([w, h])
        sample["K"] = self.Ks[id_]
        return sample


def check_voxel_misses(n_miss, n_images):
    if n_images and n_miss == n_images:
        raise NrwError("no ray of any training image hits the SfM voxels: check config.yaml's eval_bbx / sfm2gt")
    if n_miss:
        warnings.warn(f"{n_miss} of {n_images} training images have no ray that hits the SfM voxels")
