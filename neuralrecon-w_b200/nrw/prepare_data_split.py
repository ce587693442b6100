"""python -m nrw.prepare_data_split: tools/prepare_data/prepare_data_split.py with the per-pixel work on the GPU.

Selects the training views of a COLMAP scene and writes its <scene>.tsv (filename, id, split, dataset), the file every
later step reads (read_tsv, get_train_ids):

    view_selection      dataset_filter_utils.view_selection: the sparse_filtered_{n} covisibility rule, then the share of
                        each view's pixels whose ray passes through the scene sphere (csrc/viewsel.cu, one launch)
    filter_image_based_on_transient_percent   the share of each semantic map's pixels that are not a transient class
                        (counted on the device, read back once)
    roi_keep, static_keep, split_rows, tsv_bytes   the pure pieces: counts -> kept names, rows -> tsv bytes

Image sizes come from the file headers (PIL opens without decoding).  The split decision, the permutation and the tsv
stay on the host.  Deviations from the reference are listed in INTEGRATION.md.
"""
import argparse
import collections
import concurrent.futures
import csv
import ctypes
import io
import os
import shutil
import sys

import numpy as np

from . import _lib, colmap
from ._lib import NrwError, check, ptr, stream_ptr

TRANSIENT_OBJECTS = ("person", "car", "bicycle", "minibike", "tree")
INT32_MAX = (1 << 31) - 1


def get_opts(argv=None):
    p = argparse.ArgumentParser(prog="python -m nrw.prepare_data_split")
    p.add_argument("--root_dir", type=str, required=True, help="root directory of dataset")
    p.add_argument("--num_test", type=int, default=10, help="size of test set")
    p.add_argument("--min_observation", type=int, default=-1, help="min_observation for view selection")
    p.add_argument("--roi_threshold", type=float, default=0.5, help="roi_threshold to filter images")
    p.add_argument("--static_threshold", type=float, default=0.6, help="keep an image whose static share is above it; "
                   "a negative value reads no semantic map")
    p.add_argument("--nima_ckpt_path", type=str, default="weights/nima_epoch-34.pth",
                   help="accepted and ignored (the reference's NIMA filter is not called)")
    p.add_argument("--semantic_map_path", type=str, default="semantic_maps")
    p.add_argument("--seed", type=int, default=0, help="seed of the train / test permutation")
    return p.parse_args(argv)


def scene_name(root_dir):
    return os.path.basename(os.path.normpath(root_dir))


def image_size(path):
    """(width, height) from the file header; PIL reads no pixel data here"""
    from PIL import Image

    with Image.open(path) as im:
        return im.size


def pinhole_K(cam):
    """fp32 K from params[0..3] of a PINHOLE camera (view_selection's K)"""
    if cam.model != "PINHOLE":
        raise NrwError(f"view_selection: camera {cam.id} has model {cam.model}; only PINHOLE is supported")
    K = np.zeros((3, 3), dtype=np.float32)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[2, 2] = cam.params[0], cam.params[1], cam.params[2], cam.params[3], 1
    return K


def view_table(Ks, poses):
    """the kernel's view table: f32 [n, 16] = fx, fy, cx, cy, c2w[12] (c2w f64 [n, 3, 4] rounded to fp32)"""
    t = np.empty((len(Ks), 16), np.float32)
    for i, K in enumerate(Ks):
        t[i, :4] = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    t[:, 4:] = np.asarray(poses, np.float64).astype(np.float32).reshape(len(Ks), 12)
    return t


def roi_counts(views, hw, scene_origin, scene_radius, device=0):
    """ROI pixel count of every view (int64 [n]) from one nrw_view_roi_count launch and one read-back.  views f32
    [n, 16] as view_table makes it, hw [n, 2] = height, width; the origin and radius are rounded to fp32."""
    import torch

    hw = np.asarray(hw, np.int64).reshape(-1, 2)
    n = len(hw)
    if n == 0:
        return np.zeros(0, np.int64)
    if (hw < 1).any() or (hw[:, 0] * hw[:, 1] > INT32_MAX).any():
        raise NrwError("roi_counts: every view needs height, width >= 1 and height * width <= INT32_MAX")
    origin = np.asarray(scene_origin, np.float32).reshape(3)
    radius = np.float32(scene_radius)
    if not (np.isfinite(origin).all() and np.isfinite(radius) and radius > 0):
        raise NrwError(f"roi_counts: scene origin {origin} and radius {scene_radius} must be finite, radius > 0")
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    V = torch.from_numpy(np.ascontiguousarray(views, np.float32).reshape(n, 16)).to(dev)
    HW = torch.from_numpy(hw.astype(np.int32)).to(dev)
    counts = torch.empty(n, dtype=torch.int64, device=dev)
    o = (ctypes.c_float * 3)(*[float(v) for v in origin])
    check(_lib.lib().nrw_view_roi_count(ptr(V), ptr(HW), n, int((hw[:, 0] * hw[:, 1]).max()), o, float(radius), ptr(counts),
                                        stream_ptr()), "nrw_view_roi_count")
    out = counts.cpu().numpy()
    if (out < 0).any():
        raise NrwError("roi_counts: the device rejected a view size")
    return out


def roi_keep(counts, hw, roi_threshold):
    """view_selection's decision as torch makes it: count_nonzero / numel is fp32 (both rounded to fp32, one _rn
    division) and the threshold is rounded to fp32; a view is kept unless its share is below the threshold."""
    hw = np.asarray(hw, np.int64).reshape(-1, 2)
    share = np.asarray(counts, np.int64).astype(np.float32) / (hw[:, 0] * hw[:, 1]).astype(np.float32)
    return ~(share < np.float32(roi_threshold))


def static_keep(counts, sizes, static_threshold):
    """filter_image_based_on_transient_percent's decision: static_percent = count / (H * W) as a Python float, kept when
    above the threshold"""
    return [int(c) / (int(h) * int(w)) > static_threshold for c, (h, w) in zip(counts, sizes)]


def _reset_trash(root_dir):
    trash = os.path.join(root_dir, "trash_images")
    shutil.rmtree(trash, ignore_errors=True)
    os.makedirs(trash)
    return trash


def _trash(root_dir, name, prefix):
    """a rejected image, copied byte for byte under the reference's file name"""
    shutil.copyfile(os.path.join(root_dir, "dense/images", name), os.path.join(root_dir, "trash_images", f"{prefix}{name}"))


def view_selection(root_dir, scene_origin, scene_radius, min_observation, roi_threshold=0.2, device=0):
    """dataset_filter_utils.view_selection: the names (numpy str [n]) of the images kept by the covisibility rule and the
    ROI share, in images.bin order (the rescued cameras last).  Rebuilds trash_images/ with the rejected ones."""
    sparse = os.path.join(root_dir, "dense/sparse")
    for f in ("images.bin", "cameras.bin"):
        if not os.path.isfile(os.path.join(sparse, f)):
            raise NrwError(f"view_selection: {os.path.join(sparse, f)} not found")
    from .phototourism import camera_poses

    imdata = colmap.read_images(os.path.join(sparse, "images.bin"))
    camdata = colmap.read_cameras(os.path.join(sparse, "cameras.bin"))
    img_ids = list(imdata)
    image_paths = {i: imdata[i].name for i in img_ids}
    for i in img_ids:
        if imdata[i].camera_id not in camdata:
            raise NrwError(f"view_selection: image {i} uses camera {imdata[i].camera_id}, which is not in cameras.bin")
    Ks = {i: pinhole_K(camdata[imdata[i].camera_id]) for i in img_ids}
    _, poses = camera_poses([imdata[i] for i in img_ids], "view_selection")
    poses_dict = {id_: poses[k] for k, id_ in enumerate(img_ids)}
    _reset_trash(root_dir)
    if min_observation > 0:
        path = os.path.join(root_dir, f"dense/sparse_filtered_{min_observation}", "images.bin")
        if not os.path.isfile(path):
            raise NrwError(f"view_selection: {path} not found (--min_observation {min_observation})")
        img_id_filtered = list(colmap.read_images(path))
        unknown = set(img_id_filtered) - set(img_ids)
        if unknown:
            raise NrwError(f"view_selection: {path} has image ids {sorted(unknown)} that dense/sparse does not have")
        # the reference's expressions, so the rescued ids come in the same (set) order
        img_less_covis = set(img_ids) - set(img_id_filtered)
        for img_id in img_less_covis:
            cam = camdata[imdata[img_id].camera_id]
            if (cam.params[0] > 2000) and (cam.params[1] > 2000):
                img_id_filtered += [img_id]
        for v_id in set(img_ids) - set(img_id_filtered):
            _trash(root_dir, image_paths[v_id], "less_covis_")
        img_ids = img_id_filtered
    if not img_ids:
        return np.array([])
    hw = []
    for id_ in img_ids:
        w, h = image_size(os.path.join(root_dir, "dense/images", image_paths[id_]))
        hw.append((h, w))
    views = view_table([Ks[i] for i in img_ids], [poses_dict[i] for i in img_ids])
    counts = roi_counts(views, hw, scene_origin, scene_radius, device)
    keep = roi_keep(counts, hw, roi_threshold)
    filtered = []
    for id_, k in zip(img_ids, keep):
        if k:
            filtered.append(image_paths[id_])
        else:
            _trash(root_dir, image_paths[id_], "less_ROI_")
    return np.array(filtered)


def _load_map(root_dir, semantic_map_path, image_name):
    import torch

    from .phototourism import load_semantics

    m = load_semantics(root_dir, semantic_map_path, image_name.split(".")[0])
    if m.ndim < 2:
        raise NrwError(f"semantic map of {image_name} has shape {m.shape}; need [H, W]")
    return torch.from_numpy(m).pin_memory(), (int(m.shape[0]), int(m.shape[1]))


def static_counts(root_dir, semantic_map_path, names, ids, device=0, workers=4, ahead=4):
    """per image, the number of semantic-map pixels whose label is none of ids (int64 [n]), and the maps' (H, W).  A small
    thread pool reads the maps ahead of the device; one read-back at the end."""
    import torch

    L = _lib.lib()
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    counts = torch.zeros(len(names), dtype=torch.int64, device=dev)
    id_arr = (ctypes.c_int * max(1, len(ids)))(*[int(v) for v in ids])
    sizes = []
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        futs = collections.deque()
        it = iter(names)
        for name in it:
            futs.append(pool.submit(_load_map, root_dir, semantic_map_path, name))
            if len(futs) >= ahead:
                break
        k = 0
        while futs:
            f = futs.popleft()
            nxt = next(it, None)
            if nxt is not None:
                futs.append(pool.submit(_load_map, root_dir, semantic_map_path, nxt))
            m, hw = f.result()
            md = m.to(dev, non_blocking=True)
            check(L.nrw_label_static_count(ptr(md), md.numel(), id_arr, len(ids), ptr(counts[k:]), stream_ptr()),
                  "nrw_label_static_count")
            sizes.append(hw)
            k += 1
    return counts.cpu().numpy(), sizes


def filter_image_based_on_transient_percent(root_dir, semantic_map_path, image_paths, transient_objects, static_threshold=0.3,
                                            device=0):
    """dataset_filter_utils.filter_image_based_on_transient_percent: the names of image_paths [n, 1] whose share of
    pixels outside the transient classes is above static_threshold, as numpy str [m, 1].  The rejected ones are copied to
    trash_images/transient_much_<name>.  A negative threshold keeps every image without reading a map."""
    from .renderer import LABEL_IDS

    names = [str(v) for v in np.asarray(image_paths).reshape(len(image_paths), -1)[:, 0]] if len(image_paths) else []
    for t in transient_objects:
        if t not in LABEL_IDS:
            raise NrwError(f"transient class {t!r} has no label id (known: {sorted(LABEL_IDS)})")
    if static_threshold < 0 or not names:
        return np.array(names).reshape(-1, 1)
    ids = [LABEL_IDS[t] for t in transient_objects]
    counts, sizes = static_counts(root_dir, semantic_map_path, names, ids, device)
    kept = []
    for name, k in zip(names, static_keep(counts, sizes, static_threshold)):
        if k:
            kept.append(name)
        else:
            _trash(root_dir, name, "transient_much_")
    return np.array(kept).reshape(-1, 1)


def split_rows(names, num_test, dataset):
    """(filename, id, split, dataset) rows: the first num_test images are "test", the rest "train"."""
    n = len(names)
    if not 0 <= num_test <= n:
        raise NrwError(f"--num_test {num_test} needs at least that many kept images (kept {n})")
    return [(str(f), str(i), "test" if i < num_test else "train", dataset) for i, f in enumerate(names)]


def tsv_bytes(rows):
    """the bytes pandas' DataFrame.to_csv(sep='\\t', index=False) writes for these rows"""
    buf = io.StringIO()
    w = csv.writer(buf, delimiter="\t", lineterminator="\n", quoting=csv.QUOTE_MINIMAL, quotechar='"', doublequote=True)
    w.writerow(["filename", "id", "split", "dataset"])
    w.writerows(rows)
    return buf.getvalue().encode("utf-8")


def prepare(args, device=0):
    """Writes <root_dir>/<scene>.tsv; returns {"tsv": path, "names": the rows' file names, "num_test": n}."""
    from .phototourism import read_config

    if args.num_test < 0:
        raise NrwError(f"--num_test {args.num_test} must be >= 0")
    config = read_config(args.root_dir)
    for key in ("origin", "radius"):
        if key not in config:
            raise NrwError(f"{os.path.join(args.root_dir, 'config.yaml')} has no {key!r}")
    names = view_selection(args.root_dir, config["origin"], config["radius"], args.min_observation, args.roi_threshold, device)
    names = np.random.RandomState(args.seed).permutation(names)[:, np.newaxis]
    names = filter_image_based_on_transient_percent(args.root_dir, args.semantic_map_path, names, list(TRANSIENT_OBJECTS),
                                                    args.static_threshold, device)
    if names.shape[0] == 0:
        raise NrwError("prepare_data_split: no image is left after the view selection and the transient filter")
    rows = split_rows(list(names[:, 0]), args.num_test, scene_name(args.root_dir))
    path = os.path.join(args.root_dir, f"{scene_name(args.root_dir)}.tsv")
    with open(path, "wb") as f:
        f.write(tsv_bytes(rows))
    return {"tsv": path, "names": [r[0] for r in rows], "num_test": args.num_test}


def main(argv=None):
    args = get_opts(argv)
    res = prepare(args)
    print(f"wrote {res['tsv']}: {res['num_test']} test and {len(res['names']) - res['num_test']} train images")
    return 0


if __name__ == "__main__":
    sys.exit(main())
