"""python -m nrw.prepare_data_cache: tools/prepare_data/prepare_data_cache.py on the GPU ray generator.

Writes the byte layout load_split_arrays / the reference's loader reads: <root>/<cache_dir>/splits/split_i/{rays,rgbs}{d}.npz
(arr_0) with splits/{rays,rgbs}{d}_meta_info.json, or <root>/<cache_dir>/{rays,rgbs}{d}.npz when --split_to_chunks <= 0.
Rows are spilled image by image to raw files in the cache directory and every output file is written from a memory map
of them, so host memory holds one split plus the images in flight, not the whole cache."""
import argparse
import json
import os
import sys

import numpy as np

from ._lib import NrwError


def get_opts(argv=None):
    p = argparse.ArgumentParser(prog="python -m nrw.prepare_data_cache")
    p.add_argument("--root_dir", type=str, required=True, help="root directory of dataset")
    p.add_argument("--dataset_name", type=str, default="phototourism", choices=["phototourism"])
    p.add_argument("--cache_dir", type=str, default="cache", help="used as output directory of cache")
    p.add_argument("--cache_type", type=str, default="h5", choices=["h5", "npz"])
    p.add_argument("--img_downscale", type=int, default=1)
    p.add_argument("--split_to_chunks", type=int, default=-1, help="split large cache files to small chunks")
    p.add_argument("--cfg_path", type=str, help="unused (kept for the reference's command lines)")
    p.add_argument("--semantic_map_path", type=str, default=None)
    p.add_argument("--sfm_path", type=str, default=None, help="dense/<sfm_path> holds the keypoint depth model "
                   "(default: the reference's scene table, else 'sparse')")
    p.add_argument("--depth_percent", type=float, default=None, help="fraction of rows with keypoint depth after padding "
                   "(default: the reference's scene table, else 0)")
    p.add_argument("--seed", type=int, default=0, help="seed of the depth padding, the row permutation and the split padding")
    return p.parse_args(argv)


def split_padding(total, n_chunks, seed):
    """prepare_data_cache.py:189-198 with a seeded generator: (padding_index, chunk_length)"""
    pad = n_chunks - total % n_chunks
    if pad == n_chunks:
        return np.array([], dtype=np.int64), total // n_chunks
    idx = np.random.RandomState(seed).choice(total, pad, replace=False)
    return idx, (total + pad) // n_chunks


def write_splits(mm, padding_index, chunk_length, n_chunks, split_path, arr_type, img_downscale):
    """split_to_chunks (prepare_data_cache.py:78-159): chunk i = rows [i*L, (i+1)*L) of cat(rows, rows[padding_index])"""
    total = mm.shape[0]
    for i in range(n_chunks):
        a, b = i * chunk_length, (i + 1) * chunk_length
        parts = [mm[a:min(b, total)]]
        if b > total:
            parts.append(mm[np.asarray(padding_index[max(0, a - total):b - total], dtype=np.int64)])
        d = os.path.join(split_path, f"split_{i}")
        os.makedirs(d, exist_ok=True)
        np.savez_compressed(os.path.join(d, f"{arr_type}{img_downscale}.npz"), np.concatenate(parts, 0))
    meta = {"data_length": total + len(padding_index), "chunk_length": chunk_length, "n_trunks": n_chunks}
    with open(os.path.join(split_path, f"{arr_type}{img_downscale}_meta_info.json"), "w") as f:
        json.dump(meta, f)


def prepare(args, device=0):
    """Generates the cache; returns {"rows": total rows, "images": n, "missed": images without a voxel hit}."""
    import torch

    from .phototourism import RayGenerator, check_voxel_misses, depth_bounds, read_scene, scene_defaults

    if args.cache_type == "h5":
        raise NrwError("--cache_type h5 is not supported (h5py is not a dependency); use --cache_type npz")
    d_sfm, d_pct = scene_defaults(args.root_dir)
    sfm_path = d_sfm if args.sfm_path is None else args.sfm_path
    depth_percent = d_pct if args.depth_percent is None else args.depth_percent
    with_sem = args.semantic_map_path is not None
    out_dir = os.path.join(args.root_dir, args.cache_dir)
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    scene = read_scene(args.root_dir, args.img_downscale, sfm_path)
    bounds = depth_bounds(scene.xyz_world, scene.w2c, dev)
    train = [i for i in scene.img_ids if scene.splits[i] != "test"]
    gen = RayGenerator(scene, dev, with_sem, args.semantic_map_path, use_voxel=True, depth_percent=depth_percent,
                       seed=args.seed, bounds=bounds)
    C = 12 if with_sem else 11
    spill = {k: os.path.join(out_dir, f".{k}{args.img_downscale}.spill") for k in ("rays", "rgbs")}
    total, missed = 0, 0
    try:
        with open(spill["rays"], "wb") as fr, open(spill["rgbs"], "wb") as fg:
            for id_, rows, rgbs, counts in gen.images(train):
                missed += counts[1] == 0
                fr.write(rows.cpu().numpy().tobytes())
                fg.write(rgbs.cpu().numpy().tobytes())
                total += rows.shape[0]
        check_voxel_misses(missed, len(train))
        if total == 0:
            raise NrwError("prepare_data_cache: no rows")
        mm = {"rays": np.memmap(spill["rays"], dtype=np.float32, mode="r", shape=(total, C)),
              "rgbs": np.memmap(spill["rgbs"], dtype=np.float32, mode="r", shape=(total, 3))}
        if args.split_to_chunks > 0:
            split_path = os.path.join(out_dir, "splits")
            os.makedirs(split_path, exist_ok=True)
            pidx, L = split_padding(total, args.split_to_chunks, args.seed)
            for k in ("rgbs", "rays"):
                write_splits(mm[k], pidx, L, args.split_to_chunks, split_path, k, args.img_downscale)
        else:
            for k in ("rays", "rgbs"):
                np.savez_compressed(os.path.join(out_dir, f"{k}{args.img_downscale}.npz"), mm[k])
        del mm
    finally:
        for p in spill.values():
            if os.path.exists(p):
                os.remove(p)
    return {"rows": total, "images": len(train), "missed": int(missed)}


def main(argv=None):
    args = get_opts(argv)
    res = prepare(args)
    print(f"Data cache saved to {os.path.join(args.root_dir, args.cache_dir)}: {res['rows']} rows from {res['images']} images")
    return 0


if __name__ == "__main__":
    sys.exit(main())
