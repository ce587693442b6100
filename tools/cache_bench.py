"""Times ray-cache generation on a seeded synthetic scene: the per-image pass (CUDA events around RayGenerator.run on a
decoded image, so the upload and the count read-back are included) and the near/far percentiles (CUDA events), end-to-end images/s with PIL decode and npz writing timed separately, and the numpy
restatement on a few images.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/cache_bench.py --images 100 --width 1024 --height 768 --points 500000 --out cache_bench_out
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:      # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--height", type=int, default=768)
    ap.add_argument("--points", type=int, default=500000)
    ap.add_argument("--cpu_images", type=int, default=2)
    ap.add_argument("--out", default="cache_bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cache_bench needs a CUDA device")
    import util_cache
    from oracle import cache_port as cp
    from nrw.phototourism import RayGenerator, build_octrees, depth_bounds, read_scene
    from nrw.prepare_data_cache import get_opts, prepare

    util_cache.SIZES[:] = [(a.width, a.height)]
    root = os.path.join(os.path.abspath(a.out), "bench_scene")
    util_cache.write_scene(root, n_train=a.images, n_test=0, n_points=a.points, seed=0)
    dev = torch.device("cuda", 0)
    s = read_scene(root, 1, "sparse")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    depth_bounds(s.xyz_world, s.w2c, dev)
    ev[0].record()
    b = depth_bounds(s.xyz_world, s.w2c, dev)
    ev[1].record()
    torch.cuda.synchronize()
    t_bounds = ev[0].elapsed_time(ev[1])
    gen = RayGenerator(s, dev, True, "semantic_maps", use_voxel=True, bounds=b, octrees=build_octrees(root, s.config, dev))
    decoded = [gen.decode(i) for i in s.img_ids[:8]]
    t0 = time.perf_counter()
    for k, i in enumerate(s.img_ids[:8]):
        gen.decode(i)
    t_decode = (time.perf_counter() - t0) / 8 * 1e3
    gen.run(s.img_ids[0], *decoded[0])
    dev_ms = []
    for k, i in enumerate(s.img_ids[:8]):
        ev[0].record()
        gen.run(i, *decoded[k])
        ev[1].record()
        torch.cuda.synchronize()
        dev_ms.append(ev[0].elapsed_time(ev[1]))
    t0 = time.perf_counter()
    res = prepare(get_opts(["--root_dir", root, "--cache_dir", "cache", "--cache_type", "npz", "--split_to_chunks", "8",
                            "--semantic_map_path", "semantic_maps"]))
    t_e2e = time.perf_counter() - t0
    rows = np.load(os.path.join(root, "cache", "splits", "split_0", "rays1.npz"))["arr_0"]     # real rows of one split
    t0 = time.perf_counter()
    np.savez_compressed(os.path.join(a.out, "one_split.npz"), rows)
    t_npz = time.perf_counter() - t0
    os.remove(os.path.join(a.out, "one_split.npz"))
    t0 = time.perf_counter()
    for i in s.img_ids[:a.cpu_images]:
        k = s.img_ids.index(i)
        _, xys, ids = s.imdata[i]
        img = decoded[min(k, 7)][0].numpy()
        cp.image_rows(a.height, a.width, s.Ks[i], s.poses[k].astype(np.float32), i, img, b[k, 0], b[k, 1], xys, ids, s.table_xyz,
                      s.table_err, 1, s.w2c[k, 2, :4])
    t_cpu = (time.perf_counter() - t0) / max(1, a.cpu_images) * 1e3
    print(json.dumps({"card": card(), "images": a.images, "size": [a.width, a.height], "points": a.points,
                      "pass_ms_per_image_median": float(np.median(dev_ms)), "percentiles_ms_all_images": t_bounds,
                      "decode_ms_per_image": t_decode, "end_to_end_images_per_s": a.images / t_e2e,
                      "end_to_end_s": t_e2e, "npz_write_s_one_split": t_npz, "rows": res["rows"],
                      "numpy_restatement_ms_per_image_no_voxels": t_cpu}))


if __name__ == "__main__":
    main()
