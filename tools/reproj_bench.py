"""Visibility-filter timings on one GPU, written as one JSON file (--out DIR/reproj_bench.json).

A seeded scene: the marching_cubes mesh of a bumpy sphere and a second sphere beside it on a --dim^3 SDF lattice (about
2.5 M faces at the default 768), seen by --views cameras of --width x --height pixels (about 1 MP) on a ring around it;
the target points are the mesh's own vertices, as in the reference pipeline.  Timed (CUDA events, median over the
views after one warm-up view): the depth raster per view and the back-projection + nearest-point query + marking per
view, and the whole `reproj_filter` (host timer around synchronised work, index build included).  For comparison, the
reference's per-pixel correspondence loop (one KD-tree query per covered pixel) cannot run here without open3d; scipy's
cKDTree queried one pixel at a time in a Python loop over a random --loop_subsample of one view's back-projected
pixels is timed instead and extrapolated to every covered pixel of every view (labelled extrapolated).
The card's name and power limit are read with a read-only nvidia-smi query in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _scene(dim):
    from nrw.mesh import marching_cubes

    lin = torch.linspace(-1.6, 1.6, dim, device="cuda", dtype=torch.float32)
    X, Y, Z = torch.meshgrid(lin, lin, lin, indexing="ij")
    r = torch.sqrt(X * X + Y * Y + Z * Z)
    bump = 0.05 * torch.sin(7 * X) * torch.sin(6 * Y) * torch.sin(5 * Z)
    sdf = torch.minimum(r - 1.0 + bump, torch.sqrt((X - 1.0) ** 2 + (Y + 0.6) ** 2 + (Z - 0.5) ** 2) - 0.45)
    v, f, _ = marching_cubes(sdf)
    h = 3.2 / (dim - 1)
    return (-1.6 + h * v.double()), f.long()


def _cameras(rng, n, width, height):
    from util_reproj import look_at, view_matrix

    Ks, Es, whs = [], [], []
    f = 0.9 * width
    for k in range(n):
        ph = 2 * np.pi * k / n + rng.uniform(-0.05, 0.05)
        th = np.deg2rad(rng.uniform(50, 100))
        eye = rng.uniform(3.0, 4.5) * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        R, t = look_at(eye, rng.normal(size=3) * 0.2, up=(0.0, 0.0, 1.0))
        Es.append(view_matrix(R, t))
        Ks.append(np.array([[f, 0, width / 2], [0, f, height / 2], [0, 0, 1]], dtype=np.float32))
        whs.append((width, height))
    return Ks, np.array(Es), whs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="reproj_bench_out")
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--width", type=int, default=1152)
    ap.add_argument("--height", type=int, default=864)
    ap.add_argument("--voxel_size", type=float, default=0.01)
    ap.add_argument("--loop_subsample", type=int, default=20_000)
    args = ap.parse_args()
    from nrw.reprojection import DepthRenderer, VisibilityMarker, reproj_filter

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "host_cpus": os.cpu_count(), "args": vars(args)}
    rng = np.random.default_rng(0)
    v, f = _scene(args.dim)
    res["n_verts"], res["n_faces"] = int(v.shape[0]), int(f.shape[0])
    Ks, Es, whs = _cameras(rng, args.views, args.width, args.height)
    thr = 2 * np.sqrt(2) * args.voxel_size

    renderer = DepthRenderer(v, f, device=0)
    marker = VisibilityMarker(v)
    t_r, t_m = [], []
    covered = []
    for i, (K, E, (w, h)) in enumerate(zip(Ks, Es, whs)):
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record()
        depth = renderer(h, w, K, E)
        b.record()
        marker.mark(depth, K, np.linalg.inv(E), thr)
        c.record()
        torch.cuda.synchronize()
        if i > 0:
            t_r.append(a.elapsed_time(b))
            t_m.append(b.elapsed_time(c))
        covered.append(int((depth > 0).sum()))
    res["raster_ms_per_view"] = {"median": float(np.median(t_r)), "min": float(np.min(t_r)), "max": float(np.max(t_r))}
    res["mark_ms_per_view"] = {"median": float(np.median(t_m)), "min": float(np.min(t_m)), "max": float(np.max(t_m))}
    res["covered_pixels_per_view_median"] = float(np.median(covered))
    res["covered_pixels_total"] = int(np.sum(covered))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mask = reproj_filter(v, f, v, Ks, Es, whs, voxel_size=args.voxel_size)
    torch.cuda.synchronize()
    res["reproj_filter_s"] = time.perf_counter() - t0
    res["visible_points"] = int(mask.sum())
    print(json.dumps(res), flush=True)

    # per-pixel KD-tree loop on the host, subsampled and extrapolated
    from scipy.spatial import cKDTree

    from oracle import reproj_port as rp

    vh = v.cpu().numpy()
    t0 = time.perf_counter()
    tree = cKDTree(vh)
    build_s = time.perf_counter() - t0
    K, E, (w, h) = Ks[0], Es[0], whs[0]
    d = renderer(h, w, K, E).cpu().numpy()
    X = rp.backproject(d, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), np.linalg.inv(E))
    sub = X[rng.choice(len(X), min(args.loop_subsample, len(X)), replace=False)]
    t0 = time.perf_counter()
    for p in sub:
        dist, _ = tree.query(p, k=1)
        _ = dist < thr
    per = (time.perf_counter() - t0) / len(sub)
    res["host_loop"] = {"kdtree_build_s": build_s, "per_pixel_us": per * 1e6, "sampled_pixels": int(len(sub)),
                        "extrapolated_total_s": per * res["covered_pixels_total"],
                        "note": "scipy cKDTree queried one pixel at a time; extrapolated to all covered pixels"}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "reproj_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
