"""Point-cloud visibility timings on one GPU, written as one JSON file (--out DIR/voxelvis_bench.json).

A seeded scene: --points points (3 M by default) on a bumpy sphere and a second sphere beside it, voxelised at the octree
level that --voxel_size gives in the [-2, 2]^3 cube (13 by default), seen by --views cameras of --width x --height pixels
on a ring around it.  Timed per view (CUDA events, median over the views after one warm-up view), in the same run:
  * the pruned first-hit cast (nrw_voxel_cast, VoxelRenderer.cast);
  * the unpruned path: the same rays generated with torch, nrw_octree_near_far (the full walk of the training
    traversal) and a torch scatter of the hit leaves;
and the whole reproj_filter_points (host timer around synchronised work, octree build included).  For comparison, the
numpy restatement oracle/voxelvis_port.py is timed on --oracle_rays rays of one view and extrapolated to every ray of
every view (labelled extrapolated).  The card's name and power limit are read with a read-only nvidia-smi query."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")]

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

CFG = {"sfm2gt": np.eye(4).tolist(), "eval_bbx": [[-2.0, -2.0, -2.0], [2.0, 2.0, 2.0]]}


def _scene(rng, n):
    n_a = n * 3 // 4
    v = rng.normal(size=(n_a, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    bump = 1.0 + 0.05 * np.sin(7 * v[:, 0]) * np.sin(6 * v[:, 1]) * np.sin(5 * v[:, 2])
    a = v * bump[:, None]
    w = rng.normal(size=(n - n_a, 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    b = w * 0.45 + np.array([1.0, -0.6, 0.5])
    return np.concatenate([a, b])


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
    return Ks, Es, whs


def _torch_rays(h, w, K, c2w):
    """gen_rays' fp32 order in torch (the unpruned path's ray generation)"""
    M = torch.as_tensor(np.asarray(c2w, np.float64)[:3], dtype=torch.float32, device="cuda")
    fx, fy, cx, cy = (float(np.float32(K[i, j])) for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    r, c = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float32),
                          torch.arange(w, device="cuda", dtype=torch.float32), indexing="ij")
    dx, dy = ((c - cx) / fx).reshape(-1), ((r - cy) / fy).reshape(-1)
    d = torch.stack([(dx * M[k, 0] + dy * M[k, 1]) + M[k, 2] for k in range(3)], 1)
    n = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    d = (d / n[:, None]).contiguous()
    o = M[:, 3].expand(d.shape[0], 3).contiguous()
    return o, d, n


def _stats(x):
    return {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="voxelvis_bench_out")
    ap.add_argument("--points", type=int, default=3_000_000)
    ap.add_argument("--voxel_size", type=float, default=0.00025)
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--width", type=int, default=1152)
    ap.add_argument("--height", type=int, default=864)
    ap.add_argument("--oracle_rays", type=int, default=8)
    args = ap.parse_args()
    from nrw import _lib
    from nrw.reprojection import VoxelRenderer, reproj_filter_points

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "host_cpus": os.cpu_count(), "args": vars(args)}
    rng = np.random.default_rng(0)
    pts = _scene(rng, args.points)
    Ks, Es, whs = _cameras(rng, args.views, args.width, args.height)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = VoxelRenderer(pts, CFG, args.voxel_size, device=0)
    torch.cuda.synchronize()
    res["octree_build_s"] = time.perf_counter() - t0
    res["level"], res["n_leaf"] = r.level, r.n_leaf
    L = _lib.lib()
    base = int(r.tree["pyramid"][1, r.level])
    org = (C.c_float * 3)(*r.origin.tolist())
    visible_full = torch.zeros(r.n_leaf, dtype=torch.uint8, device="cuda")
    t_p, t_u, hits = [], [], []
    for i, (K, E, (w, h)) in enumerate(zip(Ks, Es, whs)):
        c2w = np.linalg.inv(E)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        n0 = int(r.n_hit.item())
        ev[0].record()
        r.cast(h, w, K, E)
        ev[1].record()
        o, d, _ = _torch_rays(h, w, K, c2w)
        R = o.shape[0]
        near, far = torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
        pid, cnt = torch.empty(R, dtype=torch.int32, device="cuda"), torch.empty(R, dtype=torch.int32, device="cuda")
        ev[2].record()
        _lib.check(L.nrw_octree_near_far(_lib.ptr(r.tree["octree"]), _lib.ptr(r.tree["prefix"]), r._pyr, r.level, _lib.ptr(o),
                                         _lib.ptr(d), R, org, r.scale, _lib.ptr(near), _lib.ptr(far), _lib.ptr(pid),
                                         _lib.ptr(cnt), _lib.stream_ptr()), "nrw_octree_near_far")
        p = pid[pid >= 0].long() - base
        visible_full[p] = 1
        ev[3].record()
        torch.cuda.synchronize()
        if i > 0:
            t_p.append(ev[0].elapsed_time(ev[1]))
            t_u.append(ev[1].elapsed_time(ev[3]))
        hits.append(int(r.n_hit.item()) - n0)
    res["same_marked_leaves"] = bool(torch.equal(r.visible, visible_full))
    res["pruned_cast_ms_per_view"] = _stats(t_p)
    res["unpruned_ms_per_view"] = _stats(t_u)
    res["unpruned_note"] = "torch ray generation + nrw_octree_near_far (full walk) + torch scatter, same rays"
    res["hit_pixels_per_view_median"] = float(np.median(hits))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mask = reproj_filter_points(pts, CFG, Ks, Es, whs, voxel_size=args.voxel_size)
    torch.cuda.synchronize()
    res["reproj_filter_points_s"] = time.perf_counter() - t0
    res["kept_points"] = int(mask.sum())
    print(json.dumps(res), flush=True)

    # numpy restatement on a few rays of one view, extrapolated
    from oracle import octree_port as op
    from oracle import voxelvis_port as vp

    tree, origin, scale, level, _ = op.gen_octree(CFG, pts, args.voxel_size, expand=0, in_sfm=False)
    K, E, (w, h) = Ks[0], Es[0], whs[0]
    o, d, _ = vp.gen_rays(h, w, K, np.linalg.inv(E))
    sel = rng.choice(len(o), args.oracle_rays, replace=False)
    t0 = time.perf_counter()
    vp.first_hit(tree, level, o[sel], d[sel], origin, scale)
    per = (time.perf_counter() - t0) / len(sel)
    total_rays = sum(w * h for w, h in whs)
    res["numpy_oracle"] = {"per_ray_ms": per * 1e3, "sampled_rays": int(len(sel)), "extrapolated_total_s": per * total_rays,
                           "note": "oracle/voxelvis_port.first_hit on sampled rays of one view; extrapolated to all rays"}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "voxelvis_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
