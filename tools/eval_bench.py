"""Evaluation timings on one GPU, written as one JSON file (--out DIR/eval_bench.json).

Seeded synthetic scenes (a noisy wavy surface with 1 % outliers):
  * point-cloud mode, 5 M predicted x 5 M ground-truth points: index build and query in each direction, and the whole
    eval_mesh (file reads timed separately);
  * mesh mode: a marching_cubes sphere mesh sampled to 10 x 2 M ground-truth points: sampling and the whole eval_mesh.
GPU figures are CUDA-event times (host timers around synchronised work for eval_mesh), median of --reps after one
warm-up.  For comparison on the same host: scipy cKDTree (workers=-1) build and query, and the reference's own per-point
loop (utils/eval_utils.py::nn_correspondance, use_o3d=False) on a random 20 k subsample of each direction, extrapolated
to the full query count (cKDTree's prediction -> ground-truth query likewise, on 50 k; see below).
The card's name and power limit are read with a read-only nvidia-smi query."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

BBX = [[-1.0, -1.0, -0.5], [1.0, 1.0, 0.5]]


_T0 = time.perf_counter()


def _log(res, out, stage):
    """progress line and the results so far (a long stage is visible as it runs)"""
    print(f"[eval_bench {time.perf_counter() - _T0:7.1f} s] {stage}", flush=True)
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "eval_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)


def _events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return {"median_ms": float(np.median(ms)), "ms": ms}


def _host(fn, reps):
    fn()
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": float(np.median(ms)), "ms": ms}


def _once(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="eval_bench_out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=5_000_000, help="points per cloud in point-cloud mode")
    ap.add_argument("--n_gt_mesh", type=int, default=2_000_000, help="ground-truth points in mesh mode")
    ap.add_argument("--loop_subsample", type=int, default=20_000)
    ap.add_argument("--ckdtree_subsample", type=int, default=50_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench: needs a CUDA device")
    from nrw.evaluation import NearestNeighbours, eval_mesh, sample_points_uniformly
    from nrw.mesh import marching_cubes, read_ply, write_ply
    from scipy.spatial import cKDTree
    from util_eval import surface_scene

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "host_cpus": os.cpu_count(), "reps": args.reps}
    rng = np.random.default_rng(0)
    lo, hi = np.array(BBX[0]), np.array(BBX[1])
    gt, pred = surface_scene(rng, args.n, args.n, lo - 0.05, hi + 0.05, noise=0.005)
    g, p = torch.from_numpy(gt).cuda(), torch.from_numpy(pred).cuda()
    _log(res, args.out, "scene")

    # ---- point-cloud mode: GPU ----
    pc = {"n_pred": len(pred), "n_gt": len(gt)}
    pc["build_pred_index"] = _events(lambda: NearestNeighbours(p), args.reps)
    pc["build_gt_index"] = _events(lambda: NearestNeighbours(g), args.reps)
    ip, ig = NearestNeighbours(p), NearestNeighbours(g)
    pc["query_gt_in_pred"] = _events(lambda: ip.query(g), args.reps)          # recall side (dist1)
    pc["query_pred_in_gt"] = _events(lambda: ig.query(p), args.reps)          # precision side (dist2)
    d1, _ = ip.query(g)
    d2, _ = ig.query(p)
    res["point_cloud_mode"] = pc
    _log(res, args.out, "gpu nearest neighbours")
    # ---- the same on the host: cKDTree, and the reference's per-point loop ----
    # A query far from a dense surface visits a great many cKDTree cells (its cells are split regions, not boxes around
    # the points), so the 1 % outliers dominate the prediction -> ground-truth direction: that direction is timed on a
    # random subsample and extrapolated linearly, as is the per-point loop in both directions.
    (kp, t_kp) = _once(lambda: cKDTree(pred))
    (kg, t_kg) = _once(lambda: cKDTree(gt))
    (kd1, _), t_q1 = _once(lambda: kp.query(gt, workers=-1))
    sub_q = np.sort(rng.choice(len(pred), args.ckdtree_subsample, replace=False))
    (kd2, _), t_q2 = _once(lambda: kg.query(pred[sub_q], workers=-1))
    pc["ckdtree_workers_all"] = {
        "build_pred_ms": t_kp, "build_gt_ms": t_kg, "query_gt_in_pred_ms": t_q1,
        "query_pred_in_gt_subsample": len(sub_q), "query_pred_in_gt_ms_on_subsample": t_q2,
        "query_pred_in_gt_ms_extrapolated": t_q2 * len(pred) / len(sub_q),
        "distances_bit_identical": bool(np.array_equal(kd1, d1.cpu().numpy()) and np.array_equal(kd2, d2[torch.from_numpy(sub_q).cuda()].cpu().numpy()))}
    del kp, kg
    _log(res, args.out, "cKDTree")
    try:
        from oracle import eval_port

        eu = eval_port.load_eval().eval_utils
        from scipy.spatial import KDTree

        loop = {"subsample": args.loop_subsample}
        for name, ref_pts, qry, dd in (("gt_in_pred", pred, gt, d1), ("pred_in_gt", gt, pred, d2)):
            sub = np.sort(rng.choice(len(qry), args.loop_subsample, replace=False))
            _, t_build = _once(lambda: KDTree(ref_pts))
            (_, rd), t_all = _once(lambda: eu.nn_correspondance(ref_pts, qry[sub], use_o3d=False))    # builds its own tree
            loop[name] = {"kdtree_build_ms": t_build, "loop_ms_on_subsample": t_all - t_build,
                          "extrapolated_ms": t_build + (t_all - t_build) * len(qry) / len(sub),
                          "subsample_distances_bit_identical": bool(np.array_equal(np.asarray(rd), dd[torch.from_numpy(sub).cuda()].cpu().numpy()))}
            _log(res, args.out, f"reference loop {name}")
        pc["reference_loop_extrapolated"] = loop
    except RuntimeError as e:                                 # no reference copy next to the tree
        pc["reference_loop_extrapolated"] = {"skipped": str(e)}
    cfg = {"eval_bbx": BBX, "sfm2gt": np.eye(4).tolist()}
    with tempfile.TemporaryDirectory() as td:
        write_ply(f"{td}/gt.ply", gt)
        write_ply(f"{td}/pred.ply", pred)
        pc["read_ply_ms"] = _host(lambda: (read_ply(f"{td}/gt.ply"), read_ply(f"{td}/pred.ply")), args.reps)
        th = [0.01 * k for k in range(1, 21)]
        pc["eval_mesh_ms"] = _host(lambda: eval_mesh(f"{td}/pred.ply", f"{td}/gt.ply", cfg, False, threshold=th, save_name="b"), args.reps)
        pc["fscores"] = json.load(open(f"{td}/eval_b/metrics.json"))["fscores"]
    _log(res, args.out, "point-cloud eval_mesh")
    del g, p, ip, ig, d1, d2
    torch.cuda.empty_cache()

    # ---- mesh mode ----
    dim, R = 512, 0.4
    lin = torch.linspace(-1, 1, dim, device="cuda")
    x = lin[:, None, None]
    y = lin[None, :, None]
    z = lin[None, None, :]
    vol = torch.sqrt(x * x + y * y + z * z) - R
    v, f, _ = marching_cubes(vol)
    verts = v.double() * (2.0 / (dim - 1)) - 1.0
    faces = f.long()
    del vol
    gen = torch.Generator().manual_seed(1)
    d = torch.randn(args.n_gt_mesh, 3, generator=gen, dtype=torch.float64)
    gtm = (d / d.norm(dim=1, keepdim=True) * R + torch.randn(args.n_gt_mesh, 3, generator=gen, dtype=torch.float64) * 0.002).numpy()
    k = args.n_gt_mesh // 100
    gtm[:k] = np.random.default_rng(2).uniform(-1, 1, (k, 3)) * [1.0, 1.0, 0.5]
    mm = {"mesh_verts": int(verts.shape[0]), "mesh_faces": int(faces.shape[0]), "n_gt": len(gtm), "n_samples": 10 * len(gtm)}
    res["mesh_mode"] = mm
    mm["sample_ms"] = _events(lambda: sample_points_uniformly(verts, faces, 10 * len(gtm)), args.reps)
    _log(res, args.out, "sampling")
    with tempfile.TemporaryDirectory() as td:
        write_ply(f"{td}/mesh.ply", verts.cpu().numpy(), faces.cpu().numpy())
        write_ply(f"{td}/gt.ply", gtm)
        mm["read_ply_ms"] = _host(lambda: (read_ply(f"{td}/gt.ply"), read_ply(f"{td}/mesh.ply")), args.reps)
        cfgm = {"eval_bbx": [[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]], "sfm2gt": np.eye(4).tolist()}
        mm["eval_mesh_ms"] = _host(lambda: eval_mesh(f"{td}/mesh.ply", f"{td}/gt.ply", cfgm, True, threshold=[0.005, 0.01, 0.02],
                                                     save_name="m"), args.reps)
        mm["fscores"] = json.load(open(f"{td}/eval_m/metrics.json"))["fscores"]
    _log(res, args.out, "mesh eval_mesh")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
