"""Ground-truth alignment check timings on one GPU, written as one JSON file (--out DIR/reproj_error_bench.json).

A seeded scene: --points GT points (20 M by default) on three planes, --views cameras of --width x --height pixels
looking at them, and --tracks SfM tracks of 4 .. 12 observations each, written as a COLMAP model and a PLY.  Timed:
  * nrw_first_hit over every track's reference observation (CUDA events, median of --reps after one warm-up), per pass
    and per view, with the default scratch (16 views per pass);
  * nrw_obs_reproj_error over every observation (CUDA events);
  * the whole gt_reproject_error, files included (host clock around synchronised work, after one warm-up run);
  * for comparison, the unmodified get_gt_point of tools/reproj_error.py (from oracle/_ref) on the GPU for
    --ref_tracks tracks at its default batch size 2, extrapolated to every track (labelled extrapolated).
Also recorded: the point loads of one pass (12 B per point) over the pass time against 3.35 TB/s, and the card's name
and power limit from a read-only nvidia-smi query."""
import argparse
import contextlib
import ctypes as C
import io
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _scene(rng, args):
    from oracle import trackerr_port as tp

    n = args.points
    k = rng.integers(0, 3, n)
    uv = rng.uniform(-3.0, 3.0, (n, 2))
    pts = np.zeros((n, 3))
    pts[k == 0] = np.c_[uv[k == 0], np.zeros((k == 0).sum())]                       # ground
    pts[k == 1] = np.c_[uv[k == 1, 0], np.full((k == 1).sum(), 1.0), uv[k == 1, 1] * 0.5 + 1.5]   # wall
    pts[k == 2] = np.c_[np.full((k == 2).sum(), -1.0), uv[k == 2, 0], uv[k == 2, 1] * 0.5 + 1.5]  # wall
    gt = pts.astype(np.float32)
    Ks, qs, Es = [], [], []
    f = 0.9 * args.width
    for i in range(args.views):
        ph = 2 * np.pi * i / args.views
        eye = np.array([4.0 * np.cos(ph), 4.0 * np.sin(ph), 3.0])
        z = -eye / np.linalg.norm(eye)
        x = np.cross(z, [0.0, 0.0, 1.0])
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        q = tp._qvec(R)
        R = tp._qrot(q)
        E = np.eye(4)
        E[:3, :3], E[:3, 3] = R, -R @ eye
        Ks.append(np.array([[f, 0, args.width / 2], [0, f, args.height / 2], [0, 0, 1]], np.float32))
        qs.append(q)
        Es.append(E)
    xys = [[] for _ in range(args.views)]
    pids = [[] for _ in range(args.views)]
    tracks, xyz = [], []
    for t in range(args.tracks):
        X = gt[rng.integers(n)].astype(np.float64)
        tr = []
        for v in rng.choice(args.views, int(rng.integers(4, 13)), replace=False):
            p = tp.projection(Ks[v], Es[v]) @ np.append(X, 1.0)
            tr.append((v, len(xys[v])))
            xys[v].append(p[:2] / p[2] + rng.normal(0, 0.5, 2))
            pids[v].append(1 + t)
        tracks.append([(v + 1, j) for v, j in tr])
        xyz.append(X)
    obj = lambda xs: np.array([np.asarray(a) for a in xs] + [None], dtype=object)[:-1]
    return {"names": np.array(["a0.jpg", "a1.jpg"] + [f"view_{i:04d}.jpg" for i in range(args.views)]),
            "gt": gt, "sfm2gt": np.eye(4), "views": (Ks, qs, Es), "xys": xys, "pids": pids, "tracks": tracks,
            "xyz": np.array(xyz), "obj": obj}


def _write(d, sc, args):
    import yaml

    from nrw.mesh import write_ply
    from oracle import trackerr_port as tp

    os.makedirs(os.path.join(d, "dense", "sparse"), exist_ok=True)
    os.makedirs(os.path.join(d, "dense", "images"), exist_ok=True)
    Ks, qs, Es = sc["views"]
    # two listed names that are not views: get_image_id skips the first two of the sorted listing
    for name in sc["names"]:
        open(os.path.join(d, "dense", "images", str(name)), "wb").close()
    tp.write_cameras(os.path.join(d, "dense", "sparse", "cameras.bin"),
                     [(1, 1, args.width, args.height, (K[0, 0], K[1, 1], K[0, 2], K[1, 2])) for K in Ks[:1]])
    tp.write_images(os.path.join(d, "dense", "sparse", "images.bin"),
                    [(i + 1, qs[i], Es[i][:3, 3], 1, str(sc["names"][i + 2]), np.array(sc["xys"][i]).reshape(-1, 2),
                      np.array(sc["pids"][i], np.int64)) for i in range(len(Ks))])
    tp.write_points3d(os.path.join(d, "dense", "sparse", "points3D.bin"), np.arange(1, len(sc["xyz"]) + 1), sc["xyz"],
                      np.full(len(sc["xyz"]), 0.1), sc["tracks"])
    with open(os.path.join(d, "config.yaml"), "w") as fh:
        yaml.safe_dump({"sfm2gt": np.eye(4).tolist()}, fh)
    write_ply(os.path.join(d, "gt.ply"), sc["gt"])
    return os.path.join(d, "gt.ply")


def _events(fn, reps):
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=20_000_000)
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--width", type=int, default=1152)
    ap.add_argument("--height", type=int, default=864)
    ap.add_argument("--tracks", type=int, default=30_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref_tracks", type=int, default=20)
    ap.add_argument("--out", default="reproj_error_bench_out")
    args = ap.parse_args()
    from nrw import _lib
    from nrw import reproj_error as R
    from nrw._lib import check, ptr, stream_ptr
    from nrw.evaluation import _scratch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "args": vars(args)}
    rng = np.random.default_rng(0)
    sc = _scene(rng, args)
    with tempfile.TemporaryDirectory() as d:
        gp = _write(d, sc, args)
        work = os.path.join(d, "work")
        os.makedirs(work)
        cwd = os.getcwd()
        os.chdir(work)
        try:
            for rep in range(2):                              # the first run warms up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):
                    loss = R.gt_reproject_error(d, gp, np.eye(4), "dense/sparse", 2, 0.4, 2, 300)
                torch.cuda.synchronize()
                res["gt_reproject_error_s"] = time.perf_counter() - t0
            r = R.track_errors(d, gp, np.eye(4), "dense/sparse", 2, 0.4, 300)
        finally:
            os.chdir(cwd)
    res["loss"] = loss
    res["n_tracks"] = len(r["track_point_ids"])
    res["n_obs"] = int(r["n_obs"])
    res["n_tracks_without_hit"] = int((r["gt_index"] < 0).sum())

    # kernel timings on the same queries
    Ks, _, Es = sc["views"]
    kept = list(r["kept_views"])
    qv = r["ref_view"].astype(np.int32)
    qxy = r["ref_xy"].astype(np.float32)
    L = _lib.lib()
    pts = torch.as_tensor(sc["gt"], device="cuda")
    views = np.stack([R._view_row(Ks[i - 1], Es[i - 1]) for i in kept])
    pix = np.rint(qxy).astype(np.int64)
    boxes = np.zeros((len(kept), 4), np.int64)
    for v in np.unique(qv):
        p = pix[qv == v]
        boxes[v] = *p.min(0), *(p.max(0) - p.min(0) + 1)
    area = boxes[:, 2] * boxes[:, 3]
    map_px = min(int(area.sum()), max(int(area.max()), R.MAP_PIXELS))
    nbytes = L.nrw_first_hit_scratch_bytes(len(qv), map_px)
    owner, scratch = _scratch(nbytes, torch.device("cuda"))
    hit = torch.empty(len(qv), dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    q_view, q_xy = torch.as_tensor(qv, device="cuda"), torch.as_tensor(qxy, device="cuda")
    cv = (C.c_double * views.size)(*views.reshape(-1).tolist())
    cb = (C.c_int * boxes.size)(*boxes.reshape(-1).tolist())
    ms = _events(lambda: check(L.nrw_first_hit(ptr(pts), pts.shape[0], cv, cb, len(kept), ptr(q_view), ptr(q_xy), len(qv),
                                               ptr(hit), ptr(status), scratch, nbytes, stream_ptr()), "nrw_first_hit"),
                 args.reps)
    assert np.array_equal(hit.cpu().numpy(), r["gt_index"])
    n_pass = -(-len(kept) // 16)
    res["first_hit_ms"] = ms
    res["first_hit_passes"] = n_pass
    res["first_hit_ms_per_pass"] = ms / n_pass
    res["first_hit_ms_per_view"] = ms / len(kept)
    res["point_load_bound_share"] = (12 * args.points / HBM_BYTES_PER_S) / (ms / n_pass / 1e3)
    Pm = np.array([R._projection(Ks[i - 1], Es[i - 1]) for i in kept])
    X = torch.as_tensor(np.asarray(sc["gt"], np.float64)[r["gt_index"][r["obs_track"]]], device="cuda")
    ov = torch.as_tensor(np.array([kept.index(i) for i in r["obs_image_id"]], np.int32), device="cuda")
    oxy = torch.as_tensor(r["obs_xy"], device="cuda")
    P = torch.as_tensor(Pm.reshape(-1, 12), device="cuda")
    err = torch.empty(len(ov), dtype=torch.float64, device="cuda")
    res["obs_error_ms"] = _events(lambda: check(L.nrw_obs_reproj_error(ptr(X), ptr(ov), ptr(oxy), len(ov), ptr(P), len(kept),
                                                                       ptr(err), None, stream_ptr()), "nrw_obs_reproj_error"),
                                  args.reps)

    # the unmodified reference's get_gt_point on the GPU, a sample of tracks, extrapolated
    from oracle import ref_import

    if ref_import.available():
        from oracle import trackerr_port as tp

        ref = tp.load_reference()
        gt = torch.as_tensor(sc["gt"], device="cuda")
        n = min(args.ref_tracks, len(qv)) // 2 * 2
        cam2gt = torch.as_tensor(np.stack([np.linalg.inv(Es[kept[v] - 1]) for v in qv[:n]]), device="cuda").float()
        K = torch.as_tensor(np.stack([Ks[kept[v] - 1] for v in qv[:n]]), device="cuda").float()
        t2d = torch.as_tensor(np.c_[np.zeros((n, 2)), r["ref_xy"][:n]], device="cuda").float()
        with contextlib.redirect_stdout(io.StringIO()):
            ref.get_gt_point(gt, cam2gt[:2], K[:2], t2d[:2])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(0, n, 2):
                ref.get_gt_point(gt, cam2gt[i:i + 2], K[i:i + 2], t2d[i:i + 2])
            torch.cuda.synchronize()
        per = (time.perf_counter() - t0) / n
        res["reference_get_gt_point_s_per_track"] = per
        res["reference_get_gt_point_s_all_tracks_extrapolated"] = per * res["n_tracks"]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "reproj_error_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
