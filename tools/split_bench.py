"""Times the scene split: the device time of one ROI launch over many views (CUDA events, median of repeated launches),
the static-label count per semantic map (CUDA events, median), and an end-to-end run on a seeded on-disk scene of JPEG
images: `python -m nrw.prepare_data_split` (as a process, and prepare() inside this one) next to the unmodified
reference prepare_data_split.py run with torch on the same GPU.  Writes one JSON file under --out with the card name and
power limit read in the same run.

    python tools/split_bench.py --views 1500 --width 1600 --height 1200 --scene_views 200 --out split_bench_out
"""
import argparse
import contextlib
import ctypes
import io
import json
import os
import runpy
import shutil
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "neuralrecon-w_b200")
for p in (ROOT, PKG, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return f"unknown ({e})"


def median_ms(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    fn()
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def ring_views(n, W, H, rng):
    """view table rows of n cameras on a ring around the origin looking near it, focal lengths from 0.5 W to 3 W"""
    rows = []
    for i in range(n):
        ang = 2 * np.pi * i / n
        C = np.array([4 * np.cos(ang), 4 * np.sin(ang), 0.5 + 0.2 * rng.standard_normal()])
        f = -(C - rng.normal(0, 0.3, 3))
        f /= np.linalg.norm(f)
        r = np.cross(f, [0, 0, 1.0])
        r /= np.linalg.norm(r)
        c2w = np.stack([r, np.cross(f, r), f], 1)
        c2w[:, 1:3] *= -1
        fx = rng.uniform(0.5, 3.0) * W
        rows.append(np.concatenate([[fx, fx * 1.01, W / 2, H / 2], np.concatenate([c2w, C[:, None]], 1).reshape(-1)]))
    return np.array(rows, np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=1500)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scene_views", type=int, default=200)
    ap.add_argument("--scene_width", type=int, default=1024)
    ap.add_argument("--scene_height", type=int, default=768)
    ap.add_argument("--out", default="split_bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("split_bench needs a CUDA device")
    import util_split
    from nrw import _lib
    from nrw.prepare_data_split import TRANSIENT_OBJECTS, get_opts, prepare
    from nrw.renderer import LABEL_IDS
    from oracle import split_port as sp

    out = os.path.abspath(a.out)
    os.makedirs(out, exist_ok=True)
    L, dev, rng = _lib.lib(), torch.device("cuda", 0), np.random.default_rng(0)
    res = {"card": card(), "torch": torch.__version__}

    # one ROI launch over all views
    V = torch.from_numpy(ring_views(a.views, a.width, a.height, rng)).to(dev)
    HW = torch.tensor([[a.height, a.width]] * a.views, dtype=torch.int32, device=dev)
    counts = torch.empty(a.views, dtype=torch.int64, device=dev)
    o = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    roi = lambda: _lib.check(L.nrw_view_roi_count(_lib.ptr(V), _lib.ptr(HW), a.views, a.height * a.width, o, 1.0,  # noqa: E731
                                                  _lib.ptr(counts), _lib.stream_ptr()), "nrw_view_roi_count")
    t_roi = median_ms(roi, a.reps)
    px = a.views * a.width * a.height
    c = counts.cpu().numpy()
    k = int(np.argmin(np.abs(c / (a.width * a.height) - 0.5)))
    exact = int(sp.roi_counts(V[k:k + 1].cpu().numpy(), [(a.height, a.width)], [0, 0, 0], 1.0)[0]) == int(c[k])
    res["roi"] = {"views": a.views, "size": [a.width, a.height], "ms_per_launch": t_roi, "gpix_per_s": px / t_roi / 1e6,
                  "median_share": float(np.median(c / (a.width * a.height))), "port_equal_on_one_view": exact}

    # static-label count per map
    lab = torch.from_numpy(rng.integers(0, 150, a.width * a.height).astype(np.float32)).to(dev)
    acc = torch.zeros(1, dtype=torch.int64, device=dev)
    ids = (ctypes.c_int * len(TRANSIENT_OBJECTS))(*[LABEL_IDS[t] for t in TRANSIENT_OBJECTS])
    lbl = lambda: _lib.check(L.nrw_label_static_count(_lib.ptr(lab), lab.numel(), ids, len(ids), _lib.ptr(acc),  # noqa: E731
                                                      _lib.stream_ptr()), "nrw_label_static_count")
    res["label_count"] = {"pixels": a.width * a.height, "ms_per_map": median_ms(lbl, a.reps)}

    # end to end on an on-disk scene
    cams = [("ring", a.scene_width, a.scene_height, float(f)) for f in rng.uniform(0.5, 3.0, a.scene_views)]
    src = os.path.join(out, "scene_src", "bench_scene")
    shutil.rmtree(os.path.dirname(src), ignore_errors=True)
    t0 = time.perf_counter()
    util_split.write_scene(src, seed=1, cameras=cams, ext="jpg")
    res["scene"] = {"views": a.scene_views, "size": [a.scene_width, a.scene_height], "write_s": time.perf_counter() - t0}
    flags = ["--num_test", "10", "--roi_threshold", "0.2", "--static_threshold", "0.5"]
    runs = {}
    for kind in ("cli", "in_process", "reference"):
        root = os.path.join(out, kind, "bench_scene")
        shutil.rmtree(os.path.dirname(root), ignore_errors=True)
        shutil.copytree(src, root)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if kind == "cli":
            env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
            r = subprocess.run([sys.executable, "-s", "-m", "nrw.prepare_data_split", "--root_dir", root] + flags, env=env,
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(r.stderr[-3000:])
        elif kind == "in_process":
            prepare(get_opts(["--root_dir", root] + flags))
        else:
            R = sp.load_split_ref()
            old = sys.argv
            sys.argv = ["prepare_data_split.py", "--root_dir", root] + flags
            try:
                np.random.seed(0)
                with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                    runpy.run_path(R.script, run_name="__main__")
            finally:
                sys.argv = old
        torch.cuda.synchronize()
        runs[kind] = time.perf_counter() - t0
        runs[kind + "_tsv"] = open(os.path.join(root, "bench_scene.tsv"), "rb").read()
    res["e2e_s"] = {k: runs[k] for k in ("cli", "in_process", "reference")}
    res["e2e_tsv_equal_to_reference"] = runs["cli_tsv"] == runs["reference_tsv"] == runs["in_process_tsv"]
    res["e2e_rows"] = len(runs["cli_tsv"].splitlines()) - 1
    for kind in ("scene_src", "cli", "in_process", "reference"):
        shutil.rmtree(os.path.join(out, kind), ignore_errors=True)
    with open(os.path.join(out, "split_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
