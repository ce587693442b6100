"""Mesh-extraction timings on one GPU, written as one JSON file (--out DIR/mesh_bench.json): marching_cubes (count,
one read-back, emit) on an analytic sphere at 512^3 and 1024^3, and extract_mesh at dim 512 on the synthetic network
split into SDF volume, marching cubes, vertex colours (with host copies) and PLY write.  CUDA events
around synchronised work; the card's name and power limit are read back with a read-only nvidia-smi query."""
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


def _timed(fn, reps):
    fn()                                                   # warm-up (module load, allocator)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, ms


def _sphere(n):
    a = torch.arange(n, device="cuda", dtype=torch.float32)
    c, R = (n - 1) / 2 + 0.3, 0.4 * n
    d2 = (a - c)[:, None, None] ** 2 + (a - c + 0.1)[None, :, None] ** 2 + (a - c - 0.2)[None, None, :] ** 2
    return d2.sqrt_().sub_(R)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="mesh_bench_out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dim", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench: needs a CUDA device")
    from nrw.mesh import _lib, extract_mesh, marching_cubes, sdf_volume
    from util_nrw import build_system, synth

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()}
    for n in (512, 1024):
        vol = _sphere(n)
        (v, f, _), ms = _timed(lambda: marching_cubes(vol), args.reps)
        res[f"mc_sphere_{n}"] = {"ms": ms, "median_ms": float(np.median(ms)), "verts": int(v.shape[0]), "faces": int(f.shape[0]),
                                 "volume_read_GB_per_s_at_2_reads": 2 * vol.numel() * 4 / (float(np.median(ms)) * 1e6),
                                 "scratch_bytes": int(_lib.lib().nrw_mc_scratch_bytes(n, n, n))}
        del vol, v, f
        torch.cuda.empty_cache()
    P = synth.make_params(seed=0)
    P["neuconw.sdf_net.lin8.bias"][0] -= 0.3           # the synthetic SDF is positive in the box: give it a surface
    r = build_system(P, synth.PathConfig(), precision="bf16x3", backend=0)["renderer"]
    dim = args.dim
    (vol, _, _), sdf_ms = _timed(lambda: sdf_volume(r, dim), 1)
    (v, f, _), mc_ms = _timed(lambda: marching_cubes(vol), args.reps)
    emb = torch.zeros(1, synth.PathConfig().n_a, device="cuda")
    t0 = time.perf_counter()
    torch.cuda.synchronize()
    full = extract_mesh(dim, 1 << 20, 1.0, [0.0, 0.0, 0.0], with_color=True, embedding_a=emb, chunk_rgb=1 << 16, renderer=r)
    torch.cuda.synchronize()
    total_s = time.perf_counter() - t0
    with tempfile.TemporaryDirectory() as td:
        t0 = time.perf_counter()
        full.export(os.path.join(td, "m.ply"))
        ply_s = time.perf_counter() - t0
    res[f"extract_mesh_{dim}"] = {
        "sdf_volume_ms": float(sdf_ms[0]), "marching_cubes_ms": mc_ms, "marching_cubes_median_ms": float(np.median(mc_ms)),
        "marching_cubes_share_of_sdf_volume": float(np.median(mc_ms)) / float(sdf_ms[0]),
        "extract_mesh_with_color_s": total_s, "ply_write_s": ply_s,
        # extract_mesh minus the separately timed SDF volume and marching cubes: vertex colours and host copies
        "colours_and_host_copies_s": total_s - (float(sdf_ms[0]) + float(np.median(mc_ms))) / 1e3,
        "verts": int(v.shape[0]), "faces": int(f.shape[0])}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "mesh_bench.json")
    with open(path, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
