"""GPU: the depth rasteriser and the back-projection marking (csrc/raster.cu, nrw.reprojection) bit for bit against the
restatement oracle/reproj_port.py, run-to-run repeatability, the face-index status bit, and `python -m nrw.reprojection`
end to end on a synthetic COLMAP scene (then `python -m nrw.evaluation` on its output)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from oracle import reproj_port as rp
from util_reproj import look_at, sdf_spheres, soup, two_sphere_mesh, view_matrix, write_scene

pytestmark = pytest.mark.gpu


def _gpu_depth(v, f, V, fx, fy, cx, cy, H, W, znear=0.05, zfar=100.0, cull=True):
    from nrw.reprojection import DepthRenderer

    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    return DepthRenderer(v, f, znear, zfar, cull, device=0)(H, W, K, V).cpu().numpy()


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _random_view(rng, spread=0.3):
    R, t = look_at(rng.normal(size=3) * spread, np.array([0.0, 0.0, 3.0]) + rng.normal(size=3) * spread,
                   up=(rng.normal() * 0.2, 1.0, 0.0))
    return view_matrix(R, t)[:3]


def _soup_cases():
    rng = np.random.default_rng(11)
    cases = []
    for i, (H, W) in enumerate([(1, 1), (7, 13), (48, 64), (31, 17)]):
        v, f = soup(rng, 400, spread=1.5, depth=(-1.5, 6.0))        # faces behind the camera and across z = znear
        cases.append((f"soup{i}_{H}x{W}", v, f, _random_view(rng), (H, W)))
    # degenerate faces: repeated indices, coincident and collinear vertices, zero-area slivers on a shared vertex
    v, f = soup(rng, 200, spread=1.0, depth=(1.0, 4.0))
    n = len(v)
    extra_v = np.concatenate([v[:10], (v[10:20] + v[20:30]) / 2])
    v = np.concatenate([v, extra_v])
    deg = [[0, 0, 1], [2, 3, 3], [4, 5, 4], [0, n, 1], [2, 3, n + 2]] + [[10 + k, n + 10 + k, 20 + k] for k in range(10)]
    f = np.concatenate([f, np.array(deg)])
    cases.append(("degenerate", v, f, np.eye(4)[:3], (40, 50)))
    # faces covering the whole screen: in front, crossing z = 0, and with one vertex behind the camera
    v = np.array([[-50, -50, 2], [50, -50, 2.5], [0, 80, 3], [-50, -50, -1], [60, -40, 4], [0, 70, 0.01],
                  [-3, -3, -2], [3, -3, 5], [0, 4, 5]], np.float64)
    f = np.array([[0, 2, 1], [0, 1, 2], [3, 5, 4], [3, 4, 5], [6, 8, 7], [6, 7, 8]])
    cases.append(("fullscreen", v, f, np.eye(4)[:3], (33, 45)))
    return cases


@pytest.mark.parametrize("name,v,f,V,hw", _soup_cases(), ids=lambda x: x if isinstance(x, str) else None)
@pytest.mark.parametrize("cull", [True, False])
def test_depth_matches_oracle(name, v, f, V, hw, cull):
    H, W = hw
    cam = (37.3, 35.9, W / 2 + 0.3, H / 2 - 0.2)
    want, _ = rp.raster_depth(v, f, V, *cam, H, W, cull=cull, box=False)
    got = _gpu_depth(v, f, V, *cam, H, W, cull=cull)
    assert _same(got, want), (name, int((got != want).sum()))
    if name.startswith("soup") and H * W > 100:
        assert (got > 0).sum() > 0


def _grid(n, z, fx, cx, rng):
    """an n x n vertex grid on the plane z whose vertices project exactly onto pixel centres (dyadic arithmetic),
    triangulated with random diagonals and randomly permuted vertex ids, so that rays run along shared edges and
    through vertices"""
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    xy = ((ij * 2 + 0.5) - cx) / fx * z
    v = np.concatenate([xy, np.full((len(xy), 1), z)], 1)
    perm = rng.permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    v = v[perm]
    faces = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            if rng.random() < 0.5:
                faces += [[a, c, b], [a, d, c]]
            else:
                faces += [[a, d, b], [b, d, c]]
    return v, inv[np.array(faces)]


@pytest.mark.parametrize("cull", [True, False])
def test_depth_on_exact_shared_edges(cull):
    rng = np.random.default_rng(12)
    fx, cx = 16.0, 8.0
    v, f = _grid(9, 2.0, fx, cx, rng)
    V = np.eye(4)[:3]
    for H, W in [(20, 20), (17, 19)]:
        want, _, cnt = rp.raster_depth(v, f, V, fx, fx, cx, cx, H, W, cull=cull, box=False, counts=True)
        got = _gpu_depth(v, f, V, fx, fx, cx, cx, H, W, cull=cull)
        assert _same(got, want)
        # every pixel centre inside the grid and off its vertices is covered exactly once
        r, c = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        inner = (c >= 1) & (c <= 15) & (r >= 1) & (r <= 15) & ~((c % 2 == 0) & (r % 2 == 0))
        inner &= (c < W) & (r < H)
        assert np.all(cnt[inner] == 1)


def test_depth_large_view_matches_oracle_and_repeats():
    from nrw.mesh import marching_cubes

    vol, lo, h = sdf_spheres([(0, 0, 0), (0.9, 0.3, -0.6)], [1.0, 0.6], (-1.3, -1.3, -1.4), (1.8, 1.3, 1.3), 0.012)
    vt, ft, _ = marching_cubes(torch.from_numpy(vol).cuda())
    v = lo + h * vt.double().cpu().numpy()
    f = ft.long().cpu().numpy()
    assert len(f) >= 100_000
    R, t = look_at((0.7, -1.1, 3.4), (0.2, 0.0, 0.0))
    V = view_matrix(R, t)[:3]
    H, W = 750, 1000
    cam = (900.0, 905.0, 500.3, 374.6)
    want, _ = rp.raster_depth(v, f, V, *cam, H, W, cull=True)
    from nrw.reprojection import DepthRenderer

    r = DepthRenderer(v, f, device=0)
    K = np.array([[cam[0], 0, cam[2]], [0, cam[1], cam[3]], [0, 0, 1]])
    a = r(H, W, K, V).cpu().numpy()
    b = r(H, W, K, V).cpu().numpy()
    assert _same(a, want) and _same(a, b) and (a > 0).mean() > 0.2


def test_face_index_status_bit():
    from nrw import _lib
    from nrw.evaluation import _scratch

    L = _lib.lib()
    rng = np.random.default_rng(13)
    v, f = soup(rng, 50, depth=(1.0, 4.0))
    f_bad = f.copy()
    f_bad[7] = [0, len(v), 1]
    f_bad[9] = [-1, 2, 3]
    vt = torch.from_numpy(v).cuda()
    depth = torch.empty(20, 30, dtype=torch.float32, device="cuda")
    status = torch.full((1,), 99, dtype=torch.int32, device="cuda")
    V = (C.c_double * 12)(*np.eye(4)[:3].reshape(-1).tolist())
    for faces, st in ((f_bad, 1), (f, 0)):
        ft = torch.from_numpy(faces).cuda()
        _, sp = _scratch(L.nrw_raster_scratch_bytes(len(v), len(faces), 20, 30), vt.device)
        assert L.nrw_raster_depth(_lib.ptr(vt), len(v), _lib.ptr(ft), len(faces), V, 20.0, 20.0, 15.0, 10.0, 20, 30, 0.05, 100.0,
                                  1, _lib.ptr(depth), _lib.ptr(status), sp, _lib.stream_ptr()) == 0
        assert int(status.item()) == st
        want, bad = rp.raster_depth(v, faces, np.eye(4)[:3], 20.0, 20.0, 15.0, 10.0, 20, 30, box=False)
        assert bad == bool(st) and _same(depth.cpu().numpy(), want)
    from nrw._lib import NrwError
    from nrw.reprojection import DepthRenderer

    with pytest.raises(NrwError, match="outside"):
        DepthRenderer(v, f_bad, device=0)
    with pytest.raises(NrwError, match="no faces"):
        DepthRenderer(v, f[:0], device=0)
    v_nan = v.copy()
    v_nan[3, 1] = np.nan
    with pytest.raises(NrwError, match="finite"):
        DepthRenderer(v_nan, f, device=0)


def _views(rng, n, S):
    Ks, Es, whs = [], [], []
    for _ in range(n):
        th, ph = np.deg2rad(rng.uniform(0, 40)), rng.uniform(0, 2 * np.pi)
        eye = rng.uniform(3.5, 6.0) * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        R, t = look_at(eye, rng.normal(size=3) * 0.2)
        Es.append(view_matrix(R, t) @ np.linalg.inv(S))
        w, h = int(rng.integers(40, 90)), int(rng.integers(30, 70))
        Ks.append(np.array([[70.3, 0, w / 2 + 0.25], [0, 69.8, h / 2 - 0.4], [0, 0, 1]], dtype=np.float32))
        whs.append((w, h))
    return Ks, np.array(Es), whs


def test_visibility_mask_matches_oracle():
    from nrw.reprojection import reproj_filter
    from util_reproj import similarity

    verts, faces, _ = two_sphere_mesh(h=0.08)
    S = similarity(5, 1.7)
    v_gt = (S[:3] @ np.concatenate([verts, np.ones((len(verts), 1))], 1).T).T
    rng = np.random.default_rng(14)
    target = v_gt + rng.normal(0, 0.02, v_gt.shape)
    Ks, Es, whs = _views(rng, 5, S)
    for voxel in (0.01, 0.04):
        got = reproj_filter(v_gt, faces, target, Ks, Es, whs, voxel_size=voxel)
        want = np.zeros(len(target), bool)
        for K, E, (w, h) in zip(Ks, Es, whs):
            fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
            d, _ = rp.raster_depth(v_gt, faces, E, fx, fy, cx, cy, h, w)
            rp.mark(want, target, rp.backproject(d, fx, fy, cx, cy, np.linalg.inv(E)), 2 * np.sqrt(2) * voxel)
        assert np.array_equal(got, want) and 0 < got.sum() < len(got)
    from nrw._lib import NrwError

    away = np.array([view_matrix(*look_at((0, 0, 10), (0, 0, 20))) for _ in range(2)])
    with pytest.raises(NrwError, match="no view"):
        reproj_filter(v_gt, faces, target, Ks[:2], away, whs[:2])


def test_cli_end_to_end(tmp_path):
    from nrw.mesh import read_ply, write_ply
    from nrw.reprojection import get_entrinsics, get_intrinsic, get_image_id, get_train_ids
    from nrw.colmap import read_cameras, read_images

    d = str(tmp_path / "scene")
    S = write_scene(d, seed=21)
    verts, faces, which = two_sphere_mesh(h=0.06)
    rng = np.random.default_rng(22)
    colors = rng.integers(0, 256, (len(verts), 3)).astype(np.uint8)
    mesh = str(tmp_path / "extracted_mesh.ply")
    write_ply(mesh, verts, faces, colors=colors)
    out = str(tmp_path / "out")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    probe = ("import runpy, sys; sys.argv = ['reprojection'] + sys.argv[1:]; runpy.run_module('nrw.reprojection', "
             "run_name='__main__'); bad = [m for m in ('pyrender', 'open3d', 'trimesh', 'ray') if m in sys.modules]; "
             "assert not bad, bad")
    cmd = [sys.executable, "-s", "-c", probe, "--src_file", mesh, "--target_file", mesh, "--data_path", d, "--output_path",
           out, "--voxel_size", "0.03", "--n_cpus", "4", "--n_gpus", "4"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    res = read_ply(f"{out}/reprojected.ply")
    with open(f"{out}/reprojected.ply", "rb") as fh:
        assert b"property double x" in fh.read(400)

    # the oracle pipeline from the same files
    m = read_ply(mesh)
    vv = np.asarray(m["vertices"], np.float64)
    homo = np.concatenate((vv, np.ones((vv.shape[0], 1))), axis=-1).T
    v_gt = (S[:3] @ homo).T
    sparse = os.path.join(d, "dense", "sparse")
    im, cams = read_images(os.path.join(sparse, "images.bin")), read_cameras(os.path.join(sparse, "cameras.bin"))
    _, _, p2i = get_image_id(im, d)
    ids = get_train_ids(d, None, p2i)
    Ks, whs = get_intrinsic(cams, ids, im)
    Es = get_entrinsics(im, ids) @ np.linalg.inv(S)
    rows = rp.pipeline(v_gt, m["faces"], v_gt, m["colors"].astype(np.float64) / 255.0, [Ks[k] for k in ids], Es,
                       [whs[k] for k in ids], voxel_size=0.03)
    assert np.array_equal(res["vertices"], rows[:, :3])
    assert np.array_equal(res["colors"], np.round(rows[:, 3:] * 255).astype(np.uint8))

    # independent of the oracle: the hidden sphere and the far half of the visible one are never kept
    index = {tuple(p): i for i, p in enumerate(v_gt)}
    kept = np.array([index[tuple(p)] for p in res["vertices"]])
    assert len(kept) > 100
    assert not np.any(which[kept] == 1)
    assert not np.any(verts[kept, 2] < 0.0)
    near = (which == 0) & (verts[:, 2] > 0.6)
    assert near[kept].sum() > 0.3 * near.sum()

    # then the evaluation reads the filtered cloud
    write_ply(str(tmp_path / "gt.ply"), v_gt[which == 0])
    cmd = [sys.executable, "-s", "-m", "nrw.evaluation", "--file_pred", f"{out}/reprojected.ply", "--file_trgt",
           str(tmp_path / "gt.ply"), "--scene_config_path", f"{d}/config.yaml", "--threshold", "0.05,0.1,0.15,0.2",
           "--save_name", "reproj"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    j = json.load(open(f"{out}/eval_reproj/metrics.json"))
    assert len(j["precs"]) == 4 and j["precs"][-1] > 0.9


def test_cli_rejects_point_clouds_and_visualize(tmp_path):
    from nrw._lib import NrwError
    from nrw.mesh import write_ply
    from nrw.reprojection import main

    d = str(tmp_path / "scene")
    write_scene(d, seed=23)
    pc = str(tmp_path / "pc.ply")
    write_ply(pc, np.random.default_rng(0).normal(size=(50, 3)))
    args = ["--src_file", pc, "--target_file", pc, "--data_path", d, "--output_path", str(tmp_path / "o")]
    with pytest.raises(NrwError, match="no faces"):
        main(args)
    with pytest.raises(NrwError, match="visualize"):
        main(args + ["--visualize"])
