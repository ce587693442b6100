"""GPU: the point-cloud visibility filter (csrc/voxelvis.cu, nrw.reprojection.VoxelRenderer / reproj_filter_points) bit
for bit against the restatement oracle/voxelvis_port.py, the pruned first-hit walk against the unpruned training
traversal (nrw_octree_near_far), the reference's get_index, view-order independence and repeatability, the error
cases, and `python -m nrw.reprojection --point_source` end to end (then `python -m nrw.evaluation` on its output)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from oracle import octree_port as op
from oracle import ref_import
from oracle import voxelvis_port as vp
from util_reproj import look_at, two_sphere_mesh, view_matrix, write_scene

pytestmark = pytest.mark.gpu

CFG = {"sfm2gt": np.eye(4).tolist(), "eval_bbx": [[-2.0, -2.0, -4.0], [2.0, 2.0, 2.0]]}
VOXEL = 0.03


@pytest.fixture(scope="module")
def cloud():
    verts, _, which = two_sphere_mesh(h=0.06)
    tree, origin, scale, level, _ = op.gen_octree(CFG, verts, VOXEL, expand=0, in_sfm=False)
    return verts, which, tree, origin, scale, level


def _K(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


def _cameras(verts):
    """(name, K, world_to_cam 4x4, (width, height))"""
    rng = np.random.default_rng(41)
    cams = []
    for k in range(3):
        th, ph = np.deg2rad(rng.uniform(0, 70)), rng.uniform(0, 2 * np.pi)
        eye = rng.uniform(3.0, 5.0) * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        R, t = look_at(eye, rng.normal(size=3) * 0.2, up=(rng.normal() * 0.2, 1.0, 0.0))
        cams.append((f"random{k}", _K(70.3, 69.8, 32.25, 23.6), view_matrix(R, t), (64, 48)))
    # axis-aligned cameras with integer principal points: exact rotations, direction components that are 0 before the
    # +1e-7, and rays along the voxel faces x = 0, y = 0 (the cube's centre is (0, 0, -1))
    R, t = look_at((0.0, 0.0, 5.0), (0.0, 0.0, 0.0))
    cams.append(("axis_z", _K(32.0, 32.0, 32.0, 24.0), view_matrix(R, t), (65, 49)))
    R, t = look_at((4.0, 0.0, -1.0), (0.0, 0.0, -1.0))
    cams.append(("axis_x", _K(16.0, 16.0, 20.0, 15.0), view_matrix(R, t), (41, 31)))
    R, t = look_at(verts[17], verts[17] + np.array([0.3, 0.2, 1.0]))      # inside an occupied voxel
    cams.append(("inside", _K(30.0, 30.0, 16.0, 12.0), view_matrix(R, t), (32, 24)))
    R, t = look_at((0.0, 0.0, 5.0), (0.0, 0.0, 10.0))                     # sees nothing
    cams.append(("away", _K(30.0, 30.0, 16.0, 12.0), view_matrix(R, t), (32, 24)))
    return cams


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def test_cast_and_lookup_match_oracle(cloud):
    from nrw.reprojection import VoxelRenderer

    verts, _, tree, origin, scale, level = cloud
    r = VoxelRenderer(verts, CFG, VOXEL, device=0)
    assert r.level == level and r.n_leaf == len(tree["levels"][level])
    assert np.array_equal(r.tree["octree"].cpu().numpy(), tree["octree"])
    visible = np.zeros(r.n_leaf, bool)
    n_hit = 0
    for name, K, E, (w, h) in _cameras(verts):
        depth, leaf = r(h, w, K, E)
        want_d, want_l = vp.cast(tree, level, origin, scale, h, w, K, np.linalg.inv(E))
        assert _same(leaf.cpu().numpy(), want_l), (name, int((leaf.cpu().numpy() != want_l).sum()))
        assert _same(depth.cpu().numpy(), want_d), name
        visible[want_l[want_l >= 0]] = True
        n_hit += int((want_l >= 0).sum())
        if name in ("inside", "away"):
            assert np.all(want_l == -1), name
        else:
            assert (want_l >= 0).mean() > 0.02, name
    assert np.array_equal(r.visible.cpu().numpy().astype(bool), visible)
    assert int(r.n_hit.item()) == n_hit
    lf, _ = vp.lookup(tree, level, (verts - origin) / scale)
    assert np.array_equal(r.point_leaves().cpu().numpy(), lf) and int(r.status.item()) == 0


def test_pruned_walk_equals_the_training_traversal(cloud):
    """leaf and depth equal nrw_octree_near_far (the unpruned walk) fed with the oracle's fp32 rays"""
    from nrw import _lib
    from nrw.reprojection import VoxelRenderer

    verts, _, tree, origin, scale, level = cloud
    r = VoxelRenderer(verts, CFG, VOXEL, device=0)
    L = _lib.lib()
    for name, K, E, (w, h) in _cameras(verts):
        o, d, n = vp.gen_rays(h, w, K, np.linalg.inv(E))
        ro, rd = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (o, d))
        R = ro.shape[0]
        near, far = (torch.empty(R, device="cuda") for _ in range(2))
        pid, cnt = (torch.empty(R, dtype=torch.int32, device="cuda") for _ in range(2))
        org = (C.c_float * 3)(*np.asarray(origin, np.float64).tolist())
        _lib.check(L.nrw_octree_near_far(_lib.ptr(r.tree["octree"]), _lib.ptr(r.tree["prefix"]), r._pyr, level,
                                         _lib.ptr(ro), _lib.ptr(rd), R, org, scale, _lib.ptr(near), _lib.ptr(far),
                                         _lib.ptr(pid), _lib.ptr(cnt), _lib.stream_ptr()), "nrw_octree_near_far")
        base = int(tree["pyramid"][1, level])
        want_l = torch.where(pid >= 0, pid - base, -1).cpu().numpy().reshape(h, w)
        want_d = (near / torch.from_numpy(n).cuda()).cpu().numpy().reshape(h, w)
        depth, leaf = r(h, w, K, E)
        assert _same(leaf.cpu().numpy(), want_l), name
        assert _same(depth.cpu().numpy(), want_d), name


@pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")
def test_reference_get_index_keeps_the_same_points(cloud, tmp_path):
    import yaml

    from nrw.reprojection import VoxelRenderer, reproj_filter_points

    verts = cloud[0]
    with open(tmp_path / "config.yaml", "w") as fh:
        yaml.safe_dump(CFG, fh)
    kr = vp.load_kaolin_renderer()
    ref = kr.kaolin_renderer(str(tmp_path), verts, VOXEL, device="cpu")
    cams = [c for c in _cameras(verts) if c[0].startswith("random")]
    Ks, Es, whs = [c[1] for c in cams], [c[2] for c in cams], [c[3] for c in cams]
    r = VoxelRenderer(verts, CFG, VOXEL, device=0)
    for K, E, (w, h) in zip(Ks, Es, whs):
        r(h, w, K, E)
    # the reference's get_index over our marked leaves (without the marks deviation 1 adds for missed pixels)
    kept = ref.get_index(r.visible.cpu().numpy().astype(bool))
    mask = reproj_filter_points(verts, CFG, Ks, Es, whs, voxel_size=VOXEL)
    assert np.array_equal(np.sort(kept), np.nonzero(mask)[0]) and 0 < mask.sum() < len(mask)


def test_mask_order_independent_and_repeatable(cloud):
    from nrw.reprojection import reproj_filter_points

    verts, _, tree, origin, scale, level = cloud
    cams = _cameras(verts)
    Ks, Es, whs = [c[1] for c in cams], [c[2] for c in cams], [c[3] for c in cams]
    a = reproj_filter_points(verts, CFG, Ks, Es, whs, voxel_size=VOXEL)
    b = reproj_filter_points(verts, CFG, Ks[::-1], Es[::-1], whs[::-1], voxel_size=VOXEL)
    c = reproj_filter_points(verts, CFG, Ks, Es, whs, voxel_size=VOXEL)
    want, _, _ = vp.filter_points(verts, CFG, Ks, Es, whs, VOXEL)
    assert np.array_equal(a, want) and np.array_equal(a, b) and np.array_equal(a, c) and 0 < a.sum() < len(a)


def test_errors(cloud):
    from nrw._lib import NrwError
    from nrw.reprojection import VoxelRenderer, reproj_filter_points

    verts = cloud[0]
    bad = verts.copy()
    bad[5, 2] = np.inf
    with pytest.raises(NrwError, match="finite"):
        VoxelRenderer(bad, CFG, VOXEL)
    with pytest.raises(NrwError, match="level"):
        VoxelRenderer(verts, CFG, 10.0)                     # level 0
    with pytest.raises(NrwError, match="level"):
        VoxelRenderer(verts, CFG, 1e-5)                     # level 19
    with pytest.raises(NrwError, match="no source point"):
        VoxelRenderer(verts + 100.0, CFG, VOXEL)
    R, t = look_at((0.0, 0.0, 5.0), (0.0, 0.0, 10.0))
    with pytest.raises(NrwError, match="no view"):
        reproj_filter_points(verts, CFG, [_K(30, 30, 16, 12)] * 2, [view_matrix(R, t)] * 2, [(32, 24)] * 2, VOXEL)


def _write_pc(path, xyz, colors):
    from nrw.mesh import write_ply

    write_ply(path, xyz, colors=colors)


def test_cli_point_source_end_to_end(tmp_path):
    from nrw._lib import NrwError
    from nrw.colmap import read_cameras, read_images
    from nrw.mesh import read_ply, write_ply
    from nrw.reprojection import get_entrinsics, get_image_id, get_intrinsic, get_train_ids, main

    d = str(tmp_path / "scene")
    S = write_scene(d, seed=43)
    verts, _, which = two_sphere_mesh(h=0.06)
    rng = np.random.default_rng(44)
    colors = rng.integers(0, 256, (len(verts), 3)).astype(np.uint8)
    src = str(tmp_path / "points.ply")
    _write_pc(src, verts, colors)
    out = str(tmp_path / "out")
    voxel = 0.2
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    probe = ("import runpy, sys; sys.argv = ['reprojection'] + sys.argv[1:]; runpy.run_module('nrw.reprojection', "
             "run_name='__main__'); bad = [m for m in ('pyrender', 'open3d', 'trimesh', 'ray', 'kaolin') "
             "if m in sys.modules]; assert not bad, bad")
    cmd = [sys.executable, "-s", "-c", probe, "--src_file", src, "--target_file", src, "--data_path", d, "--output_path",
           out, "--voxel_size", str(voxel), "--point_source"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    res = read_ply(f"{out}/reprojected.ply")
    with open(f"{out}/reprojected.ply", "rb") as fh:
        assert b"property double x" in fh.read(400)

    # the oracle pipeline from the same files
    m = read_ply(src)
    vv = np.asarray(m["vertices"], np.float64)
    v_gt = (S[:3] @ np.concatenate((vv, np.ones((vv.shape[0], 1))), axis=-1).T).T
    sparse = os.path.join(d, "dense", "sparse")
    im, cams = read_images(os.path.join(sparse, "images.bin")), read_cameras(os.path.join(sparse, "cameras.bin"))
    _, _, p2i = get_image_id(im, d)
    ids = get_train_ids(d, None, p2i)
    Ks, whs = get_intrinsic(cams, ids, im)
    Es = get_entrinsics(im, ids) @ np.linalg.inv(S)
    import yaml

    cfg = yaml.safe_load(open(os.path.join(d, "config.yaml")))
    rows = vp.pipeline(v_gt, v_gt, m["colors"].astype(np.float64) / 255.0, cfg, [Ks[k] for k in ids], Es,
                       [whs[k] for k in ids], voxel_size=voxel)
    assert np.array_equal(res["vertices"], rows[:, :3])
    assert np.array_equal(res["colors"], np.round(rows[:, 3:] * 255).astype(np.uint8))

    # independent of the oracle: the occluded sphere is never kept, the near cap of the visible one mostly is
    index = {tuple(p): i for i, p in enumerate(v_gt)}
    kept = np.array([index[tuple(p)] for p in res["vertices"]])
    assert len(kept) > 100
    assert not np.any(which[kept] == 1)
    near = (which == 0) & (verts[:, 2] > 0.6)
    assert near[kept].sum() > 0.5 * near.sum()

    # then the evaluation reads the filtered cloud
    write_ply(str(tmp_path / "gt.ply"), v_gt[which == 0])
    cmd = [sys.executable, "-s", "-m", "nrw.evaluation", "--file_pred", f"{out}/reprojected.ply", "--file_trgt",
           str(tmp_path / "gt.ply"), "--scene_config_path", f"{d}/config.yaml", "--threshold", "0.05,0.1,0.15,0.2",
           "--save_name", "reproj"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    j = json.load(open(f"{out}/eval_reproj/metrics.json"))
    assert len(j["precs"]) == 4 and j["precs"][-1] > 0.9

    # a target with another point count is refused
    other = str(tmp_path / "other.ply")
    _write_pc(other, verts[:-1], colors[:-1])
    with pytest.raises(NrwError, match="point count|points and the source"):
        main(["--src_file", src, "--target_file", other, "--data_path", d, "--output_path", out, "--point_source"])
