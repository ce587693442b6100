"""CPU checks of the point-cloud visibility filter: the numpy restatement oracle/voxelvis_port.py against the unmodified
utils/kaolin_renderer.py (per-pixel first leaf, depth, vertex_table), each documented deviation from the reference on a
constructed input, the argument checks of the nrw_voxel_* exports and the --point_source flag."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import yaml

from oracle import octree_port as op
from oracle import ref_import
from oracle import voxelvis_port as vp
from util_reproj import look_at, two_sphere_mesh, view_matrix

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")


def _config(d, lo, hi):
    os.makedirs(d, exist_ok=True)
    cfg = {"sfm2gt": np.eye(4).tolist(), "eval_bbx": [list(map(float, lo)), list(map(float, hi))]}
    with open(os.path.join(d, "config.yaml"), "w") as fh:
        yaml.safe_dump(cfg, fh)
    return cfg


def _views(rng, n, H, W):
    Ks, Es = [], []
    for _ in range(n):
        th, ph = np.deg2rad(rng.uniform(0, 60)), rng.uniform(0, 2 * np.pi)
        eye = rng.uniform(4.0, 6.0) * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        R, t = look_at(eye, rng.normal(size=3) * 0.2, up=(rng.normal() * 0.2, 1.0, 0.0))
        Es.append(view_matrix(R, t))
        Ks.append(np.array([[60.3, 0, W / 2 + 0.3], [0, 59.7, H / 2 - 0.2], [0, 0, 1]], dtype=np.float32))
    return Ks, Es, [(W, H)] * n


@pytest.fixture(scope="module")
def kr():
    return vp.load_kaolin_renderer()


@needs_ref
def test_oracle_matches_kaolin_renderer(kr, tmp_path):
    verts, _, _ = two_sphere_mesh(h=0.08)
    cfg = _config(str(tmp_path), (-2.0, -2.0, -4.0), (2.0, 2.0, 2.0))
    voxel = 0.05
    ref = kr.kaolin_renderer(str(tmp_path), verts, voxel, device="cpu")
    tree, origin, scale, level, _ = op.gen_octree(cfg, verts, voxel, expand=0, in_sfm=False)
    assert level == ref.level and np.array_equal(tree["octree"], ref.octree.numpy())
    base = int(tree["pyramid"][1, level])
    assert int(ref.base_ind) == base and int(ref.voxel_num) == len(tree["levels"][level])

    # vertex_table
    lf, not_leaf = vp.lookup(tree, level, (verts - origin) / scale)
    assert not not_leaf and np.array_equal(ref.pt2vid.numpy(), lf.astype(np.int64))

    rng = np.random.default_rng(31)
    H, W = 48, 64
    Ks, Es, whs = _views(rng, 4, H, W)
    n_pix = n_bad = n_hit = 0
    for K, c2w, h, w in vp.views(Ks, Es, whs):
        _, depth_ref = ref(h, w, K, c2w)
        leaf_ref = np.where(ref.pids < 0, -1, ref.pids)
        depth, leaf = vp.cast(tree, level, origin, scale, h, w, K, c2w)
        same = leaf == leaf_ref
        n_pix += leaf.size
        n_bad += int((~same).sum())
        n_hit += int((leaf >= 0).sum())
        hit = same & (leaf >= 0)
        want = depth_ref.astype(np.float64) - 0.02
        assert np.all(np.abs(depth[hit] - want[hit]) <= 1e-5 * np.abs(want[hit]))
        assert np.all(depth[leaf < 0] == 0)
    assert n_bad <= 1e-4 * n_pix, (n_bad, n_pix)
    assert n_hit > 0.1 * n_pix


@needs_ref
def test_deviation_missed_pixels_mark_nothing(kr, tmp_path):
    """the reference marks leaf voxel_num - 1 - base_ind for every view with a miss (numpy negative indexing of pid - 1),
    or raises IndexError when base_ind >= voxel_num; a miss marks nothing here"""
    verts, _, _ = two_sphere_mesh(h=0.08)
    cfg = _config(str(tmp_path), (-2.0, -2.0, -4.0), (2.0, 2.0, 2.0))
    ref = kr.kaolin_renderer(str(tmp_path), verts, 0.05, device="cpu")
    R, t = look_at((0.0, 0.0, 6.0), (0.0, 0.0, 12.0))                  # looks away: every pixel misses
    E = view_matrix(R, t)
    K = np.array([[40.0, 0, 10.0], [0, 40.0, 8.0], [0, 0, 1]], np.float32)
    ref(16, 20, K, np.linalg.inv(E))
    indices_all = np.zeros(int(ref.voxel_num), bool)
    indices_all[ref.pids.reshape(-1)] = True                        # utils/reproj_filter.py's marking
    assert np.nonzero(indices_all)[0].tolist() == [int(ref.voxel_num) - 1 - int(ref.base_ind)]
    mask, n_hit, _ = vp.filter_points(verts, cfg, [K], [E], [(20, 16)], 0.05)
    assert n_hit == 0 and not mask.any()

    one = np.array([[0.3, 0.2, 0.1]])                                 # one leaf, base_ind = level >= voxel_num
    ref1 = kr.kaolin_renderer(str(tmp_path), one, 0.05, device="cpu")
    ref1(16, 20, K, np.linalg.inv(E))
    with pytest.raises(IndexError):
        np.zeros(int(ref1.voxel_num), bool)[ref1.pids.reshape(-1)] = True


@needs_ref
def test_deviation_points_outside_the_cube(kr, tmp_path):
    """vertex_table applies its cube mask twice, so any source point outside the cube raises; here it maps to -1"""
    cfg = _config(str(tmp_path), (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    pts = np.array([[0.5, 0.5, 0.5], [-0.25, 0.1, 0.7], [3.0, 0.0, 0.0], [0.2, -1.0, 0.0]])
    with pytest.raises(IndexError):
        kr.kaolin_renderer(str(tmp_path), pts, 0.25, device="cpu")
    tree, origin, scale, level, _ = op.gen_octree(cfg, pts, 0.25, expand=0, in_sfm=False)
    lf, not_leaf = vp.lookup(tree, level, (pts - origin) / scale)
    assert not not_leaf and lf[2] == -1 and lf[3] == -1 and lf[0] >= 0 and lf[1] >= 0


@needs_ref
def test_deviation_clamped_quantisation(kr, tmp_path):
    """a point just inside the cube whose 2^L (x+1)/2 rounds to 2^L: the builder clamps it into the last cell, the
    reference's vertex_table floors without a clamp, drops it and fails its own assertion"""
    cfg = _config(str(tmp_path), (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    x = np.nextafter(1.0, 0.0)
    pts = np.array([[0.5, 0.5, 0.5], [x, 0.0, 0.0]])
    with pytest.raises(AssertionError):
        kr.kaolin_renderer(str(tmp_path), pts, 0.25, device="cpu")
    tree, origin, scale, level, _ = op.gen_octree(cfg, pts, 0.25, expand=0, in_sfm=False)
    assert level == 3
    lf, not_leaf = vp.lookup(tree, level, (pts - origin) / scale)
    assert not not_leaf and lf.tolist() == [1, 0]
    assert tree["levels"][level].tolist()[lf[1]] == [7, 4, 4]


@needs_ref
def test_deviation_pid_is_an_exact_int(kr, monkeypatch):
    """get_near_far carries the hierarchy index in fp32: 2^24 + 1 comes back as 2^24"""
    gv = __import__("tools.prepare_data.generate_voxel", fromlist=["get_near_far"])
    big = 2 ** 24 + 1

    class Trace:
        @staticmethod
        def unbatched_raytrace(*a, **k):
            return torch.tensor([0], dtype=torch.int32), torch.tensor([big], dtype=torch.int32), torch.tensor([[0.5]])

    monkeypatch.setattr(gv, "spc_render", Trace)
    spc = {"points": None, "pyramid": None, "prefix": None}
    _, _, pid = gv.get_near_far(torch.zeros(1, 3), torch.ones(1, 3), None, torch.zeros(3), 1.0, 25, spc, return_pts=True)
    assert int(pid[0, 0]) == 2 ** 24 != big


def test_oracle_rays_and_first_hit_rules():
    """direction order and the miss rule of a camera inside an occupied voxel"""
    K = np.array([[10.0, 0, 2.0], [0, 10.0, 1.0], [0, 0, 1]], np.float32)
    o, d, n = vp.gen_rays(3, 5, K, np.eye(4)[:3])
    assert np.array_equal(d[7], np.float32([0, 0, 1])) and n[7] == 1                # pixel (c, r) = (cx, cy): no +1/2
    assert np.allclose(np.linalg.norm(d, axis=1), 1, atol=1e-6)
    cfg = {"eval_bbx": [[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]]}
    pts = np.array([[0.01, 0.02, 0.03], [0.01, 0.02, 0.6]])
    tree, origin, scale, level, _ = op.gen_octree(cfg, pts, 0.05, expand=0, in_sfm=False)
    inside = np.eye(4)
    inside[:3, 3] = -pts[0]                                           # the camera sits in the first point's voxel
    depth, leaf = vp.cast(tree, level, origin, scale, 3, 5, K, np.linalg.inv(inside))
    assert np.all(leaf == -1) and np.all(depth == 0)


def test_voxel_exports_reject_bad_arguments():
    from nrw import _lib

    L = _lib.lib()
    err = L.nrw_last_error
    fake = 1 << 20                                                   # never dereferenced: the checks come first
    pyr = (C.c_int * 8)(1, 1, 2, 0, 0, 1, 2, 4)                      # level 2: 1, 1, 2 nodes
    org = (C.c_float * 3)(0, 0, 0)
    V = (C.c_double * 12)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0)
    bad = (C.c_double * 12)(1, 0, 0, float("nan"), 0, 1, 0, 0, 0, 0, 1, 0)
    huge = (C.c_double * 12)(1, 0, 0, 1e300, 0, 1, 0, 0, 0, 0, 1, 0)

    def vc(octree=fake, prefix=fake, pyramid=pyr, level=2, origin=org, scale=1.0, c2w=V, fx=10.0, fy=10.0, cx=1.0,
           cy=1.0, H=4, W=4):
        return L.nrw_voxel_cast(octree, prefix, pyramid, level, origin, scale, c2w, fx, fy, cx, cy, H, W, None, None, None,
                                None, None)

    assert vc(octree=None) != 0 and b"null" in err()
    assert vc(prefix=None) != 0 and b"null" in err()
    assert vc(pyramid=None) != 0 and b"null" in err()
    assert vc(level=0) != 0 and b"level" in err()
    assert vc(level=17) != 0 and b"level" in err()
    assert vc(pyramid=(C.c_int * 8)(1, 1, 0, 0, 0, 1, 2, 2)) != 0 and b"leaf" in err()
    assert vc(origin=None) != 0 and b"origin" in err()
    assert vc(origin=(C.c_float * 3)(0, float("inf"), 0)) != 0 and b"origin" in err()
    assert vc(scale=0.0) != 0 and b"scale" in err()
    assert vc(scale=float("nan")) != 0 and b"scale" in err()
    assert vc(c2w=None) != 0 and b"null" in err()
    assert vc(c2w=bad) != 0 and b"finite" in err()
    assert vc(c2w=huge) != 0 and b"finite" in err()
    assert vc(fx=0.0) != 0 and b"intrinsics" in err()
    assert vc(fy=-1.0) != 0 and b"intrinsics" in err()
    assert vc(cx=float("nan")) != 0 and b"intrinsics" in err()
    assert vc(H=0) != 0 and b"image" in err()
    assert vc(W=-3) != 0 and b"image" in err()
    assert vc(H=1 << 16, W=1 << 16) != 0 and b"INT32_MAX" in err()

    def vl(octree=fake, pyramid=pyr, level=2, points=fake, n=5, leaf=fake, status=fake):
        return L.nrw_voxel_lookup(octree, fake, pyramid, level, points, n, leaf, status, None)

    assert vl(octree=None) != 0 and b"null" in err()
    assert vl(level=-1) != 0 and b"level" in err()
    assert vl(n=-1) != 0 and b"n_points" in err()
    assert vl(n=1 << 31) != 0 and b"n_points" in err()
    assert vl(points=None) != 0 and b"null" in err()
    assert vl(leaf=None) != 0 and b"null" in err()
    assert vl(status=None) != 0 and b"status" in err()


def test_point_source_flag():
    from nrw.reprojection import get_opts

    base = ["--src_file", "a.ply", "--target_file", "b.ply", "--data_path", "d", "--output_path", "o"]
    assert get_opts(base).point_source is False
    assert get_opts(base + ["--point_source"]).point_source is True
