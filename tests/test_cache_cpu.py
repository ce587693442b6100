"""Ray-cache generation without a GPU: the numpy restatement (oracle/cache_port.py) against the unmodified reference
(get_rays, get_colmap_depth, read_images_binary, split_to_chunks through cache_port.load_cache_ref), numpy's percentile
and cv2's nearest resize; the CLI's flags and the argument checks of the new C exports."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import cache_port as cp  # noqa: E402


def test_percentile_restatement_equals_numpy():
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 7, 999, 1000, 1001, 12345):
        z = np.sort(rng.lognormal(1.0, 1.0, n))
        for q in (0.1, 99.9, 0.0, 100.0, 50.0, 37.3):
            assert cp.percentile_linear(z, q) == np.percentile(z, q), (n, q)


def test_depth_bounds_match_numpy_on_reference_matmul():
    rng = np.random.default_rng(1)
    xyz = rng.uniform(-2, 2, (5000, 3))
    w2c = []
    for _ in range(4):
        A = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        w2c.append(np.concatenate([np.concatenate([A, rng.uniform(-1, 1, (3, 1)) + [[0], [0], [4]]], 1), [[0, 0, 0, 1]]], 0))
    ours = cp.depth_bounds(xyz, w2c)
    xyz_h = np.concatenate([xyz, np.ones((len(xyz), 1))], -1)
    for i, w in enumerate(w2c):
        z = (xyz_h @ w.T)[:, 2]
        z = z[z > 0]
        ref = np.array([np.percentile(z, 0.1), np.percentile(z, 99.9)])
        np.testing.assert_allclose(ours[i], ref, rtol=1e-12)


@pytest.mark.parametrize("shape,ds", [((67, 1001), 2), ((61, 81), 3), ((73, 95), 1), ((49, 63), 4), ((45, 65), 7)])
def test_label_index_rule_equals_cv2_nearest(shape, ds):
    cv2 = pytest.importorskip("cv2")
    sem = np.random.default_rng(2).integers(0, 200, shape).astype(np.float32)
    H, W = shape[0] // ds, shape[1] // ds
    ref = cv2.resize(sem, (W, H), interpolation=cv2.INTER_NEAREST).reshape(-1)
    np.testing.assert_array_equal(cp.label(sem, H, W), ref)


def _ref():
    from oracle import ref_import

    if not ref_import.available():
        pytest.skip("reference tree not present")
    return cp.load_cache_ref()


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import util_cache

    root = str(tmp_path_factory.mktemp("cache_cpu") / "synth_scene")
    util_cache.write_scene(root, n_train=4, n_test=1, n_points=1500, seed=1)
    return root


def test_rays_match_reference_get_rays():
    """Each direction component is within 2 ulp of 1.0 (the norm of the unit direction) of the reference's get_rays;
    per-component relative ulps are meaningless for components that cancel to near zero."""
    import torch

    R = _ref()
    rng = np.random.default_rng(3)
    for t in range(12):
        H, W = 61 + t, 81 + 2 * t
        K = np.array([[70.3 + t, 0, W / 2], [0, 71.1, H / 2], [0, 0, 1]], np.float32)
        A = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        c2w = np.concatenate([A, rng.standard_normal((3, 1))], 1).astype(np.float32)
        ro, rd = R.get_rays(R.get_ray_directions(H, W, K), torch.from_numpy(c2w))
        o, d, _ = cp.rays(H, W, K, c2w)
        np.testing.assert_array_equal(o, ro.numpy())
        assert (np.abs(d - rd.numpy()) <= 2 * np.spacing(np.float32(1))).all()


@pytest.mark.parametrize("ds", [1, 2])
def test_keypoint_depth_matches_reference_get_colmap_depth(scene, ds):
    from nrw.phototourism import read_scene

    R = _ref()
    s = read_scene(scene, ds, "sparse")
    n_dup = 0
    for i, id_ in enumerate(s.img_ids):
        _, xys, ids = s.imdata[id_]
        K = s.Ks[id_]
        W, H = int(round(K[0, 2] * 2)), int(round(K[1, 2] * 2))     # the synthetic principal points are image centres
        _, _, nrm = cp.rays(H, W, K, s.poses[i].astype(np.float32))
        depth, weight, win = cp.depth_weight(H, W, nrm, xys, ids, s.table_xyz, s.table_err, ds, s.w2c[i, 2, :4])
        rd, rw = cp.ref_colmap_depth(R, s.table_xyz, s.table_err, xys, ids, s.poses[i], K, W, H, ds)
        np.testing.assert_array_equal(depth != 0, rd != 0)          # the same depth pixels
        np.testing.assert_allclose(depth, rd, rtol=1e-5, atol=0)
        np.testing.assert_allclose(weight, rw, rtol=1e-5, atol=0)
        # pixels hit by several keypoints: the reference keeps the last one, and so does the oracle
        pix, ok = cp.keypoint_winners(xys, ids, len(s.table_err), ds, H, W)
        for p in np.unique(pix[ok]):
            hits = np.nonzero(pix == p)[0]
            zs = cp.camera_z(s.table_xyz[ids[hits]], s.w2c[i])
            if len(hits) > 1 and np.ptp(zs) > 1e-3 * np.abs(zs).max():      # distinguishable at the 1e-5 depth check
                n_dup += 1
                assert win[int(p)] == hits[-1]
    assert n_dup > 0


def test_read_images_with_points_equals_reference(scene):
    from nrw import colmap

    R = _ref()
    path = os.path.join(scene, "dense", "sparse", "images.bin")
    ref = R.read_images_binary(path)
    ours = colmap.read_images(path, with_points=True)
    assert list(ref) == list(ours)
    for k, (im, xys, pids) in ours.items():
        r = ref[k]
        assert (r.id, r.name, r.camera_id) == (im.id, im.name, im.camera_id)
        np.testing.assert_array_equal(r.qvec, im.qvec)
        np.testing.assert_array_equal(r.tvec, im.tvec)
        np.testing.assert_array_equal(r.xys, xys)
        np.testing.assert_array_equal(r.point3D_ids, pids)
        assert xys.dtype == np.float64 and pids.dtype == np.int64


@pytest.mark.parametrize("n_chunks", [3, 5, 4])
def test_split_files_equal_reference_split_to_chunks(tmp_path, n_chunks):
    import types

    import torch
    from nrw.prepare_data_cache import split_padding, write_splits

    R = _ref()
    rng = np.random.default_rng(n_chunks)
    parts = [rng.standard_normal((n, 12)).astype(np.float32) for n in (37, 1, 50, 15)]
    rows = np.concatenate(parts, 0)
    total = rows.shape[0]
    pidx, L = split_padding(total, n_chunks, seed=9)
    args = types.SimpleNamespace(split_to_chunks=n_chunks, img_downscale=2, cache_type="npz")
    (tmp_path / "ref").mkdir()
    (tmp_path / "ours").mkdir()
    R.split_to_chunks([torch.from_numpy(p) for p in parts], total, L, str(tmp_path / "ref"), args, pidx, "rays")
    write_splits(rows, pidx, L, n_chunks, str(tmp_path / "ours"), "rays", 2)
    for i in range(n_chunks):
        a = np.load(tmp_path / "ref" / f"split_{i}" / "rays2.npz")["arr_0"]
        b = np.load(tmp_path / "ours" / f"split_{i}" / "rays2.npz")["arr_0"]
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    assert (tmp_path / "ref" / "rays2_meta_info.json").read_text() == (tmp_path / "ours" / "rays2_meta_info.json").read_text()


def test_keypoint_last_wins_and_out_of_frame():
    xys = np.array([[1.2, 1.1], [0.8, 0.9], [10.0, 1.0], [-0.6, 0.0], [2.0, 2.0]])
    ids = np.array([0, 1, 2, 0, -1])
    table_xyz = np.array([[0, 0, 2.0], [0, 0, 3.0], [0, 0, 4.0]])
    table_err = np.array([1.0, 2.0, 3.0])
    nrm = np.ones(16, np.float32)
    depth, weight, win = cp.depth_weight(4, 4, nrm, xys, ids, table_xyz, table_err, 1, [0.0, 0.0, 1.0, 0.0])
    assert win == {5: 1}                                     # keypoint 1 lands on (1,1) after keypoint 0 and wins
    assert depth[5] == np.float32(3.0) and (depth != 0).sum() == 1
    mean = (1.0 + 2.0) / 2
    assert weight[5] == np.float32(2 * np.exp(-(2.0 / mean) ** 2))


def test_padding_count_rule():
    assert cp.padding_count(100, 10, 0.2) == int(np.ceil((0.2 * 100 - 10) / 0.8))
    assert cp.padding_count(100, 50, 0.2) == 0                # negative: none (the reference raises)
    assert cp.padding_count(100, 0, 0.2) == 0                 # no depth row: none (the reference raises)
    assert cp.padding_count(100, 10, 0.0) == 0


def test_split_writer_matches_chunk_rule(tmp_path):
    from nrw.prepare_data_cache import split_padding, write_splits

    rows = np.arange(103 * 3, dtype=np.float32).reshape(103, 3)
    pidx, L = split_padding(103, 5, seed=4)
    assert len(pidx) == 2 and L == 21
    np.testing.assert_array_equal(pidx, np.random.RandomState(4).choice(103, 2, replace=False))
    write_splits(rows, pidx, L, 5, str(tmp_path), "rays", 2)
    ref = cp.split_chunks(rows, 5, pidx)
    for i in range(5):
        got = np.load(tmp_path / f"split_{i}" / "rays2.npz")["arr_0"]
        assert got.tobytes() == ref[i].tobytes()
    assert split_padding(100, 5, 0)[0].size == 0             # pad == n_chunks -> no padding


def test_cli_parses_reference_flags():
    from nrw.prepare_data_cache import get_opts

    a = get_opts(["--root_dir", "/x/brandenburg_gate", "--dataset_name", "phototourism", "--cache_dir", "cache_sgs",
                  "--cache_type", "npz", "--img_downscale", "2", "--split_to_chunks", "64", "--semantic_map_path",
                  "semantic_maps"])
    assert (a.cache_type, a.img_downscale, a.split_to_chunks, a.semantic_map_path) == ("npz", 2, 64, "semantic_maps")
    assert a.sfm_path is None and a.depth_percent is None and a.seed == 0
    from nrw.phototourism import scene_defaults

    assert scene_defaults("/x/brandenburg_gate") == ("../neuralsfm", 0.2)
    assert scene_defaults("/x/palacio_de_bellas_artes/") == ("../neuralsfm", 0.4)
    assert scene_defaults("/x/some_other_scene") == ("sparse", 0.0)


def test_generator_rejects_depth_percent_outside_unit_interval():
    from nrw._lib import NrwError
    from nrw.phototourism import RayGenerator

    for bad in (1.0, -0.2, 2.0):
        with pytest.raises(NrwError):
            RayGenerator(None, "cpu", False, depth_percent=bad)


def test_cli_rejects_h5(tmp_path):
    from nrw._lib import NrwError
    from nrw.prepare_data_cache import get_opts, prepare

    with pytest.raises(NrwError):
        prepare(get_opts(["--root_dir", str(tmp_path), "--cache_type", "h5"]))


def _lib_or_skip():
    from nrw import _lib

    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("libnrw.so not built")
    return _lib, _lib.lib()


def test_raygen_exports_reject_bad_arguments():
    _lib, L = _lib_or_skip()
    assert L.nrw_raygen_scratch_bytes(0, 10, 1, 0, 1) < 0
    assert L.nrw_raygen_scratch_bytes(10, 10, 1, -1, 100) < 0
    assert L.nrw_raygen_scratch_bytes(10, 10, 1, 0, 0) < 0
    assert L.nrw_depth_range_scratch_bytes(0, 1) < 0
    assert L.nrw_depth_range_scratch_bytes(1 << 20, 1 << 12) < 0
    assert L.nrw_raygen_capacity(10, 10, 0.0) == 100
    for bad in (1.0, 1.5, -0.1, float("nan"), float("inf"), 1 - 1e-12):
        assert L.nrw_raygen_capacity(10, 10, bad) < 0, bad
    assert L.nrw_raygen_capacity(0, 10, 0.2) < 0
    dummy = C.c_void_p(16)

    def cfg(**kw):
        g = _lib.RaygenCfg()
        g.height, g.width, g.img_downscale = 10, 10, 1
        g.fx, g.fy, g.cx, g.cy = 10.0, 10.0, 5.0, 5.0
        g.c2w[:] = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]
        g.w2c_z[:] = [0, 0, 1, 0]
        for k, v in kw.items():
            setattr(g, k, v)
        return g

    def call(g, cap=100, nk=0, sem=None):
        return L.nrw_raygen_image(C.byref(g), dummy, sem, None, None, nk, None, None, 0, dummy, dummy, cap, dummy, dummy, dummy,
                                  None)

    assert call(cfg(fx=0.0)) != 0
    assert call(cfg(fy=float("nan"))) != 0
    assert call(cfg(img_downscale=0)) != 0
    assert call(cfg(depth_percent=1.0)) != 0
    assert call(cfg(depth_percent=0.3), cap=100) != 0          # capacity below nrw_raygen_capacity
    assert call(cfg(), nk=5) != 0                              # keypoints without a point table
    assert call(cfg(with_label=1, sem_height=20, sem_width=20)) != 0   # label without a map
    assert call(cfg(with_label=1, sem_height=21, sem_width=30), sem=dummy) != 0   # map // ds != image
    assert call(cfg(use_voxel=1)) != 0                         # null octrees
    g = cfg(use_voxel=1)
    for ref in (g.sfm, g.expanded):
        ref.octree, ref.prefix, ref.level, ref.scale = 16, 16, 17, 1.0
    assert call(g) != 0                                        # level out of range
    g.c2w[3] = float("inf")
    assert call(cfg(c2w=g.c2w)) != 0
    assert L.nrw_depth_range(dummy, 10, dummy, 1, -1.0, 50.0, dummy, None, dummy, dummy, None) != 0
    assert L.nrw_depth_range(dummy, 10, None, 1, 0.1, 99.9, dummy, None, dummy, dummy, None) != 0
