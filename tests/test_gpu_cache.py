"""Ray-cache generation on the GPU (csrc/raygen.cu) against the numpy restatement (oracle/cache_port.py) on a seeded
synthetic scene (tests/util_cache.py): rows and rgbs bit for bit, voxel near/far against the octree tracer, the
depth_percent padding, the per-image near/far percentiles, the split writer and the drop-in dataset."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import util_cache  # noqa: E402
from oracle import cache_port as cp  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def scene_dir(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("cache") / "synth_scene")
    info = util_cache.write_scene(root, n_train=10, n_test=2, n_points=3000, seed=0)
    return info


def _scene(root, ds):
    from nrw.phototourism import read_scene

    return read_scene(root, ds, "sparse")


def _oracle(s, id_, sem_path="semantic_maps", with_sem=True):
    from nrw.phototourism import load_image, load_semantics

    i = s.img_ids.index(id_)
    img = load_image(os.path.join(s.root_dir, "dense/images", s.image_paths[id_]), s.img_downscale)
    sem = load_semantics(s.root_dir, sem_path, s.image_paths[id_].split(".")[0]) if with_sem else None
    b = cp.depth_bounds(s.xyz_world, s.w2c[i:i + 1])[0]
    _, xys, ids = s.imdata[id_]
    return cp.image_rows(img.shape[0], img.shape[1], s.Ks[id_], s.poses[i].astype(np.float32), id_, img, b[0], b[1], xys, ids,
                         s.table_xyz, s.table_err, s.img_downscale, s.w2c[i, 2, :4], sem), img


def _assert_rows(got, ref):
    np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize("ds", [1, 2])
def test_rows_equal_oracle_without_voxels(scene_dir, ds):
    from nrw.phototourism import RayGenerator, depth_bounds

    s = _scene(scene_dir["root"], ds)
    b = depth_bounds(s.xyz_world, s.w2c, DEV)
    gen = RayGenerator(s, DEV, True, "semantic_maps", use_voxel=False, bounds=b)
    n_depth = 0
    for id_, rows, rgbs, counts in gen.images(s.img_ids):
        (ref_rows, ref_rgb), img = _oracle(s, id_)
        assert counts[0] == counts[1] == img.shape[0] * img.shape[1]
        _assert_rows(rows.cpu().numpy(), ref_rows)
        np.testing.assert_array_equal(rgbs.cpu().numpy(), ref_rgb)
        n_depth += int((ref_rows[:, -2] > 0).sum())
    assert n_depth > 100


def test_depth_matches_reference_get_colmap_depth_on_device(scene_dir):
    """The unmodified get_colmap_depth run on cuda:0 agrees with the pass's depth and weight columns to 1e-5.  Pixels hit
    by several keypoints are left out: torch's CUDA scatter picks an unspecified one of them (the CPU run of the
    reference, compared in test_cache_cpu.py, keeps the last, as the pass does)."""
    from oracle import ref_import
    from nrw.phototourism import RayGenerator, depth_bounds

    if not ref_import.available():
        pytest.skip("reference tree not present")
    R = cp.load_cache_ref()
    for ds in (1, 2):
        s = _scene(scene_dir["root"], ds)
        gen = RayGenerator(s, DEV, False, use_voxel=False, bounds=depth_bounds(s.xyz_world, s.w2c, DEV))
        for i, id_ in enumerate(s.img_ids[:6]):
            img, sem = gen.decode(id_)
            rows, _, _ = gen.run(id_, img, sem)
            H, W = int(img.shape[0]), int(img.shape[1])
            _, xys, ids = s.imdata[id_]
            rd, rw = cp.ref_colmap_depth(R, s.table_xyz, s.table_err, xys, ids, s.poses[i], s.Ks[id_], W, H, ds, device=DEV)
            pix, ok = cp.keypoint_winners(xys, ids, len(s.table_err), ds, H, W)
            uniq, cnt = np.unique(pix[ok], return_counts=True)
            single = np.ones(H * W, bool)
            single[uniq[cnt > 1]] = False
            got = rows.cpu().numpy()
            np.testing.assert_array_equal(got[:, 9] != 0, rd != 0)
            np.testing.assert_allclose(got[single, 9], rd[single], rtol=1e-5, atol=0)
            np.testing.assert_allclose(got[single, 10], rw[single], rtol=1e-5, atol=0)


def test_depth_bounds_bit_exact(scene_dir):
    from nrw.phototourism import depth_bounds

    s = _scene(scene_dir["root"], 1)
    np.testing.assert_array_equal(depth_bounds(s.xyz_world, s.w2c, DEV), cp.depth_bounds(s.xyz_world, s.w2c))


def _near_far(tree, origin, scale, level, o, d):
    from nrw import _lib

    L, R = _lib.lib(), o.shape[0]
    near, far = (torch.empty(R, device=DEV) for _ in range(2))
    pid, cnt = (torch.empty(R, dtype=torch.int32, device=DEV) for _ in range(2))
    so = (C.c_float * 3)(*[float(v) for v in origin])
    _lib.check(L.nrw_octree_near_far(_lib.ptr(tree["octree"]), _lib.ptr(tree["prefix"]), None, level, _lib.ptr(o), _lib.ptr(d), R, so,
                                     scale, _lib.ptr(near), _lib.ptr(far), _lib.ptr(pid), _lib.ptr(cnt), _lib.stream_ptr()), "near_far")
    return near, far


def test_voxel_columns_match_octree_tracer(scene_dir):
    from nrw.phototourism import RayGenerator, build_octrees, depth_bounds

    s = _scene(scene_dir["root"], 1)
    b = depth_bounds(s.xyz_world, s.w2c, DEV)
    octs = build_octrees(s.root_dir, s.config, DEV)
    plain = RayGenerator(s, DEV, True, "semantic_maps", use_voxel=False, bounds=b)
    vox = RayGenerator(s, DEV, True, "semantic_maps", use_voxel=True, bounds=b, octrees=octs)
    kept_total = 0
    for id_ in s.img_ids[:4]:
        img, sem = plain.decode(id_)
        full, full_rgb, _ = plain.run(id_, img, sem)
        rows, rgbs, counts = vox.run(id_, img, sem)
        o, d = full[:, 0:3].contiguous(), full[:, 3:6].contiguous()
        n_sfm, _ = _near_far(*octs[0][:1], octs[0][1], octs[0][2], octs[0][3], o, d)
        n_exp, f_exp = _near_far(*octs[1][:1], octs[1][1], octs[1][2], octs[1][3], o, d)
        keep = n_sfm > 0
        f_exp = torch.where(n_exp > 0, f_exp + np.float32(s.config["voxel_size"]), f_exp)
        assert counts[1] == int(keep.sum())
        kept_total += counts[1]
        exp = full[keep].clone()
        exp[:, 6], exp[:, 7] = n_exp[keep], f_exp[keep]
        assert torch.equal(rows, exp)
        assert torch.equal(rgbs, full_rgb[keep])
    assert kept_total > 0


def test_depth_percent_padding_is_seeded_permutation(scene_dir):
    from nrw.phototourism import RayGenerator, build_octrees, depth_bounds

    s = _scene(scene_dir["root"], 2)
    b = depth_bounds(s.xyz_world, s.w2c, DEV)
    octs = build_octrees(s.root_dir, s.config, DEV)
    base = RayGenerator(s, DEV, True, "semantic_maps", use_voxel=True, bounds=b, octrees=octs)
    pad = [RayGenerator(s, DEV, True, "semantic_maps", use_voxel=True, depth_percent=0.8, seed=s_, bounds=b, octrees=octs)
           for s_ in (7, 7, 8)]
    for id_ in s.img_ids[:3]:
        img, sem = base.decode(id_)
        r0, g0, c0 = base.run(id_, img, sem)
        outs = [g.run(id_, img, sem) for g in pad]
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        n, v = c0[1], int((r0[:, -2] > 0).sum())
        npad = cp.padding_count(n, v, 0.8)
        rows, rgbs, c = outs[0]
        assert c[1:] == [n, v, npad] and rows.shape[0] == n + npad and npad > 0
        assert not torch.equal(rows, outs[2][0])
        both = torch.cat([rows, rgbs], 1).cpu().numpy()
        ref = torch.cat([r0, g0], 1).cpu().numpy()
        # every unpadded row once, the rest are copies of depth-valid rows of the same image
        u, cnt = np.unique(both, axis=0, return_counts=True)
        ur, cr = np.unique(ref, axis=0, return_counts=True)
        idx = {row.tobytes(): k for k, row in enumerate(u)}
        extra = cnt.copy()
        for row, k in zip(ur, cr):
            extra[idx[row.tobytes()]] -= k
        assert (extra >= 0).all() and extra.sum() == npad
        assert (u[extra > 0][:, 10] > 0).all()                 # padding copies carry keypoint depth (column 10)


def test_no_padding_when_count_is_negative_or_no_row_has_depth(scene_dir):
    """Deviation from the reference, which raises in both cases: the image gets no padding rows and is only permuted."""
    from nrw.phototourism import RayGenerator, build_octrees, depth_bounds

    s = _scene(scene_dir["root"], 2)
    b = depth_bounds(s.xyz_world, s.w2c, DEV)
    octs = build_octrees(s.root_dir, s.config, DEV)
    id_ = s.img_ids[0]
    no_kp = s._replace(imdata=dict(s.imdata))
    im, xys, ids = no_kp.imdata[id_]
    no_kp.imdata[id_] = (im, xys[:0], ids[:0])
    for scene, p, why in ((s, 0.01, "negative"), (no_kp, 0.4, "no depth row")):
        base = RayGenerator(scene, DEV, True, "semantic_maps", use_voxel=True, bounds=b, octrees=octs)
        pad = RayGenerator(scene, DEV, True, "semantic_maps", use_voxel=True, depth_percent=p, seed=3, bounds=b, octrees=octs)
        img, sem = base.decode(id_)
        r0, g0, c0 = base.run(id_, img, sem)
        r1, g1, c1 = pad.run(id_, img, sem)
        n, v = c0[1], int((r0[:, -2] > 0).sum())
        assert n > 0 and (v == 0) == (why == "no depth row")
        if why == "negative":
            assert p * n - v < 0
        assert c1 == [n, n, v, 0], why
        a = torch.cat([r0, g0], 1).cpu().numpy()
        b1 = torch.cat([r1, g1], 1).cpu().numpy()
        np.testing.assert_array_equal(np.unique(a, axis=0, return_counts=True)[1], np.unique(b1, axis=0, return_counts=True)[1])
        np.testing.assert_array_equal(np.unique(a, axis=0), np.unique(b1, axis=0))


def test_cli_splits_load_into_raycache(scene_dir, tmp_path):
    from nrw.prepare_data_cache import get_opts, prepare
    from nrw.raycache import RayCache, load_split_arrays

    root = scene_dir["root"]
    a = get_opts(["--root_dir", root, "--cache_dir", "c_split", "--cache_type", "npz", "--img_downscale", "2",
                  "--split_to_chunks", "3", "--semantic_map_path", "semantic_maps", "--seed", "5"])
    r1 = prepare(a)
    b = get_opts(["--root_dir", root, "--cache_dir", "c_one", "--cache_type", "npz", "--img_downscale", "2",
                  "--semantic_map_path", "semantic_maps", "--seed", "5"])
    r2 = prepare(b)
    assert r1["rows"] == r2["rows"] and r1["images"] == scene_dir["n_train"]
    one = np.load(os.path.join(root, "c_one", "rays2.npz"))["arr_0"]
    one_rgb = np.load(os.path.join(root, "c_one", "rgbs2.npz"))["arr_0"]
    meta = json.load(open(os.path.join(root, "c_split", "splits", "rays2_meta_info.json")))
    names = [f"split_{i}" for i in range(3)]
    rays, rgbs = load_split_arrays(root, "c_split/splits", names, 2)
    total = one.shape[0]
    pidx = np.random.RandomState(5).choice(total, 3 - total % 3, replace=False) if total % 3 else np.array([], np.int64)
    np.testing.assert_array_equal(rays, np.concatenate([one, one[pidx]], 0))
    np.testing.assert_array_equal(rgbs, np.concatenate([one_rgb, one_rgb[pidx]], 0))
    assert meta == {"data_length": total + len(pidx), "chunk_length": (total + len(pidx)) // 3, "n_trunks": 3}
    assert not [f for f in os.listdir(os.path.join(root, "c_one")) if f.endswith(".spill")]
    cache = RayCache(rays, rgbs, 256, DEV, seed=0)
    from nrw.train import TrainSystem

    sysm = TrainSystem(DEV, n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4, n_vocab=64, chunk_rows=8192,
                       batch_size=256)
    batch = cache.next_batch()
    assert batch["n_valid"] > 0
    assert torch.isfinite(sysm.training_step(batch))


def test_val_dataset_sample_equals_oracle(scene_dir):
    from nrw.phototourism import PhototourismDataset

    ds = PhototourismDataset(scene_dir["root"], split="val", img_downscale=1, semantic_map_path="semantic_maps",
                             with_semantics=True, device=0)
    assert ds.img_downscale == 8 and len(ds) == 1
    s = ds.scene
    smp = ds[0]
    (ref_rows, ref_rgb), img = _oracle(s, ds.val_id)
    np.testing.assert_array_equal(smp["rays"].numpy(), ref_rows[:, :8])
    np.testing.assert_array_equal(smp["rgbs"].numpy(), ref_rgb)
    np.testing.assert_array_equal(smp["semantics"].numpy()[:, 0], ref_rows[:, 9])
    assert smp["img_wh"].tolist() == [img.shape[1], img.shape[0]]
    assert (smp["ts"] == ds.val_id).all()


def test_split_comes_from_own_tsv_row(scene_dir):
    s = _scene(scene_dir["root"], 1)
    names = [s.image_paths[i] for i in s.img_ids if s.splits[i] != "test"]
    assert names == [f"img_{k:03d}.png" for k in range(scene_dir["n_train"])]


def test_unsupported_splits_raise(scene_dir):
    from nrw._lib import NrwError
    from nrw.phototourism import PhototourismDataset

    for kw in ({"split": "eval"}, {"split": "test"}, {"shared_cache": True}):
        with pytest.raises(NrwError):
            PhototourismDataset(scene_dir["root"], **kw)
