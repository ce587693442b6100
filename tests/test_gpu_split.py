"""GPU: the scene split (csrc/viewsel.cu, nrw.prepare_data_split).  ROI counts bit for bit against the restatement
oracle/split_port.py on the synthetic scene and on adversarial views (inside the sphere, facing away, grazing, mixed sizes
in one launch, more than 65,535 views, a view above 2^24 pixels), static counts against numpy, the argument checks, and
`python -m nrw.prepare_data_split` end to end against the unmodified reference script run with torch on the same GPU,
followed by `nrw.prepare_data_cache` on the tsv it wrote."""
import ctypes as C
import os
import runpy
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from oracle import split_port as sp
import util_split

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def scene_src(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("split_gpu") / "split_scene")
    util_split.write_scene(root, seed=11)
    return root


def _scene_views(root):
    from nrw import colmap
    from nrw import prepare_data_split as P
    from nrw.phototourism import camera_poses

    im = colmap.read_images(os.path.join(root, "dense/sparse/images.bin"))
    cams = colmap.read_cameras(os.path.join(root, "dense/sparse/cameras.bin"))
    ids = list(im)
    _, poses = camera_poses([im[i] for i in ids], "test")
    hw = [P.image_size(os.path.join(root, "dense/images", im[i].name))[::-1] for i in ids]
    return P.view_table([P.pinhole_K(cams[im[i].camera_id]) for i in ids], poses), np.array(hw)


def _look(C_, target, up=(0.0, 0.0, 1.0)):
    """c2w [3, 4] (columns 1:2 negated, as read_meta makes them) of a camera at C_ looking at target"""
    f = np.asarray(target, float) - C_
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    if np.linalg.norm(r) < 1e-6:
        r = np.cross(f, [0.0, 1.0, 0.0])
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    c2w = np.stack([r, d, f], 1)                 # COLMAP camera axes (right, down, forward) in world coordinates
    c2w[:, 1:3] *= -1
    return np.concatenate([c2w, np.asarray(C_, float)[:, None]], 1)


def _row(fx, fy, cx, cy, c2w):
    return np.concatenate([[fx, fy, cx, cy], np.asarray(c2w, np.float64).reshape(-1)]).astype(np.float32)


def _adversarial(rng, s, R):
    views, hw = [], []
    s = np.asarray(s, float)
    # inside the sphere, several directions
    for k in range(3):
        views.append(_row(60, 61, 40.3, 30.1, _look(s + rng.uniform(-0.5, 0.5, 3) * R, s + rng.standard_normal(3))))
        hw.append((61, 81))
    # facing away from outside
    C_ = s + np.array([3.0, 0.5, 0.2]) * R
    views.append(_row(70, 70, 50, 40, _look(C_, C_ + (C_ - s))))
    hw.append((79, 101))
    # grazing: the silhouette runs through the image, at several offsets from the limb
    for off in (1.0, 0.999, 1.001, 0.98, 1.02):
        C_ = s + np.array([0.0, -4.0, 0.3]) * R
        f = (s - C_) / np.linalg.norm(s - C_)
        side = np.cross(f, [0, 0, 1.0])
        side /= np.linalg.norm(side)
        views.append(_row(400.0, 401.0, 63.5, 47.5, _look(C_, s + side * R * off)))
        hw.append((95, 127))
    # random cameras of mixed sizes
    for k in range(12):
        C_ = s + rng.standard_normal(3) * 3 * R
        views.append(_row(rng.uniform(30, 900), rng.uniform(30, 900), rng.uniform(0, 200), rng.uniform(0, 150),
                          _look(C_, s + rng.standard_normal(3) * R)))
        hw.append((int(rng.integers(1, 160)), int(rng.integers(1, 220))))
    return np.array(views), np.array(hw)


def test_roi_counts_equal_port_on_scene_and_adversarial_views(scene_src):
    from nrw.prepare_data_split import roi_counts

    views, hw = _scene_views(scene_src)
    got = roi_counts(views, hw, util_split.ORIGIN, util_split.RADIUS, 0)
    np.testing.assert_array_equal(got, sp.roi_counts(views, hw, util_split.ORIGIN, util_split.RADIUS))
    assert got.min() == 0 and (got == hw[:, 0] * hw[:, 1]).sum() >= 2
    rng = np.random.default_rng(3)
    for s, R in (([0.1, -0.2, 0.3], 1.0), ([5.0, -3.0, 2.0], 0.37), ([0.0, 0.0, 0.0], 12.5)):
        av, ah = _adversarial(rng, s, R)
        # mixed sizes in one launch: the scene's views and the adversarial ones together
        v_all, h_all = np.concatenate([views, av]), np.concatenate([hw, ah])
        got = roi_counts(v_all, h_all, s, R, 0)
        want = sp.roi_counts(v_all, h_all, s, R)
        np.testing.assert_array_equal(got, want)
        n_sc = len(views)
        assert (got[n_sc:n_sc + 3] == 61 * 81).all()             # inside the sphere
        assert got[n_sc + 3] == 0                                  # facing away
        grazing = got[n_sc + 4:n_sc + 9] / (95 * 127)
        assert ((grazing > 0.05) & (grazing < 0.95)).all()


def test_roi_counts_chunk_views_past_grid_limit():
    """more than 65,535 views: the launch is chunked over gridDim.y"""
    from nrw.prepare_data_split import roi_counts

    rng = np.random.default_rng(8)
    n = 65535 + 4471
    s, R = np.array([0.0, 0.0, 0.0]), 1.0
    base = np.stack([_row(3, 3, 1, 1, _look(s + rng.standard_normal(3) * 2.0, s + rng.standard_normal(3) * 0.8))
                     for _ in range(256)])
    pick = rng.integers(0, 256, n)
    views = base[pick]
    hw = np.stack([rng.integers(1, 4, n), rng.integers(1, 5, n)], 1)
    got = roi_counts(views, hw, s, R, 0)
    # the port per distinct (view, size) pair
    cache = {}
    want = np.empty(n, np.int64)
    for i in range(n):
        key = (int(pick[i]), int(hw[i, 0]), int(hw[i, 1]))
        if key not in cache:
            cache[key] = int(sp.roi_counts(base[pick[i]][None], hw[i][None], s, R)[0])
        want[i] = cache[key]
    np.testing.assert_array_equal(got, want)
    assert 0 < want[65535:].sum() < (hw[65535:, 0] * hw[65535:, 1]).sum()


def test_roi_count_above_2_24_pixels_and_fp32_share():
    from nrw.prepare_data_split import roi_counts, roi_keep

    H, W = 4099, 4101                                    # 16.8 M pixels: the fp32 share rounds
    s, R = np.array([0.0, 0.0, 0.0]), 1.0
    v = _row(3000.0, 3001.0, 2049.7, 2050.2, _look(np.array([0.3, -3.5, 0.4]), [0.05, 0.02, -0.03]))[None]
    got = roi_counts(v, [(H, W)], s, R, 0)
    want = sp.roi_counts(v, [(H, W)], s, R)
    assert got[0] == want[0] and 0 < got[0] < H * W
    assert H * W != int(np.float32(H * W))                # the pixel count itself rounds in fp32
    share = np.float32(got[0]) / np.float32(H * W)
    assert roi_keep(got, [(H, W)], float(share))[0] and not roi_keep(got, [(H, W)], float(np.nextafter(share, np.float32(2))))[0]


def test_invalid_view_on_device_gets_minus_one():
    from nrw import _lib

    L = _lib.lib()
    rng = np.random.default_rng(2)
    views = torch.from_numpy(np.stack([_row(50, 50, 20, 15, _look(rng.standard_normal(3) * 3, [0, 0, 0])) for _ in range(4)])).to(DEV)
    hw = torch.tensor([[30, 40], [0, 5], [31, 41], [40, 40]], dtype=torch.int32, device=DEV)
    counts = torch.full((4,), 7, dtype=torch.int64, device=DEV)
    o = (C.c_float * 3)(0.0, 0.0, 0.0)
    assert L.nrw_view_roi_count(_lib.ptr(views), _lib.ptr(hw), 4, 31 * 41, o, 1.0, _lib.ptr(counts), _lib.stream_ptr()) == 0
    got = counts.cpu().numpy()
    assert got[1] == -1 and got[3] == -1                  # a zero height, and 1600 pixels > max_hw
    want = sp.roi_counts(views.cpu().numpy()[[0, 2]], [(30, 40), (31, 41)], [0, 0, 0], 1.0)
    np.testing.assert_array_equal(got[[0, 2]], want)


def test_static_counts_equal_numpy(scene_src):
    from nrw import _lib
    from nrw.prepare_data_split import TRANSIENT_OBJECTS, static_counts
    from nrw.renderer import LABEL_IDS

    ids = [LABEL_IDS[t] for t in TRANSIENT_OBJECTS]
    names = [f"img_{i:03d}.png" for i in range(len(util_split.CAMERAS))]
    counts, sizes = static_counts(scene_src, "semantic_maps", names, ids, 0)
    for name, c, hw in zip(names, counts, sizes):
        sem = np.load(os.path.join(scene_src, "semantic_maps", name.replace(".png", ".npz")))["arr_0"]
        assert hw == sem.shape and c == sp.static_count(sem, ids), name
    assert counts[names.index(util_split.FULLY_TRANSIENT)] == 0
    # up to 8 ids, none, and accumulation into one counter
    L = _lib.lib()
    rng = np.random.default_rng(4)
    acc = torch.zeros(1, dtype=torch.int64, device=DEV)
    total = 0
    for n_ids, n in ((8, 1_000_003), (0, 777), (3, 1), (5, 4_194_304 + 17)):
        sem = rng.integers(0, 150, n).astype(np.float32)
        q = [int(v) for v in rng.choice(150, n_ids, replace=False)]
        d = torch.from_numpy(sem).to(DEV)
        arr = (C.c_int * max(1, n_ids))(*q)
        assert L.nrw_label_static_count(_lib.ptr(d), n, arr, n_ids, _lib.ptr(acc), _lib.stream_ptr()) == 0
        total += int((~np.isin(sem, np.array(q, np.float32))).sum())
    assert int(acc.item()) == total


def test_bad_arguments_give_nrw_err_arg():
    from nrw import _lib

    L = _lib.lib()
    views = torch.zeros((2, 16), dtype=torch.float32, device=DEV)
    hw = torch.ones((2, 2), dtype=torch.int32, device=DEV)
    counts = torch.zeros(2, dtype=torch.int64, device=DEV)
    o = (C.c_float * 3)(0.0, 0.0, 0.0)
    sp_ = _lib.stream_ptr()
    P = _lib.ptr

    def roi(n=2, max_hw=1, origin=o, r=1.0, v=views, h=hw, c=counts):
        return L.nrw_view_roi_count(P(v), P(h), n, max_hw, origin, r, P(c), sp_)

    assert roi() == 0
    for kw in ({"n": 0}, {"n": -3}, {"max_hw": 0}, {"max_hw": (1 << 31)}, {"r": 0.0}, {"r": -2.0}, {"r": float("nan")},
               {"r": float("inf")}, {"origin": (C.c_float * 3)(0.0, float("inf"), 0.0)}, {"origin": None}, {"v": None},
               {"h": None}, {"c": None}):
        assert roi(**kw) == -1, kw                       # NRW_ERR_ARG
    labels = torch.full((10,), 200.0, dtype=torch.float32, device=DEV)     # no id below matches
    cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
    ids = (C.c_int * 9)(*range(9))
    assert L.nrw_label_static_count(P(labels), 10, ids, 8, P(cnt), sp_) == 0
    for args in ((P(labels), 10, ids, 9), (P(labels), 10, ids, -1), (P(labels), -1, ids, 2), (None, 10, ids, 2),
                 (P(labels), 10, None, 2), (P(labels), 10, (C.c_int * 1)(-1), 1), (P(labels), 10, (C.c_int * 1)(1 << 24), 1)):
        assert L.nrw_label_static_count(*args, P(cnt), sp_) == -1, args
    assert L.nrw_label_static_count(P(labels), 10, ids, 2, None, sp_) == -1
    torch.cuda.synchronize()
    assert int(cnt.item()) == 10                          # only the one good call counted


def test_cli_end_to_end_equals_reference_script_then_cache(scene_src, tmp_path):
    """python -m nrw.prepare_data_split writes the tsv bytes the unmodified prepare_data_split.py writes with torch on
    this GPU after np.random.seed(seed); nrw.prepare_data_cache then builds a cache from it without the test images"""
    from oracle import ref_import

    if not ref_import.available():
        pytest.skip("reference tree not present")
    pytest.importorskip("pandas")
    seed, roi, static, num_test = 5, 0.25, 0.5, 2
    ours, ref = str(tmp_path / "ours" / "split_scene"), str(tmp_path / "ref" / "split_scene")
    shutil.copytree(scene_src, ours)
    shutil.copytree(scene_src, ref)
    # no ROI share within the measured tolerance of the threshold, so the reference's rays decide every view alike
    views, hw = _scene_views(scene_src)
    share = sp.roi_counts(views, hw, util_split.ORIGIN, util_split.RADIUS) / (hw[:, 0] * hw[:, 1])
    assert np.abs(share - roi).min() > sp.ROI_TOLERANCE

    flags = ["--num_test", str(num_test), "--min_observation", "3", "--roi_threshold", str(roi), "--static_threshold",
             str(static)]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    r = subprocess.run([sys.executable, "-s", "-m", "nrw.prepare_data_split", "--root_dir", ours, "--seed", str(seed)] + flags,
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]

    R = sp.load_split_ref()
    old = sys.argv
    sys.argv = ["prepare_data_split.py", "--root_dir", ref] + flags
    try:
        np.random.seed(seed)
        runpy.run_path(R.script, run_name="__main__")
    finally:
        sys.argv = old
    tsv_ours = open(os.path.join(ours, "split_scene.tsv"), "rb").read()
    assert tsv_ours == open(os.path.join(ref, "split_scene.tsv"), "rb").read()
    assert sorted(os.listdir(os.path.join(ours, "trash_images"))) == sorted(os.listdir(os.path.join(ref, "trash_images")))

    from nrw import colmap
    from nrw.prepare_data_cache import get_opts, prepare

    lines = [ln.split("\t") for ln in tsv_ours.decode().splitlines()[1:]]
    assert [ln[2] for ln in lines] == ["test"] * num_test + ["train"] * (len(lines) - num_test)
    by_name = {im.name: i for i, im in colmap.read_images(os.path.join(ours, "dense/sparse/images.bin")).items()}
    train = {by_name[ln[0]] for ln in lines if ln[2] == "train"}
    test = {by_name[ln[0]] for ln in lines if ln[2] == "test"}
    res = prepare(get_opts(["--root_dir", ours, "--cache_type", "npz", "--semantic_map_path", "semantic_maps"]))
    assert res["images"] == len(train) and res["rows"] > 0
    rays = np.load(os.path.join(ours, "cache", "rays1.npz"))["arr_0"]
    ts = set(np.unique(rays[:, 8]).astype(int).tolist())
    assert ts <= train and not ts & test and len(ts) >= len(train) // 2
