"""Scene split without a GPU: the numpy restatement of the ROI rule (oracle/split_port.py) against the unmodified
view_selection, the decision against torch's own expression, the tsv against the unmodified prepare_data_split.py with
real pandas, the trash_images names, the label ids, each documented deviation and the argument checks of the new C
exports.  The device counts are replaced by the restatement (the GPU tests show they are equal bit for bit)."""
import ctypes as C
import os
import runpy
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import split_port as sp  # noqa: E402

import util_split  # noqa: E402


def _ref():
    from oracle import ref_import

    if not ref_import.available():
        pytest.skip("reference tree not present")
    return sp.load_split_ref()


@pytest.fixture
def cpu_cuda(monkeypatch):
    """the reference calls .cuda(); on the CPU it is the identity"""
    import torch

    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)


@pytest.fixture
def port_counts(monkeypatch):
    """nrw.prepare_data_split with the restatement in place of the two device counts"""
    from nrw import prepare_data_split as P
    from nrw.phototourism import load_semantics

    def roi_counts(views, hw, scene_origin, scene_radius, device=0):
        return sp.roi_counts(views, hw, np.asarray(scene_origin, np.float32), np.float32(scene_radius))

    def static_counts(root_dir, semantic_map_path, names, ids, device=0):
        maps = [load_semantics(root_dir, semantic_map_path, n.split(".")[0]) for n in names]
        return np.array([sp.static_count(m, ids) for m in maps], np.int64), [m.shape[:2] for m in maps]

    monkeypatch.setattr(P, "roi_counts", roi_counts)
    monkeypatch.setattr(P, "static_counts", static_counts)
    return P


@pytest.fixture(scope="module")
def scene_src(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("split_src") / "split_scene")
    util_split.write_scene(root, seed=3)
    return root


@pytest.fixture
def scene(scene_src, tmp_path):
    root = str(tmp_path / "split_scene")
    shutil.copytree(scene_src, root)
    return root


def _views(root, min_observation=-1):
    """(names, view table, hw) of the views view_selection scores, in its order"""
    from nrw import colmap
    from nrw import prepare_data_split as P
    from nrw.phototourism import camera_poses

    im = colmap.read_images(os.path.join(root, "dense/sparse/images.bin"))
    cams = colmap.read_cameras(os.path.join(root, "dense/sparse/cameras.bin"))
    ids = list(im)
    _, poses = camera_poses([im[i] for i in ids], "test")
    hw = []
    for i in ids:
        w, h = P.image_size(os.path.join(root, "dense/images", im[i].name))
        hw.append((h, w))
    return [im[i].name for i in ids], P.view_table([P.pinhole_K(cams[im[i].camera_id]) for i in ids], poses), np.array(hw)


def _args(root, **kw):
    from nrw.prepare_data_split import get_opts

    argv = ["--root_dir", root]
    for k, v in kw.items():
        argv += [f"--{k}", str(v)]
    return get_opts(argv)


def test_roi_shares_match_reference_view_selection(scene, cpu_cuda):
    """the unmodified view_selection, run at thresholds midway between consecutive shares of the restatement, keeps
    exactly the views the restatement keeps"""
    from nrw.prepare_data_split import roi_keep

    R = _ref()
    names, views, hw = _views(scene)
    counts = sp.roi_counts(views, hw, util_split.ORIGIN, util_split.RADIUS)
    share = np.sort(np.unique(counts.astype(np.float32) / (hw[:, 0] * hw[:, 1]).astype(np.float32)))
    assert share[0] == 0 and share[-1] == 1 and len(share) >= 8
    for thr in (share[1:] + share[:-1]) / 2:
        ref = R.view_selection(scene, util_split.ORIGIN, util_split.RADIUS, -1, roi_threshold=float(thr))
        ours = [n for n, k in zip(names, roi_keep(counts, hw, float(thr))) if k]
        assert list(ref) == ours, thr


def test_roi_share_difference_to_reference_rays_is_bounded(scene):
    """deviation 4: the reference's matmul + torch.norm rays can decide a grazing pixel differently; the per-view share
    differs by at most split_port.ROI_TOLERANCE"""
    R = _ref()
    names, views, hw = _views(scene)
    worst = 0.0
    for v, (H, W) in zip(views, hw):
        K = np.array([[v[0], 0, v[2]], [0, v[1], v[3]], [0, 0, 1]], np.float32)
        ours = sp.roi_count(int(H), int(W), K, v[4:].reshape(3, 4), util_split.ORIGIN, util_split.RADIUS)
        ref = sp.ref_roi_count(R, int(H), int(W), K, v[4:].reshape(3, 4), util_split.ORIGIN, util_split.RADIUS)
        worst = max(worst, abs(ours - ref) / (H * W))
    assert worst <= sp.ROI_TOLERANCE, worst


def test_roi_decision_equals_torch_expression():
    """count_nonzero / numel is fp32 and the threshold is rounded to fp32, including views above 2^24 pixels"""
    import torch

    from nrw.prepare_data_split import roi_keep

    rng = np.random.default_rng(5)
    hw = [(67, 1001), (4097, 4097), (5000, 4000), (1, 1), (3, 7), (8191, 4099)]
    for H, W in hw:
        n = H * W
        cand = {0, n, n // 2, n // 3, n - 1, 1} | set(int(x) for x in rng.integers(0, n + 1, 40))
        for thr in (0.2, 0.5, 1 / 3, 0.1 + 1e-9, float(np.float32(0.5)) + 1e-12):
            for c in cand:
                tor = bool(torch.tensor(c, dtype=torch.int64) / n < thr)
                assert roi_keep([c], [(H, W)], thr)[0] == (not tor), (H, W, c, thr)
                # the share itself is the fp32 division torch computes
                assert np.float32(c) / np.float32(n) == (torch.tensor(c, dtype=torch.int64) / n).item()


def test_port_counts_equal_brute_force_geometry():
    """the restatement's inside test on a camera at the sphere centre (every pixel) and one facing away (none)"""
    K = np.array([[50.0, 0, 20.0], [0, 50.0, 15.0], [0, 0, 1]], np.float32)
    c2w = np.eye(3, 4, dtype=np.float32)
    assert sp.roi_count(30, 40, K, c2w, [0, 0, 0], 1.0) == 1200
    c2w[:, 3] = [0, 0, -5]                       # looking down -z from z = -5, away from the sphere at the origin
    assert sp.roi_count(30, 40, K, c2w, [0, 0, 0], 1.0) == 0
    assert sp.roi_count(30, 40, K, c2w, [0, 0, -10], 4.0) == 1200     # the sphere fills the view
    o, d = sp.rays_rows(3, 9, 40, K, c2w)
    from oracle import cache_port

    co, cd, _ = cache_port.rays(30, 40, K, c2w)
    assert o.tobytes() == co[3 * 40:9 * 40].tobytes() and d.tobytes() == cd[3 * 40:9 * 40].tobytes()


def _run_reference_script(root, seed, argv):
    R = _ref()
    import pandas  # noqa: F401  (real pandas writes the reference's tsv)

    old = sys.argv
    sys.argv = ["prepare_data_split.py", "--root_dir", root] + argv
    try:
        np.random.seed(seed)
        runpy.run_path(R.script, run_name="__main__")
    finally:
        sys.argv = old


@pytest.mark.parametrize("seed,min_obs,roi,static,num_test", [(0, -1, 0.2, 0.6, 2), (7, 3, 0.35, 0.5, 3), (1, 3, 0.0, -1.0, 0)])
def test_tsv_and_trash_equal_reference_script(scene, tmp_path, cpu_cuda, port_counts, seed, min_obs, roi, static, num_test):
    """the unmodified prepare_data_split.py after np.random.seed(seed) with real pandas writes the same tsv bytes and
    trash_images names as prepare() with --seed"""
    pytest.importorskip("pandas")
    P = port_counts
    flags = {"num_test": num_test, "min_observation": min_obs, "roi_threshold": roi, "static_threshold": static}
    argv = sum([[f"--{k}", str(v)] for k, v in flags.items()], [])
    _run_reference_script(scene, seed, argv)
    tsv = os.path.join(scene, "split_scene.tsv")
    ref_bytes = open(tsv, "rb").read()
    ref_trash = sorted(os.listdir(os.path.join(scene, "trash_images")))
    os.remove(tsv)
    res = P.prepare(_args(scene, seed=seed, **flags))
    assert res["tsv"] == tsv
    assert open(tsv, "rb").read() == ref_bytes
    assert sorted(os.listdir(os.path.join(scene, "trash_images"))) == ref_trash
    if static >= 0:
        assert f"transient_much_{util_split.FULLY_TRANSIENT}" in ref_trash
    if min_obs == 3:
        assert f"less_covis_{util_split.COVIS_DROPPED}" in ref_trash
        assert f"less_covis_{util_split.COVIS_RESCUED}" not in ref_trash
    assert len(ref_bytes.splitlines()) == len(res["names"]) + 1


def test_tsv_bytes_equal_pandas():
    pd = pytest.importorskip("pandas")
    from nrw.prepare_data_split import split_rows, tsv_bytes

    names = np.array(["a.jpg", "b c.png", 'q"uote.jpg', "t\tab.jpg", "x,y.jpg", "ünï.png"])
    rows = split_rows(list(names), 2, "scene")
    n = len(names)
    content = np.concatenate((names[:, None], np.arange(n)[:, None],
                              np.concatenate((np.repeat("test", 2), np.repeat("train", n - 2)))[:, None],
                              np.repeat("scene", n)[:, None]), 1)
    import io

    buf = io.BytesIO()
    pd.DataFrame(content, columns=["filename", "id", "split", "dataset"]).to_csv(buf, sep="\t", index=False)
    assert tsv_bytes(rows) == buf.getvalue()


def test_label_ids_match_reference_mapping():
    from nrw.prepare_data_split import TRANSIENT_OBJECTS
    from nrw.renderer import LABEL_IDS

    m = _ref().get_label_id_mapping()
    for k, v in LABEL_IDS.items():
        assert m[k] == v, k
    assert set(TRANSIENT_OBJECTS) <= set(LABEL_IDS) and LABEL_IDS["tree"] == 4


# ---- deviations ---------------------------------------------------------------------------------------------------
def test_deviation_seeded_permutation(scene, port_counts):
    P = port_counts
    a = P.prepare(_args(scene, seed=3, num_test=1, static_threshold=-1))["names"]
    b = P.prepare(_args(scene, seed=3, num_test=1, static_threshold=-1))["names"]
    c = P.prepare(_args(scene, seed=4, num_test=1, static_threshold=-1))["names"]
    assert a == b and a != c and sorted(a) == sorted(c)
    kept = P.view_selection(scene, util_split.ORIGIN, util_split.RADIUS, -1, 0.5)
    assert a == list(np.random.RandomState(3).permutation(kept))


def test_deviation_trash_is_a_byte_copy(scene, port_counts):
    P = port_counts
    P.prepare(_args(scene, num_test=1, min_observation=3, roi_threshold=0.5, static_threshold=0.3))
    trash = os.listdir(os.path.join(scene, "trash_images"))
    assert trash
    for t in trash:
        name = t.split("_", 2)[-1] if t.startswith(("less_ROI_", "less_covis_")) else t[len("transient_much_"):]
        src = open(os.path.join(scene, "dense/images", name), "rb").read()
        assert open(os.path.join(scene, "trash_images", t), "rb").read() == src


def test_deviation_non_pinhole_raises(scene, port_counts):
    from nrw._lib import NrwError

    util_split.set_camera_model(scene, 2)
    with pytest.raises(NrwError, match="PINHOLE"):
        port_counts.view_selection(scene, util_split.ORIGIN, util_split.RADIUS, -1, 0.2)


def test_deviation_scene_name_of_normalised_root(scene, port_counts):
    res = port_counts.prepare(_args(scene + "/", num_test=1, static_threshold=-1))
    assert os.path.basename(res["tsv"]) == "split_scene.tsv"
    lines = open(res["tsv"]).read().splitlines()
    assert all(line.split("\t")[3] == "split_scene" for line in lines[1:])


def test_deviation_errors(scene, port_counts):
    from nrw._lib import NrwError

    P = port_counts
    with pytest.raises(NrwError, match="num_test"):
        P.prepare(_args(scene, num_test=100, static_threshold=-1))
    with pytest.raises(NrwError, match="sparse_filtered_5"):
        P.prepare(_args(scene, min_observation=5))
    with pytest.raises(NrwError, match="no image"):
        P.prepare(_args(scene, roi_threshold=1.5, static_threshold=-1))
    os.remove(os.path.join(scene, "semantic_maps", "img_002.npz"))
    with pytest.raises(NrwError, match="semantic map"):
        P.prepare(_args(scene, roi_threshold=0.0, num_test=1))


def test_deviation_negative_static_threshold_reads_no_map(scene, port_counts):
    shutil.rmtree(os.path.join(scene, "semantic_maps"))
    res = port_counts.prepare(_args(scene, num_test=2, roi_threshold=0.0, static_threshold=-0.5,
                                    nima_ckpt_path="/nonexistent/nima.pth"))
    assert sorted(res["names"]) == [f"img_{i:03d}.png" for i in range(len(util_split.CAMERAS))]


def test_cli_parses_reference_flags():
    from nrw.prepare_data_split import get_opts

    a = get_opts(["--root_dir", "/x/brandenburg_gate", "--num_test", "10", "--min_observation", "-1", "--roi_threshold", "0",
                  "--static_threshold", "0", "--nima_ckpt_path", "weights/nima.pth", "--semantic_map_path", "semantic_maps"])
    assert (a.num_test, a.min_observation, a.roi_threshold, a.static_threshold, a.seed) == (10, -1, 0.0, 0.0, 0)
    d = get_opts(["--root_dir", "x"])
    assert (d.num_test, d.min_observation, d.roi_threshold, d.static_threshold, d.semantic_map_path) == \
        (10, -1, 0.5, 0.6, "semantic_maps")


# ---- argument checks of the C exports -----------------------------------------------------------------------------
def _lib_or_skip():
    from nrw import _lib

    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("libnrw.so not built")
    return _lib.lib()


def test_viewsel_exports_reject_bad_arguments():
    L = _lib_or_skip()
    dummy = C.c_void_p(16)
    o = (C.c_float * 3)(0.0, 0.0, 0.0)
    bad_o = (C.c_float * 3)(0.0, float("nan"), 0.0)
    ok = dict(views=dummy, hw=dummy, n=4, max_hw=100, o=o, r=1.0, counts=dummy)

    def roi(**kw):
        a = dict(ok, **kw)
        return L.nrw_view_roi_count(a["views"], a["hw"], a["n"], a["max_hw"], a["o"], a["r"], a["counts"], None)

    assert roi(n=0) == -1
    assert roi(max_hw=0) == -1
    assert roi(max_hw=1 << 31) == -1
    for r in (0.0, -1.0, float("nan"), float("inf")):
        assert roi(r=r) == -1, r
    assert roi(o=bad_o) == -1
    assert roi(o=None) == -1
    assert roi(views=None) == -1 and roi(hw=None) == -1 and roi(counts=None) == -1
    ids = (C.c_int * 9)(*range(9))
    assert L.nrw_label_static_count(dummy, 10, ids, 9, dummy, None) == -1
    assert L.nrw_label_static_count(dummy, 10, ids, -1, dummy, None) == -1
    assert L.nrw_label_static_count(dummy, -1, ids, 3, dummy, None) == -1
    assert L.nrw_label_static_count(None, 10, ids, 3, dummy, None) == -1
    assert L.nrw_label_static_count(dummy, 10, ids, 3, None, None) == -1
    assert L.nrw_label_static_count(dummy, 10, None, 3, dummy, None) == -1
    big = (C.c_int * 1)(1 << 24)
    assert L.nrw_label_static_count(dummy, 10, big, 1, dummy, None) == -1
