"""GPU: the ground-truth alignment check (csrc/gtproj.cu, nrw.reproj_error) against the restatement
oracle/trackerr_port.py with exact index equality (duplicates, shared pixels, pixels outside the image, misses, points
behind the camera, several passes), the error kernel within 1e-9 px, the whole check against the reference rows of
tests/golden/reproj_error.npz, the CLI in a temporary working directory, repeatability and every NrwError case."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, PKG, ROOT
from oracle import make_reproj_golden as mg
from oracle import trackerr_port as tp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return mg.unpack(np.load(os.path.join(GOLDEN, "reproj_error.npz"), allow_pickle=False)), \
        np.load(os.path.join(GOLDEN, "reproj_error.npz"), allow_pickle=False)


@pytest.fixture(scope="module")
def scene_dir(tmp_path_factory, golden):
    d = str(tmp_path_factory.mktemp("gtproj") / "scene")
    gp = tp.write_scene(d, golden[0])
    return d, gp


def _views(n, rng, w=40, h=30):
    Ks, Es = [], []
    for _ in range(n):
        a = rng.normal(size=3) * 0.2
        c, s = np.cos(a), np.sin(a)
        R = (np.array([[1, 0, 0], [0, c[0], -s[0]], [0, s[0], c[0]]]) @ np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]]))
        E = np.eye(4)
        E[:3, :3], E[:3, 3] = R, [rng.normal() * 0.1, rng.normal() * 0.1, 3.0]
        Es.append(E)
        Ks.append(np.array([[35.0, 0, w / 2 + 0.3], [0, 34.0, h / 2 - 0.2], [0, 0, 1]], np.float32))
    return Ks, Es


def _adversarial(seed=5, n=40000, n_views=20):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1.5, 1.5, (n, 3)).astype(np.float32)
    pts[:2000, 2] = rng.uniform(-6, -3.5, 2000)             # behind every camera (z_cam < 0)
    pts = np.concatenate([pts, pts[rng.choice(n, 3000)]])    # exact duplicates at later indices
    Ks, Es = _views(n_views, rng)
    qv = rng.integers(0, n_views, 3000)
    qxy = rng.uniform(-8, 48, (3000, 2)).astype(np.float32)  # inside and outside the 40 x 30 image
    qxy[::7] = qxy[1::7][: len(qxy[::7])]                    # queries that share a pixel
    qv[::7] = qv[1::7][: len(qv[::7])]
    qxy[::11] += 300.0                                       # far outside: no point lands there
    return pts, Ks, Es, qv, qxy


def _oracle_hits(pts, Ks, Es, qv, qxy):
    return tp.first_hit(pts, np.stack([tp.view_row(K, E) for K, E in zip(Ks, Es)]), qv, qxy)


def test_first_hit_matches_oracle_and_pass_layout():
    from nrw import reproj_error as R

    pts, Ks, Es, qv, qxy = _adversarial()
    want = _oracle_hits(pts, Ks, Es, qv, qxy)
    assert (want == -1).any() and (want >= 0).sum() > 1000
    one = R.first_hits(pts, Ks, Es, qv, qxy).cpu().numpy()
    np.testing.assert_array_equal(one, want)
    # the largest box fills the whole map: one view per pass
    pix = np.rint(qxy).astype(np.int64)
    areas = [np.prod(pix[qv == v].max(0) - pix[qv == v].min(0) + 1) if (qv == v).any() else 0 for v in range(len(Ks))]
    many = R.first_hits(pts, Ks, Es, qv, qxy, map_pixels=int(max(areas))).cpu().numpy()
    np.testing.assert_array_equal(many, want)


def test_first_hit_duplicates_go_to_the_smaller_index():
    from nrw import reproj_error as R

    K = np.array([[10.0, 0, 0], [0, 10.0, 0], [0, 0, 1]], np.float32)
    p = np.array([[0.3, 0.2, 2.0], [0.1, 0.1, 1.0], [0.3, 0.2, 2.0], [0.1, 0.1, 1.0], [-0.1, -0.1, -1.0]], np.float32)
    q = np.array([[1.0, 1.0], [1.4, 0.6], [2.0, 1.0], [5.0, 5.0]], np.float32)
    hit = R.first_hits(p, [K], [np.eye(4)], [0, 0, 0, 0], q)
    # (1, 1): points 1 and 3 (depth 1) and 4 (behind the camera, same pixel); (2, 1): points 0 and 2 (u = 1.5 rounds
    # half to even); (5, 5): nothing
    assert hit.cpu().tolist() == [1, 1, 0, -1]


def test_obs_error_kernel_matches_oracle():
    from nrw import reproj_error as R

    rng = np.random.default_rng(3)
    Ks, Es = _views(7, rng)
    P = np.stack([tp.projection(K, E) for K, E in zip(Ks, Es)])
    X = rng.normal(size=(5000, 3))
    v = rng.integers(0, 7, 5000)
    xy = rng.uniform(0, 40, (5000, 2))
    err, uv = R.obs_errors(X, v, xy, P, with_uv=True)
    we, wuv = tp.obs_error(X, v, xy, P)
    np.testing.assert_allclose(err.cpu().numpy(), we, rtol=0, atol=1e-9)
    np.testing.assert_allclose(uv.cpu().numpy(), wuv, rtol=0, atol=1e-9)


def test_track_errors_match_golden(golden, scene_dir):
    from nrw import reproj_error as R

    sc, z = golden
    d, gp = scene_dir
    r = R.track_errors(d, gp, sc["sfm2gt"], "dense/sparse", sc["track_length"], sc["reproj_error"], sc["img_reproj_error"])
    np.testing.assert_array_equal(r["gt_index"], z["ref_gt_index"])
    np.testing.assert_allclose(r["errors"], z["ref_errors"], rtol=0, atol=1e-3)
    assert abs(r["loss"] - float(z["ref_loss"])) < 1e-4
    np.testing.assert_array_equal(r["track_xyz"], z["ref_colmap_sfm"])
    # kept views and every row equal the restatement's
    from test_reproj_error_cpu import _oracle_run

    o = _oracle_run(d, sc)
    np.testing.assert_array_equal(r["kept_views"], o["kept_views"])
    np.testing.assert_array_equal(r["gt_index"], o["gt_index"])
    np.testing.assert_allclose(r["errors"], o["errors"], rtol=0, atol=1e-9)
    # two runs give identical bits
    r2 = R.track_errors(d, gp, sc["sfm2gt"], "dense/sparse", sc["track_length"], sc["reproj_error"], sc["img_reproj_error"])
    assert r2["loss"] == r["loss"] and r2["errors"].tobytes() == r["errors"].tobytes()
    assert r2["image_errors"].tobytes() == r["image_errors"].tobytes()


def test_cli_end_to_end(golden, scene_dir, tmp_path):
    from nrw.mesh import read_ply
    from PIL import Image

    sc, z = golden
    d, gp = scene_dir
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    out = subprocess.run([sys.executable, "-m", "nrw.reproj_error", "--data_dir", d, "--gt_pcd_path", gp, "--track_length",
                          str(sc["track_length"]), "--reproj_error", str(sc["reproj_error"]), "--img_reproj_error",
                          str(sc["img_reproj_error"])], cwd=tmp_path, env=env, capture_output=True, text=True, check=True)
    assert "selected 5 view for testing." in out.stdout
    assert f"/{len(z['ref_errors'])}, 0 tracks without" in out.stdout
    np.testing.assert_array_equal(read_ply(str(tmp_path / "samples/reproject/colmap_sfm.ply"))["vertices"], z["ref_colmap_sfm"])
    S_inv = np.linalg.inv(sc["sfm2gt"])
    g = sc["gt"][z["ref_gt_index"]].astype(np.float64)
    np.testing.assert_allclose(read_ply(str(tmp_path / "samples/reproject/gt.ply"))["vertices"],
                               (S_inv[:3, :3] @ g.T).T + S_inv[:3, 3], rtol=0, atol=1e-12)
    pngs = sorted(os.listdir(tmp_path / "reprojects"))
    assert len(pngs) == 5
    img = np.asarray(Image.open(tmp_path / "reprojects" / pngs[0]))
    assert img.shape == (int(sc["wh"][0][1]), int(sc["wh"][0][0]), 3)
    assert ((img == (255, 0, 0)).all(-1)).any() and ((img == (0, 255, 0)).all(-1) | (img == (255, 0, 0)).all(-1)
                                                     | (img == 0).all(-1)).all()


def test_errors(golden, scene_dir, tmp_path):
    from nrw import reproj_error as R
    from nrw._lib import NrwError
    from nrw.mesh import write_ply

    sc, _ = golden
    d, gp = scene_dir
    args = ("dense/sparse", sc["track_length"], sc["reproj_error"])
    with pytest.raises(NrwError, match="not found"):
        R.track_errors(d, str(tmp_path / "none.ply"), sc["sfm2gt"], *args, sc["img_reproj_error"])
    bad = sc["gt"].copy()
    bad[3, 1] = np.nan
    write_ply(str(tmp_path / "nan.ply"), bad)
    with pytest.raises(NrwError, match="non-finite"):
        R.track_errors(d, str(tmp_path / "nan.ply"), sc["sfm2gt"], *args, sc["img_reproj_error"])
    with pytest.raises(NrwError, match="no view"):
        R.track_errors(d, gp, sc["sfm2gt"], *args, 0.0)
    with pytest.raises(NrwError, match="no track"):
        R.track_errors(d, gp, sc["sfm2gt"], "dense/sparse", 10 ** 6, sc["reproj_error"], sc["img_reproj_error"])
    write_ply(str(tmp_path / "far.ply"), np.full((1, 3), 1e4, np.float32))
    with pytest.raises(NrwError, match="no track's reference pixel"):
        R.track_errors(d, str(tmp_path / "far.ply"), sc["sfm2gt"], *args, sc["img_reproj_error"])
    with pytest.raises(NrwError, match="config.yaml"):
        R.main(["--data_dir", str(tmp_path), "--gt_pcd_path", gp])
    with pytest.raises(NrwError, match="2\\^32"):
        R.first_hits(torch.empty(1 << 32, 3, dtype=torch.float32, device="meta"), [], [], [], np.zeros((0, 2)))
    K = np.eye(3, dtype=np.float32)
    with pytest.raises(NrwError, match="view index"):
        R.first_hits(np.zeros((1, 3)), [K], [np.eye(4)], [1], np.zeros((1, 2)))
    import shutil

    # a non-PINHOLE camera
    d2 = str(tmp_path / "radial")
    shutil.copytree(d, d2)
    cams = [(k + 1, 2, int(w), int(h), (K_[0, 0], K_[0, 2], K_[1, 2], 0.0)) for k, (K_, (w, h)) in enumerate(zip(sc["K"], sc["wh"]))]
    tp.write_cameras(os.path.join(d2, "dense", "sparse", "cameras.bin"), cams)
    with pytest.raises(NrwError, match="PINHOLE"):
        R.track_errors(d2, gp, sc["sfm2gt"], *args, sc["img_reproj_error"])
