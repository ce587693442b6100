"""Ground-truth alignment check without a GPU: the numpy restatement oracle/trackerr_port.py against the unmodified
tools/reproj_error.py (get_gt_point track by track, image_reproj_error, the whole gt_reproject_error) on a seeded scene
built for exact comparison, the golden file against a fresh reference run, each documented deviation, the track reader,
and nrw.reproj_error's host logic with the restatement in place of the two device kernels."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from oracle import make_reproj_golden as mg
from oracle import ref_import
from oracle import trackerr_port as tp
from conftest import GOLDEN

GOLDEN_FILE = os.path.join(GOLDEN, "reproj_error.npz")


@pytest.fixture
def cpu_cuda(monkeypatch):
    """the reference calls .cuda(); on the CPU it is the identity"""
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)


@pytest.fixture(scope="module")
def scene():
    return tp.make_scene(seed=mg.SEED)


def _ref():
    if not ref_import.available():
        pytest.skip("reference tree not present")
    return tp.load_reference()


def _read(d):
    from nrw import colmap

    base = os.path.join(d, "dense", "sparse")
    im = colmap.read_images(os.path.join(base, "images.bin"), with_points=True)
    cams = colmap.read_cameras(os.path.join(base, "cameras.bin"))
    pts = colmap.read_points3d(os.path.join(base, "points3D.bin"), with_tracks=True)
    return im, cams, pts


def _oracle_run(d, sc, gt=None, **kw):
    from nrw import reproj_error as R

    im, cams, pts = _read(d)
    img_ids, _ = R.get_image_id(im, d)
    ims = {k: v[0] for k, v in im.items()}
    E = dict(zip(img_ids, R.get_entrinsics(ims, img_ids)))
    K, _ = R.get_intrinsic(cams, img_ids, ims)
    views = {k: (v[1], v[2]) for k, v in im.items()}
    args = dict(track_length=sc["track_length"], reproj_error=sc["reproj_error"], img_reproj_error=sc["img_reproj_error"])
    args.update(kw)
    return tp.gt_reproject_error(img_ids, views, K, E, pts, sc["gt"] if gt is None else gt, np.array(sc["sfm2gt"]), **args)


@pytest.fixture
def port_kernels(monkeypatch):
    """nrw.reproj_error with the restatement in place of the two device kernels"""
    from nrw import reproj_error as R

    def first_hits(points, intrinsics, world_to_cams, query_view, query_xy, device=0, map_pixels=None):
        views = np.stack([tp.view_row(K, E) for K, E in zip(intrinsics, world_to_cams)])
        return torch.as_tensor(tp.first_hit(np.asarray(points, np.float32), views, query_view, query_xy))

    def obs_errors(X, view, xy, projections, device=0, with_uv=False):
        e, uv = tp.obs_error(X, view, np.asarray(xy, np.float64), np.asarray(projections).reshape(-1, 3, 4))
        return (torch.as_tensor(e), torch.as_tensor(uv)) if with_uv else torch.as_tensor(e)

    monkeypatch.setattr(R, "first_hits", first_hits)
    monkeypatch.setattr(R, "obs_errors", obs_errors)
    return R


def _run_ref(ref, d, gp, sc, batch_size=2, **kw):
    args = dict(track_length=sc["track_length"], reproj_error=sc["reproj_error"], img_reproj_error=sc["img_reproj_error"])
    args.update(kw)
    cwd = os.getcwd()
    os.chdir(d)
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            loss = ref.gt_reproject_error(d, gp, np.array(sc["sfm2gt"]), "dense/sparse", args["track_length"],
                                          args["reproj_error"], batch_size, args["img_reproj_error"])
    finally:
        os.chdir(cwd)
    return float(loss), np.asarray(ref.plt.plot.call_args[0][1], np.float64)


def test_read_points3d_tracks_match_reference(tmp_path, scene):
    ref = _ref()
    tp.write_scene(str(tmp_path), scene)
    _, _, pts = _read(str(tmp_path))
    rp = ref.read_points3d_binary(str(tmp_path / "dense" / "sparse" / "points3D.bin"))
    assert list(pts["id"]) == list(rp.keys())
    off = pts["track_offsets"]
    for r, p in enumerate(rp.values()):
        assert np.array_equal(pts["track_image_id"][off[r]:off[r + 1]], p.image_ids)
        assert np.array_equal(pts["track_point2d_idx"][off[r]:off[r + 1]], p.point2D_idxs)
        assert pts["track_length"][r] == len(p.point2D_idxs)
    plain = _read_plain(str(tmp_path))
    assert set(plain) == {"id", "xyz", "rgb", "error", "track_length"}


def _read_plain(d):
    from nrw import colmap

    return colmap.read_points3d(os.path.join(d, "dense", "sparse", "points3D.bin"))


def test_get_gt_point_track_by_track(tmp_path, scene, cpu_cuda):
    """the unmodified get_gt_point on each track's reference observation equals the restatement's first hit"""
    ref = _ref()
    gp = tp.write_scene(str(tmp_path), scene)
    r = _oracle_run(str(tmp_path), scene)
    assert (r["gt_index"] >= 0).all()
    gt = torch.from_numpy(np.asarray(ref.o3d.io.read_point_cloud(gp).points)).float()
    S = np.array(scene["sfm2gt"])
    first = np.searchsorted(r["obs_track"], np.arange(len(r["track_point_ids"])))
    ids = list(scene["ids"])
    for t, f in enumerate(first):
        k = ids.index(int(r["kept_views"][r["obs_view"][f]]))
        cam2gt = torch.from_numpy(S @ np.linalg.inv(scene["E"][k]))[None].float()
        K = torch.from_numpy(scene["K"][k])[None].float()
        q = torch.tensor([[0.0, 0.0, *r["obs_xy"][f]]]).float()
        row = ref.get_gt_point(gt, cam2gt, K, q).reshape(-1, 4)[0, :3]
        assert torch.equal(row, gt[r["gt_index"][t]]), t


def test_image_reproj_error_matches_reference(tmp_path, scene, cpu_cuda):
    ref = _ref()
    tp.write_scene(str(tmp_path), scene)
    d = str(tmp_path)
    base = os.path.join(d, "dense", "sparse")
    imdata = ref.read_images_binary(os.path.join(base, "images.bin"))
    camdata = ref.read_cameras_binary(os.path.join(base, "cameras.bin"))
    pts3d = ref.read_points3d_binary(os.path.join(base, "points3D.bin"))
    img_ids, _ = ref.get_image_id(imdata, d)
    E = ref.get_entrinsics(imdata, img_ids)
    Ed = {i: E[k] for k, i in enumerate(img_ids)}
    K, _ = ref.get_intrinsic(camdata, img_ids, imdata)
    with contextlib.redirect_stderr(io.StringIO()):
        want = ref.image_reproj_error(imdata, pts3d, img_ids, Ed, K).numpy()[:, 0]
    r = _oracle_run(d, scene)
    np.testing.assert_allclose(r["image_errors"], want, rtol=0, atol=1e-3)
    assert list(r["kept_views"]) == [i for i, e in zip(img_ids, want) if e < scene["img_reproj_error"]]
    assert len(r["kept_views"]) == len(img_ids) - 1          # the scene has one view with bad keypoints


def test_whole_check_matches_reference_and_golden(tmp_path, scene, cpu_cuda):
    ref = _ref()
    d = str(tmp_path)
    gp = tp.write_scene(d, scene)
    loss, errors = _run_ref(ref, d, gp, scene)
    r = _oracle_run(d, scene)
    assert r["obs_used"].all()
    np.testing.assert_allclose(r["errors"], errors, rtol=0, atol=1e-3)
    assert abs(r["loss"] - loss) < 1e-4
    np.testing.assert_array_equal(ref.written["samples/reproject/colmap_sfm.ply"], scene["pt_xyz"][
        np.searchsorted(scene["pt_id"], r["track_point_ids"])])
    # the golden file holds the same scene and the same reference rows
    z = np.load(GOLDEN_FILE, allow_pickle=False)
    g = mg.unpack(z)
    assert np.array_equal(g["gt"], scene["gt"]) and np.array_equal(g["sfm2gt"], scene["sfm2gt"])
    assert all(np.array_equal(a, b) for a, b in zip(g["track"], scene["track"]))
    assert all(np.array_equal(a, b) for a, b in zip(g["xys"], scene["xys"]))
    assert float(z["ref_loss"]) == loss
    np.testing.assert_array_equal(z["ref_errors"], errors)
    np.testing.assert_array_equal(z["ref_gt_index"], r["gt_index"])


def test_module_host_logic_and_files(tmp_path, scene, port_kernels, capsys):
    """nrw.reproj_error (restatement kernels) writes the reference's rows and images"""
    R = port_kernels
    d = str(tmp_path / "scene")
    gp = tp.write_scene(d, scene)
    r = _oracle_run(d, scene)
    work = tmp_path / "work"
    work.mkdir()
    cwd = os.getcwd()
    os.chdir(work)
    try:
        loss = R.gt_reproject_error(d, gp, np.array(scene["sfm2gt"]), "dense/sparse", scene["track_length"],
                                    scene["reproj_error"], 2, scene["img_reproj_error"])
    finally:
        os.chdir(cwd)
    assert loss == r["loss"]
    out = capsys.readouterr().out
    assert f"selected {len(r['kept_views'])} view for testing." in out
    assert f"avg re-projection error {r['loss']}, {len(r['errors'])}/{len(r['obs_view'])}, 0 tracks" in out
    from nrw.mesh import read_ply

    sfm = read_ply(str(work / "samples" / "reproject" / "colmap_sfm.ply"))["vertices"]
    np.testing.assert_array_equal(sfm, scene["pt_xyz"][np.searchsorted(scene["pt_id"], r["track_point_ids"])])
    S_inv = np.linalg.inv(np.array(scene["sfm2gt"]))
    g = scene["gt"][r["gt_index"]].astype(np.float64)
    np.testing.assert_allclose(read_ply(str(work / "samples" / "reproject" / "gt.ply"))["vertices"],
                               (S_inv[:3, :3] @ g.T).T + S_inv[:3, 3], rtol=0, atol=1e-12)
    pngs = sorted(os.listdir(work / "reprojects"))
    names = dict(zip(scene["ids"].tolist(), scene["names"].tolist()))
    assert pngs == sorted(f"{names[int(i)]}.png" for i in np.unique(r["kept_views"][r["obs_view"]]))
    from PIL import Image

    k = int(r["kept_views"][r["obs_view"][0]])
    img = np.asarray(Image.open(work / "reprojects" / f"{names[k]}.png"))
    m = r["kept_views"][r["obs_view"]] == k
    red = np.trunc(r["obs_xy"][m]).astype(np.int64)
    assert (img[red[:, 1], red[:, 0]] == (255, 0, 0)).all()
    assert img.shape == (int(scene["wh"][0][1]), int(scene["wh"][0][0]), 3)


def test_deviation_no_hit_track_is_dropped_and_reference_depends_on_batch(tmp_path, scene, cpu_cuda, port_kernels):
    """deviation 1: a track whose reference pixel gets no GT point.  The reference takes GT point 0 for it when another
    track of its batch hits, and raises from torch.max of an empty tensor when it is alone in its batch."""
    ref = _ref()
    d = str(tmp_path)
    tp.write_scene(d, scene)
    r0 = _oracle_run(d, scene)
    first = np.searchsorted(r0["obs_track"], np.arange(len(r0["track_point_ids"])))
    t = 0                                        # remove every GT point on the first track's reference pixel
    k = list(scene["ids"]).index(int(r0["kept_views"][r0["obs_view"][first[t]]]))
    view = tp.view_row(scene["K"][k], scene["E"][k] @ np.linalg.inv(scene["sfm2gt"]))
    pu, pv, _, front = tp.pixels(scene["gt"], view)
    qx, qy = np.rint(r0["obs_xy"][first[t]].astype(np.float32).astype(np.float64))
    gt = scene["gt"][~(front & (pu == qx) & (pv == qy))]
    gp = str(tmp_path / "gt_miss.ply")
    from nrw.mesh import write_ply

    write_ply(gp, gt)
    r = _oracle_run(d, scene, gt=gt)
    assert r["gt_index"][t] == -1 and (r["gt_index"][1:] >= 0).all()
    assert not r["obs_used"][r["obs_track"] == t].any()
    loss2, err2 = _run_ref(ref, d, gp, scene, batch_size=2)
    assert len(err2) == len(r["obs_view"])              # the reference keeps the track, with GT point 0
    assert abs(loss2 - r["loss"]) > 1e-3
    with pytest.raises(RuntimeError):
        _run_ref(ref, d, gp, scene, batch_size=1)
    # nrw counts the track and drops it from the mean; the batch size changes nothing
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        with contextlib.redirect_stdout(io.StringIO()) as out:
            losses = [port_kernels.gt_reproject_error(d, gp, np.array(scene["sfm2gt"]), "dense/sparse", scene["track_length"],
                                                      scene["reproj_error"], b, scene["img_reproj_error"]) for b in (1, 2)]
    finally:
        os.chdir(cwd)
    assert losses[0] == losses[1] == r["loss"]
    assert f"{int(r['obs_used'].sum())}/{len(r['obs_view'])}, 1 tracks without" in out.getvalue()


def test_deviation_invalid_keypoints_left_out(tmp_path, scene, cpu_cuda):
    """deviation 2: keypoints with point3D id -1 or an id missing from points3D.bin.  The reference projects the point
    with the largest id for -1 and a row of ones for a missing id; nrw leaves both out of the view's mean."""
    ref = _ref()
    sc = dict(scene)
    sc["xys"], sc["pids"] = scene["xys"].copy(), scene["pids"].copy()
    k = 4
    sc["xys"][k] = np.concatenate([scene["xys"][k], [[10.0, 10.0], [20.0, 30.0]]])
    sc["pids"][k] = np.concatenate([scene["pids"][k], [-1, 1001]])
    empty = 5                                   # a tested view whose every keypoint is invalid
    sc["pids"][empty] = np.full(len(scene["pids"][empty]), -1)
    sc["track"] = np.array([np.array([p for p in t if p[0] != scene["ids"][empty]]).reshape(-1, 2)
                            for t in scene["track"]] + [None], dtype=object)[:-1]
    d = str(tmp_path)
    tp.write_scene(d, sc)
    base = os.path.join(d, "dense", "sparse")
    imdata = ref.read_images_binary(os.path.join(base, "images.bin"))
    pts3d = ref.read_points3d_binary(os.path.join(base, "points3D.bin"))
    img_ids, _ = ref.get_image_id(imdata, d)
    E = ref.get_entrinsics(imdata, img_ids)
    K, _ = ref.get_intrinsic(ref.read_cameras_binary(os.path.join(base, "cameras.bin")), img_ids, imdata)
    with contextlib.redirect_stderr(io.StringIO()):
        want = ref.image_reproj_error(imdata, pts3d, img_ids, {i: E[j] for j, i in enumerate(img_ids)}, K).numpy()[:, 0]
    r = _oracle_run(d, sc)
    pos = img_ids.index(int(sc["ids"][k]))
    assert abs(r["image_errors"][pos] - want[pos]) > 1.0        # the reference counts the two invalid keypoints
    others = [j for j in range(len(img_ids)) if j != pos and img_ids[j] != int(sc["ids"][empty])]
    np.testing.assert_allclose(r["image_errors"][others], want[others], rtol=0, atol=1e-3)
    e = img_ids.index(int(sc["ids"][empty]))
    assert np.isnan(r["image_errors"][e]) and int(sc["ids"][empty]) not in r["kept_views"]


def test_deviation_fp64_projection_at_a_pixel_edge(cpu_cuda):
    """deviation 3: a point 4e-7 px past a pixel edge in fp64 is on pixel 11; the reference's fp32 projection rounds it
    to 10.5 and then, half to even, to pixel 10, so it picks the farther point B instead"""
    ref = _ref()
    a = np.float32(np.nextafter(np.float32(0.105), np.float32(1)))
    pts = np.array([[a, 0.0, 1.0], [0.112, 0.0, 2.0]], np.float32)
    pts[1, 0] = np.float32(0.112 * 2.0)                          # u = 11.2 at depth 2
    K = np.array([[100.0, 0, 0], [0, 100.0, 0], [0, 0, 1]], np.float32)
    hit = tp.first_hit(pts, tp.view_row(K, np.eye(4))[None], [0], np.array([[11.2, 0.0]], np.float32))
    assert hit[0] == 0
    row = ref.get_gt_point(torch.from_numpy(pts), torch.eye(4)[None], torch.from_numpy(K)[None],
                           torch.tensor([[0.0, 0.0, 11.2, 0.0]]))
    assert torch.equal(row.reshape(-1, 4)[0, :3], torch.from_numpy(pts[1]))


def test_get_image_id_skips_the_first_two_names(tmp_path, scene):
    from nrw import reproj_error as R

    d = str(tmp_path)
    tp.write_scene(d, scene)
    im, _, _ = _read(d)
    ids, names = R.get_image_id(im, d)
    assert ids == [int(i) for i in scene["ids"][2:]]
    assert names[int(scene["ids"][0])] == scene["names"][0]
    open(os.path.join(d, "dense", "images", "zz_not_in_model.jpg"), "wb").close()
    with pytest.raises(KeyError):
        R.get_image_id(im, d)
