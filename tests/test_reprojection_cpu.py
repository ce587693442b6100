"""CPU checks of the visibility filter: the COLMAP readers and camera helpers of nrw.reprojection against the
unmodified reference (utils/reproj_filter.py, tools/reproj_error.py, utils/colmap_utils.py), the numpy restatement
oracle/reproj_port.py against the reference's back-projection and against analytic scenes, and the argument checks of
the nrw_raster_* / nrw_reproject_* exports."""
import os

import numpy as np
import pytest

from oracle import ref_import
from oracle import reproj_port as rp
from util_reproj import look_at, soup, two_sphere_mesh, view_matrix, write_scene

needs_ref = pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("scene"))
    S = write_scene(d, seed=3)
    return d, S


@pytest.fixture(scope="module")
def ref(scene):
    pytest.importorskip("pandas")
    return rp.load_reproj(scene[0])


@needs_ref
def test_colmap_readers_match_reference(ref, scene):
    from nrw.colmap import read_cameras, read_images

    sparse = os.path.join(scene[0], "dense", "sparse")
    ours, theirs = read_cameras(os.path.join(sparse, "cameras.bin")), ref.colmap_utils.read_cameras_binary(
        os.path.join(sparse, "cameras.bin"))
    assert list(ours) == list(theirs)
    for k, c in theirs.items():
        o = ours[k]
        assert (o.id, o.model, o.width, o.height) == (c.id, c.model, c.width, c.height)
        assert np.array_equal(o.params, c.params)
    ours, theirs = read_images(os.path.join(sparse, "images.bin")), ref.colmap_utils.read_images_binary(
        os.path.join(sparse, "images.bin"))
    assert list(ours) == list(theirs)
    for k, im in theirs.items():
        o = ours[k]
        assert (o.id, o.camera_id, o.name) == (im.id, im.camera_id, im.name)
        assert np.array_equal(o.qvec, im.qvec) and np.array_equal(o.tvec, im.tvec)
        assert np.array_equal(o.qvec2rotmat(), im.qvec2rotmat())


@needs_ref
def test_camera_helpers_match_reference(ref, scene):
    from nrw import reprojection as R
    from nrw.colmap import read_cameras, read_images

    d = scene[0]
    sparse = os.path.join(d, "dense", "sparse")
    im_o, cam_o = read_images(os.path.join(sparse, "images.bin")), read_cameras(os.path.join(sparse, "cameras.bin"))
    im_r = ref.colmap_utils.read_images_binary(os.path.join(sparse, "images.bin"))
    cam_r = ref.colmap_utils.read_cameras_binary(os.path.join(sparse, "cameras.bin"))
    a_o, b_o, p_o = R.get_image_id(im_o, d)
    a_r, b_r, p_r = ref.reproj_filter.get_image_id(im_r, d)
    assert (a_o, b_o, p_o) == (a_r, b_r, p_r)
    ids = R.get_train_ids(d, a_o, p_o)
    assert ids == ref.reproj_filter.get_train_ids(d, a_r, p_r) and len(ids) == 6       # the id-less train row is dropped
    assert np.array_equal(R.get_entrinsics(im_o, ids), ref.reproj_error.get_entrinsics(im_r, ids))
    K_o, wh_o = R.get_intrinsic(cam_o, ids, im_o)
    K_r, wh_r = ref.reproj_error.get_intrinsic(cam_r, ids, im_r)
    assert wh_o == wh_r
    for k in ids:
        assert K_o[k].dtype == np.float32 and np.array_equal(K_o[k], K_r[k])


def test_train_ids_and_camera_errors(tmp_path):
    from nrw import reprojection as R
    from nrw._lib import NrwError
    from nrw.colmap import Camera, Image
    from util_reproj import write_tsv

    with pytest.raises(NrwError, match="no \\*.tsv"):
        R.get_train_ids(str(tmp_path), [], {})
    write_tsv(str(tmp_path / "b.tsv"), [("x.jpg", 1, "train")])
    write_tsv(str(tmp_path / "a.tsv"), [("y.jpg", 2, "train"), ("z.jpg", "nan", "train"), ("w.jpg", 3, "test")])
    assert R.get_train_ids(str(tmp_path), [], {"y.jpg": 7, "w.jpg": 8}) == [7]          # a.tsv: first in sorted order
    with pytest.raises(NrwError, match="y.jpg"):
        R.get_train_ids(str(tmp_path), [], {"w.jpg": 8})
    cams = {1: Camera(1, "SIMPLE_RADIAL", 10, 10, np.ones(4))}
    ims = {5: Image(5, np.array([1.0, 0, 0, 0]), np.zeros(3), 1, "y.jpg")}
    with pytest.raises(NrwError, match="PINHOLE"):
        R.get_intrinsic(cams, [5], ims)


@needs_ref
def test_oracle_backprojection_matches_reference(ref):
    rng = np.random.default_rng(4)
    H, W = 37, 53
    depth = (rng.random((H, W)) * 5 + 0.5).astype(np.float32)
    depth[rng.random((H, W)) < 0.3] = 0
    K = np.array([[61.3, 0, 25.7], [0, 59.9, 18.2], [0, 0, 1]], dtype=np.float32)
    R, t = look_at(rng.normal(size=3) * 3, rng.normal(size=3))
    pose = np.linalg.inv(view_matrix(R, t) @ np.linalg.inv(np.diag([2.0, 2.0, 2.0, 1.0])))
    mine = rp.backproject(depth, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), pose)
    theirs = ref.reproj_filter.reproject(H, W, depth, K, pose, depth > 0)
    assert mine.shape == theirs.shape
    scale = np.abs(theirs).max()
    assert np.abs(mine - theirs).max() < 2e-6 * scale        # the reference inverts K in float32
    from nrw.reprojection import reproject

    assert np.array_equal(reproject(H, W, depth, K, pose, depth > 0), mine)


def _cam(fx=50.0, fy=50.0, cx=20.0, cy=15.0):
    return fx, fy, cx, cy


def test_oracle_plane_at_known_depth():
    # a big square at z = 3 facing the camera (two triangles, counter-clockwise as seen from the camera)
    v = np.array([[-10, -10, 3], [10, -10, 3], [10, 10, 3], [-10, 10, 3]], np.float64)
    f_front = np.array([[0, 2, 1], [0, 3, 2]])
    V = np.eye(4)[:3]
    for cull in (True, False):
        d, bad, cnt = rp.raster_depth(v, f_front, V, *_cam(), 30, 40, cull=cull, counts=True)
        assert not bad and np.all(d == np.float32(3.0)) and np.all(cnt == 1)
    d, _ = rp.raster_depth(v, f_front[:, ::-1], V, *_cam(), 30, 40, cull=True)
    assert np.all(d == 0)                                     # back faces culled
    d, _ = rp.raster_depth(v, f_front[:, ::-1], V, *_cam(), 30, 40, cull=False)
    assert np.all(d == np.float32(3.0))
    d, _ = rp.raster_depth(v, f_front, V, *_cam(), 30, 40, znear=3.5)
    assert np.all(d == 0)                                     # in front of znear
    d, _ = rp.raster_depth(v, f_front, V, *_cam(), 30, 40, zfar=2.5)
    assert np.all(d == 0)


def test_oracle_pixel_centre_convention():
    # a vertical edge x/z = (c + 0.5 - cx)/fx through the centres of column 10: that column belongs to exactly one
    # side (the tie rule), the columns left of it to the left face only
    fx, fy, cx, cy = 40.0, 40.0, 16.0, 12.0
    z = 2.0
    xe = (10 + 0.5 - cx) / fx * z
    v = np.array([[-5, -5, z], [xe, -5, z], [xe, 5, z], [-5, 5, z], [5, -5, z], [5, 5, z]], np.float64)
    f = np.array([[0, 2, 1], [0, 3, 2], [1, 2, 5], [1, 5, 4]])
    V = np.eye(4)[:3]
    d, _, cnt = rp.raster_depth(v, f, V, fx, fy, cx, cy, 24, 32, cull=True, counts=True)
    assert np.all(cnt == 1) and np.all(d == np.float32(z))
    d_left, _ = rp.raster_depth(v, f[:2], V, fx, fy, cx, cy, 24, 32, cull=True)
    assert np.all(d_left[:, :10] > 0) and np.all(d_left[:, 11:] == 0)
    # column 10's centre lies on the edge 1-2, which face [1, 2, 5] runs in ascending order: it owns the pixels
    assert np.all(d_left[:, 10] == 0)
    # a horizontal edge y/z = (r + 0.5 - cy)/fy: the same rule on rows
    ye = (7 + 0.5 - cy) / fy * z
    v2 = np.array([[-5, -5, z], [5, -5, z], [5, ye, z], [-5, ye, z]], np.float64)
    d2, _ = rp.raster_depth(v2, np.array([[0, 2, 1], [0, 3, 2]]), V, fx, fy, cx, cy, 24, 32, cull=True)
    assert np.all(d2[:7] > 0) and np.all(d2[8:] == 0)


def test_oracle_sphere_from_many_cameras():
    # closed marching-cubes sphere: every pixel whose analytic ray clearly hits gets a depth close to the analytic one,
    # clear misses stay empty, and no pixel is covered twice (front faces only)
    verts, faces, which = two_sphere_mesh(h=0.1)
    keep = which[faces].max(1) == 0
    f = faces[keep]
    rng = np.random.default_rng(5)
    H, W, fx = 40, 52, 45.0
    for _ in range(6):
        eye = rng.normal(size=3)
        eye *= rng.uniform(2.5, 5.0) / np.linalg.norm(eye)
        R, t = look_at(eye, rng.normal(size=3) * 0.2)
        V = view_matrix(R, t)[:3]
        cx, cy = W / 2 + rng.uniform(-2, 2), H / 2 + rng.uniform(-2, 2)
        d, bad, cnt = rp.raster_depth(verts, f, V, fx, fx, cx, cy, H, W, cull=True, counts=True)
        assert not bad and cnt.max() <= 1
        c, r = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
        dirs = np.stack([(c - cx) / fx, (r - cy) / fx, np.ones_like(c)], -1) @ R      # world ray directions (z = 1)
        o = eye
        a = (dirs ** 2).sum(-1)
        b = 2 * (dirs @ o)
        disc = b * b - 4 * a * (o @ o - 1.0)
        miss_margin, hit_margin = 0.3, 0.3
        sq = np.sqrt(np.maximum(disc, 0))
        t_hit = (-b - sq) / (2 * a)
        # ray clearly inside the silhouette of the (slightly smaller than r = 1) marching-cubes sphere
        dist_axis = np.sqrt(np.maximum(o @ o - (b / 2) ** 2 / a, 0))
        clear_hit = dist_axis < 1 - hit_margin
        clear_miss = dist_axis > 1 + miss_margin * 0.1
        assert np.all(d[clear_hit] > 0) and np.all(d[clear_miss] == 0)
        assert np.abs(d[clear_hit] - t_hit[clear_hit]).max() < 0.05


def test_oracle_box_is_conservative():
    # the pixel box never drops a pixel the whole-image test accepts: soups crossing the near plane and behind the
    # camera, both cull modes
    rng = np.random.default_rng(6)
    v, f = soup(rng, 300, spread=1.5, depth=(-1.0, 5.0))
    V = np.eye(4)[:3]
    for cull in (True, False):
        a, _ = rp.raster_depth(v, f, V, 30.0, 31.0, 16.3, 11.8, 23, 33, cull=cull, box=True)
        b, _ = rp.raster_depth(v, f, V, 30.0, 31.0, 16.3, 11.8, 23, 33, cull=cull, box=False)
        assert np.array_equal(a.view(np.int32), b.view(np.int32)) and (a > 0).sum() > 100


def test_raster_and_reproject_exports_reject_bad_arguments():
    import ctypes as C

    from nrw import _lib

    L = _lib.lib()
    err = L.nrw_last_error
    V = (C.c_double * 12)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0)
    bad = (C.c_double * 12)(1, 0, 0, float("nan"), 0, 1, 0, 0, 0, 0, 1, 0)
    fake = 1 << 20                                                   # never dereferenced: the checks come first
    assert L.nrw_raster_scratch_bytes(0, 1, 4, 4) < 0 and b"n_verts" in err()
    assert L.nrw_raster_scratch_bytes(3, -1, 4, 4) < 0 and b"n_faces" in err()
    assert L.nrw_raster_scratch_bytes(3, 1, 0, 4) < 0 and b"image" in err()
    assert L.nrw_raster_scratch_bytes(3, 1, 1 << 16, 1 << 16) < 0 and b"INT32_MAX" in err()
    assert L.nrw_raster_scratch_bytes(3, 1, 1, 1) > 0
    assert L.nrw_reproject_scratch_bytes(4, 0) < 0 and b"image" in err()
    assert L.nrw_reproject_scratch_bytes(1, 1) > 0

    def rd(nv=3, faces=fake, nf=1, view=V, fx=10.0, fy=10.0, cx=1.0, cy=1.0, H=4, W=4, zn=0.05, zf=100.0, cull=1,
           depth=fake, status=fake, scratch=fake):
        return L.nrw_raster_depth(fake, nv, faces, nf, view, fx, fy, cx, cy, H, W, zn, zf, cull, depth, status, scratch, None)

    assert rd(nv=0) != 0 and b"n_verts" in err()
    assert rd(nf=-1) != 0 and b"n_faces" in err()
    assert rd(H=0) != 0 and b"image" in err()
    assert rd(fx=0.0) != 0 and b"intrinsics" in err()
    assert rd(cy=float("inf")) != 0 and b"intrinsics" in err()
    assert rd(zn=0.0) != 0 and b"znear" in err()
    assert rd(zn=2.0, zf=1.0) != 0 and b"znear" in err()
    assert rd(zf=1e39) != 0 and b"zfar" in err()
    assert rd(cull=2) != 0 and b"cull_back" in err()
    assert rd(view=None) != 0 and b"null" in err()
    assert rd(view=bad) != 0 and b"finite" in err()
    assert rd(faces=None) != 0 and b"null" in err()
    assert rd(status=None) != 0 and b"null" in err()
    assert rd(scratch=fake + 8) != 0 and b"aligned" in err()

    def rm(depth=fake, H=4, W=4, fx=10.0, pose=V, index=fake, n=5, thr=0.1, visible=fake, scratch=fake):
        return L.nrw_reproject_mark(depth, H, W, fx, 10.0, 1.0, 1.0, pose, index, n, thr, visible, None, scratch, None)

    assert rm(H=-1) != 0 and b"image" in err()
    assert rm(fx=-1.0) != 0 and b"intrinsics" in err()
    assert rm(pose=bad) != 0 and b"finite" in err()
    assert rm(pose=None) != 0 and b"null" in err()
    assert rm(n=0) != 0 and b"n_ref" in err()
    assert rm(thr=float("nan")) != 0 and b"threshold" in err()
    assert rm(visible=None) != 0 and b"null" in err()
    assert rm(index=fake + 16) != 0 and b"aligned" in err()
