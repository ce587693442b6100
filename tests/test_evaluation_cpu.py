"""CPU checks of the evaluation: the numpy restatement oracle/eval_port.py against the unmodified reference
(utils/eval_utils.py), the PLY and COLMAP readers, and the argument checks of the nrw_nn_* / nrw_mesh_sample exports."""
import os

import numpy as np
import pytest

from oracle import eval_port as ep
from oracle import ref_import
from util_eval import sfm_points, write_points3d

BBX = [[-1.0, -0.5, -0.8], [1.2, 0.9, 0.6]]
needs_ref = pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")


@pytest.fixture(scope="module")
def ref():
    return ep.load_eval()


@needs_ref
@pytest.mark.parametrize("grid", [False, True])
def test_oracle_nn_matches_reference(ref, grid):
    rng = np.random.default_rng(1 + grid)
    if grid:                                           # many exact ties and duplicate points
        a = rng.integers(-4, 5, (400, 3)).astype(np.float64)
        b = rng.integers(-5, 6, (300, 3)).astype(np.float64) + rng.integers(0, 2, (300, 1)) * 0.5
    else:
        a = rng.normal(0, 1, (500, 3)) * 1e3
        b = rng.normal(0, 1, (300, 3)) * 1e3
    ri, rd = ref.eval_utils.nn_correspondance(a, b, use_o3d=False)
    d, i = ep.nn_brute(a, b)
    assert np.array_equal(d, np.asarray(rd))
    if not grid:
        assert np.array_equal(i, np.asarray(ri))          # scipy's tie order is its own; the distances are the contract
    assert np.array_equal(ref.eval_utils.nn_correspondance(a[:0], b, use_o3d=False)[1], [])


@needs_ref
def test_oracle_crops_and_metrics_match_reference(ref, tmp_path, monkeypatch):
    eu = ref.eval_utils
    rng = np.random.default_rng(5)
    pts = rng.uniform(-1.5, 1.5, (4000, 3))
    assert np.array_equal(ep.bbx_crop(pts, BBX), eu.bbx_crop(pts, BBX))
    d1, d2 = rng.random(1000) * 0.3, rng.random(700) * 0.3
    for t in (0.01, 0.05, 0.1, 0.3, 0.5):
        r, o = eu._compute(d1, d2, t), ep.compute(d1, d2, t)
        assert r == o
    # SfM filter and crop, SfM points inside and outside the box
    xyz, err, tl = sfm_points(rng, 3000, *BBX)
    write_points3d(str(tmp_path / "points3D.bin"), xyz, err, tl)
    T = np.eye(4)
    T[:3, :3] = [[0.9, -0.1, 0.05], [0.1, 0.95, 0.0], [-0.03, 0.02, 1.1]]
    T[:3, 3] = [0.1, -0.2, 0.3]
    from nrw.evaluation import filtered_sfm

    r = eu.filtered_sfm(str(tmp_path), T, track_length=12, reproj_error=1.5)
    keep = (tl > 12) & (err < 1.5)
    xyz1 = np.concatenate([xyz[keep], np.ones((keep.sum(), 1))], 1)
    assert np.array_equal(r, (T[:3] @ xyz1.T).T)
    assert np.array_equal(filtered_sfm(str(tmp_path), T, track_length=12, reproj_error=1.5), r)
    monkeypatch.setattr(eu.spc_ops, "points_to_morton", ep.morton16, raising=False)
    for voxel in (0.1, 0.3):
        src = rng.uniform(-1.3, 1.4, (3000, 3))
        got = eu.point_crop(src, r, voxel, BBX, batch_size=8, device="cpu")
        exp = ep.point_crop(src, r, voxel, BBX)
        assert 0 < len(exp) < len(src) and np.array_equal(got, exp)


def test_oracle_sampling_rules():
    rng = np.random.default_rng(0)
    v = rng.random((40, 3))
    f = rng.integers(0, 40, (2500, 3))
    f[:7] = [3, 3, 5]                                   # zero-area faces at the start of the first tile
    f[1500:1510] = [2, 2, 2]
    a = ep.face_areas(v, f)
    p, fid = ep.sample_points(v, f, 20000, seed=7)
    assert (a[fid] > 0).all()
    pref = ep.area_prefix(a)
    assert np.array_equal(pref[:1024], np.cumsum(a[:1024])) and abs(pref[-1] / a.sum() - 1) < 1e-12
    p2, fid2 = ep.sample_points(v, f, 20000, seed=7)
    assert np.array_equal(p, p2) and np.array_equal(fid, fid2)
    assert not np.array_equal(ep.sample_points(v, f, 100, seed=8)[1], fid[:100])
    # the samples lie in their triangles: barycentric weights a, b, c >= 0 summing to 1
    p0, p1, p2_ = v[f[fid, 0]], v[f[fid, 1]], v[f[fid, 2]]
    w = np.linalg.lstsq(np.stack([p1 - p0, p2_ - p0], -1)[0], (p - p0)[0], rcond=None)[0]
    assert (w > -1e-9).all() and w.sum() < 1 + 1e-9


def _ply_bytes(fmt, vprops, vrows, fcount_t, fidx_t, faces, extra_face_prop=False):
    np_t = {"float": "f4", "double": "f8", "uchar": "u1", "int": "i4", "short": "i2", "uint": "u4", "char": "i1", "ushort": "u2"}
    head = ["ply", f"format {fmt} 1.0", "comment test", f"element vertex {len(vrows)}"]
    head += [f"property {t} {n}" for n, t in vprops]
    if faces is not None:
        head += [f"element face {len(faces)}", f"property list {fcount_t} {fidx_t} vertex_indices"]
        if extra_face_prop:
            head += ["property uchar flags"]
    head += ["end_header"]
    out = ("\n".join(head) + "\n").encode()
    if fmt == "ascii":
        lines = [" ".join(str(x) for x in r) for r in vrows]
        if faces is not None:
            lines += [" ".join(str(x) for x in [len(fc)] + list(fc) + ([7] if extra_face_prop else [])) for fc in faces]
        return out + ("\n".join(lines) + "\n").encode()
    bo = "<" if fmt == "binary_little_endian" else ">"
    dt = np.dtype([(n, bo + np_t[t]) for n, t in vprops])
    v = np.array([tuple(r) for r in vrows], dtype=dt)
    out += v.tobytes()
    if faces is not None:
        for fc in faces:
            out += np.array([len(fc)], bo + np_t[fcount_t]).tobytes() + np.array(fc, bo + np_t[fidx_t]).tobytes()
            if extra_face_prop:
                out += b"\x07"
    return out


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("xyz_t", ["float", "double", "int"])
@pytest.mark.parametrize("count_t", ["uchar", "int"])
def test_read_ply_formats(tmp_path, fmt, xyz_t, count_t):
    from nrw.mesh import read_ply

    rng = np.random.default_rng(0)
    n = 12
    xyz = {"int": rng.integers(-50, 50, (n, 3)), "float": (rng.random((n, 3)) * 10).astype(np.float32),
           "double": rng.random((n, 3)) * 10}[xyz_t]
    col = rng.integers(0, 256, (n, 3))
    vprops = [("x", xyz_t), ("y", xyz_t), ("z", xyz_t), ("red", "uchar"), ("green", "uchar"), ("blue", "uchar"), ("quality", "short")]
    rows = [list(xyz[i]) + list(col[i]) + [int(i) - 5] for i in range(n)]
    faces = rng.integers(0, n, (9, 3))
    p = tmp_path / "a.ply"
    p.write_bytes(_ply_bytes(fmt, vprops, rows, count_t, "int" if count_t == "uchar" else "uint", faces.tolist(), extra_face_prop=True))
    r = read_ply(str(p))
    assert np.array_equal(r["vertices"], xyz) and np.array_equal(r["colors"], col) and r["normals"] is None
    assert r["faces"].dtype == np.int64 and np.array_equal(r["faces"], faces)
    p.write_bytes(_ply_bytes(fmt, vprops[:3], [rw[:3] for rw in rows], count_t, "int", None))     # a point cloud
    r = read_ply(str(p))
    assert np.array_equal(r["vertices"], xyz) and r["faces"].shape == (0, 3) and r["colors"] is None


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
def test_read_ply_rejects_polygons(tmp_path, fmt):
    from nrw._lib import NrwError
    from nrw.mesh import read_ply

    p = tmp_path / "q.ply"
    rows = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, 1.0, 0.0], [0.0, 1.0, 0.0]]
    p.write_bytes(_ply_bytes(fmt, [("x", "float"), ("y", "float"), ("z", "float")], rows, "uchar", "int", [[0, 1, 2], [0, 1, 2, 3]]))
    with pytest.raises(NrwError, match="triangle"):
        read_ply(str(p))


def test_write_ply_point_cloud_round_trip(tmp_path):
    from nrw.mesh import read_ply, write_ply

    rng = np.random.default_rng(3)
    v = rng.random((30, 3)).astype(np.float32)
    write_ply(str(tmp_path / "p.ply"), v)
    r = read_ply(str(tmp_path / "p.ply"))
    assert np.array_equal(r["vertices"], v) and r["normals"] is None and r["faces"].shape == (0, 3)
    c = rng.integers(0, 256, (30, 3)).astype(np.uint8)
    write_ply(str(tmp_path / "c.ply"), v, colors=c)
    r = read_ply(str(tmp_path / "c.ply"))
    assert np.array_equal(r["vertices"], v) and np.array_equal(r["colors"], c)


@needs_ref
def test_colmap_reader_matches_reference(tmp_path):
    from nrw.colmap import read_points3d

    ref_import._install_stubs()
    import sys

    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    from utils.colmap_utils import read_points3d_binary  # type: ignore

    rng = np.random.default_rng(9)
    xyz, err, tl = sfm_points(rng, 200, *BBX)
    path = str(tmp_path / "points3D.bin")
    write_points3d(path, xyz, err, tl)
    ours = read_points3d(path)
    theirs = read_points3d_binary(path)
    assert len(theirs) == len(ours["xyz"])
    for k, (pid, p) in enumerate(theirs.items()):
        assert ours["id"][k] == pid and np.array_equal(ours["xyz"][k], p.xyz) and ours["error"][k] == p.error
        assert ours["track_length"][k] == len(p.point2D_idxs) and np.array_equal(ours["rgb"][k], p.rgb)
    open(path, "ab").close()
    with open(path, "r+b") as fh:
        fh.truncate(os.path.getsize(path) - 5)
    from nrw._lib import NrwError

    with pytest.raises(NrwError, match="truncated"):
        read_points3d(path)


def test_nn_and_sample_exports_reject_bad_arguments():
    from nrw import _lib

    L = _lib.lib()
    err = L.nrw_last_error
    assert L.nrw_nn_index_bytes(0) < 0 and b"n_ref" in err()
    assert L.nrw_nn_index_bytes(1 << 31) < 0 and b"INT32_MAX" in err()
    assert 0 < L.nrw_nn_index_bytes(5_000_000) < 200 * 5_000_000
    assert L.nrw_nn_query_scratch_bytes(-1) < 0 and b"n_query" in err()
    assert L.nrw_nn_query_scratch_bytes(0) >= 0
    assert L.nrw_mesh_sample_scratch_bytes(0) < 0 and b"n_faces" in err()
    fake = 1 << 20                                                   # never dereferenced: the checks come first
    assert L.nrw_nn_build(None, 10, fake, None) != 0 and b"null" in err()
    assert L.nrw_nn_build(fake, 0, fake, None) != 0 and b"n_ref" in err()
    assert L.nrw_nn_build(fake, 10, fake + 16, None) != 0 and b"aligned" in err()
    assert L.nrw_nn_query(fake, 0, fake, 5, fake, fake, fake, None) != 0 and b"n_ref" in err()
    assert L.nrw_nn_query(fake, 10, fake, -1, fake, fake, fake, None) != 0 and b"n_query" in err()
    assert L.nrw_nn_query(fake, 10, fake, 1 << 31, fake, fake, fake, None) != 0 and b"n_query" in err()
    assert L.nrw_nn_query(None, 10, fake, 5, fake, fake, fake, None) != 0 and b"null" in err()
    assert L.nrw_nn_query(fake, 10, fake, 5, fake, fake, fake + 8, None) != 0 and b"aligned" in err()
    assert L.nrw_nn_query(fake, 10, None, 5, fake, fake, fake, None) != 0 and b"null" in err()
    assert L.nrw_nn_query(fake, 10, fake, 5, fake, None, fake, None) != 0 and b"null" in err()
    assert L.nrw_nn_query(fake, 10, None, 0, None, None, fake, None) == 0            # nothing to do
    assert L.nrw_mesh_sample(fake, 0, fake, 4, 10, 0, fake, None, fake, fake, None) != 0 and b"vertices" in err()
    assert L.nrw_mesh_sample(fake, 3, fake, 0, 10, 0, fake, None, fake, fake, None) != 0 and b"faces" in err()
    assert L.nrw_mesh_sample(fake, 3, fake, 1, -1, 0, fake, None, fake, fake, None) != 0 and b"samples" in err()
    assert L.nrw_mesh_sample(fake, 3, fake, 1, 10, 0, fake, None, None, fake, None) != 0 and b"status" in err()
    assert L.nrw_mesh_sample(fake, 3, fake, 1, 10, 0, None, None, fake, fake, None) != 0 and b"output" in err()
    assert L.nrw_mesh_sample(fake, 3, fake, 1, 10, 0, fake, None, fake, fake + 64, None) != 0 and b"aligned" in err()
