"""GPU: exact nearest neighbours and surface sampling (csrc/nnsearch.cu, nrw.evaluation) bit for bit against the
restatement oracle/eval_port.py and scipy, the crops, and eval_mesh end to end against the unmodified reference's own
eval_mesh (utils/eval_mesh.py, use_o3d=False), in mesh mode on a marching-cubes sphere, and through the CLI."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from oracle import eval_port as ep
from oracle import ref_import
from util_eval import sfm_points, surface_scene, write_points3d

pytestmark = pytest.mark.gpu


def _torch_nn(ref, q, chunk=1024):
    """brute force on the device with explicit elementwise fp64 ops (no fused kernels): (dist, smallest index)"""
    ref, q = ref.cuda().double(), q.cuda().double()
    ar = torch.arange(ref.shape[0], device="cuda")
    dist = torch.empty(q.shape[0], dtype=torch.float64, device="cuda")
    idx = torch.empty(q.shape[0], dtype=torch.int64, device="cuda")
    for a in range(0, q.shape[0], chunk):
        qq = q[a:a + chunk]
        dx = qq[:, None, 0] - ref[None, :, 0]
        dy = qq[:, None, 1] - ref[None, :, 1]
        dz = qq[:, None, 2] - ref[None, :, 2]
        d2 = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
        m = d2.min(1).values
        idx[a:a + chunk] = torch.where(d2 == m[:, None], ar, ref.shape[0]).min(1).values
        dist[a:a + chunk] = torch.sqrt(m)
    return dist, idx


def _nn(ref, q):
    from nrw.evaluation import NearestNeighbours

    return NearestNeighbours(ref).query(q)


def _sphere(g, n, r=1.0):
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    return d / d.norm(dim=1, keepdim=True) * r


def _cases():
    g = torch.Generator().manual_seed(0)
    yield "uniform", torch.rand(30000, 3, generator=g, dtype=torch.float64) * 10, torch.rand(100000, 3, generator=g, dtype=torch.float64) * 10
    yield "shell", _sphere(g, 40000) * 50, _sphere(g, 60000) * 50 + torch.randn(60000, 3, generator=g, dtype=torch.float64) * 0.1
    grid = torch.randint(-6, 7, (20000, 3), generator=g).double()           # duplicates and exact ties
    yield "grid_ties", grid, (torch.randint(-8, 9, (50000, 3), generator=g).double() + torch.randint(0, 2, (50000, 1), generator=g) * 0.5)
    ref = torch.rand(40000, 3, generator=g, dtype=torch.float64)
    q = torch.rand(50000, 3, generator=g, dtype=torch.float64)
    k = q.shape[0] // 100
    q[:k] = (torch.rand(k, 3, generator=g, dtype=torch.float64) - 0.5) * 2e3      # 1 % far outliers (10^3 x the extent)
    ref[:k // 2] = (torch.rand(k // 2, 3, generator=g, dtype=torch.float64) - 0.5) * 2e3
    yield "outliers", ref, q
    ref = torch.rand(20000, 3, generator=g, dtype=torch.float64) * 1e3 + 1e3
    yield "self", ref, ref[torch.randperm(20000, generator=g)]
    for n in (1, 31, 32, 33):
        yield f"tiny{n}", torch.rand(n, 3, generator=g, dtype=torch.float64), torch.rand(100000, 3, generator=g, dtype=torch.float64) * 3 - 1


CASES = list(_cases())


@pytest.mark.parametrize("name,ref,q", CASES, ids=[c[0] for c in CASES])
def test_nn_matches_oracle_bit_for_bit(name, ref, q):
    d, i = _nn(ref, q)
    rd, ri = _torch_nn(ref, q)
    assert torch.equal(d.view(torch.int64), rd.view(torch.int64))
    assert torch.equal(i, ri)
    if name == "self":
        assert (d == 0).all()
    if name == "tiny1":
        assert (i == 0).all()


def test_nn_matches_numpy_oracle_and_reference_arithmetic():
    rng = np.random.default_rng(4)
    ref, q = rng.normal(0, 1, (3000, 3)) * 1e3, rng.normal(0, 1, (2000, 3)) * 1e3
    d, i = _nn(ref, q)
    rd, ri = ep.nn_brute(ref, q)
    assert np.array_equal(d.cpu().numpy(), rd) and np.array_equal(i.cpu().numpy(), ri)


def test_nn_large_matches_ckdtree():
    from scipy.spatial import cKDTree

    rng = np.random.default_rng(11)
    n = 2_000_000
    ref = rng.normal(0, 1, (n, 3)) * [300.0, 200.0, 50.0] + 1e3
    q = rng.normal(0, 1, (n, 3)) * [300.0, 200.0, 50.0] + 1e3
    d, _ = _nn(ref, q)
    kd, _ = cKDTree(ref).query(q, workers=-1)
    assert np.array_equal(d.cpu().numpy(), kd)


def test_nn_invariant_under_query_permutation_and_repeatable():
    g = torch.Generator().manual_seed(3)
    ref = torch.randint(0, 20, (100000, 3), generator=g).double() * 0.25
    q = torch.rand(200000, 3, generator=g, dtype=torch.float64) * 5
    d, i = _nn(ref, q)
    d2, i2 = _nn(ref, q)
    assert torch.equal(d, d2) and torch.equal(i, i2)
    p = torch.randperm(q.shape[0], generator=g)
    dp, ip = _nn(ref, q[p])
    assert torch.equal(dp, d[p.cuda()]) and torch.equal(ip, i[p.cuda()])


def _mesh(seed, n_faces=5000, n_verts=1200, zero=True):
    rng = np.random.default_rng(seed)
    v = rng.normal(0, 1, (n_verts, 3)) * [3.0, 2.0, 1.0] + 100.0
    f = rng.integers(0, n_verts, (n_faces, 3))
    if zero:
        f[:5] = [7, 7, 9]                                   # zero area at the start
        f[2047:2060, 1] = f[2047:2060, 0]                   # degenerate across a tile border
        f[-3:] = [4, 4, 4]                                  # and at the end
    return v, f


@pytest.mark.parametrize("seed", [0, 1])
def test_sampling_matches_oracle(seed):
    from nrw.evaluation import sample_points_uniformly

    v, f = _mesh(seed)
    n = 200000
    p, fid = sample_points_uniformly(v, f, n, seed=seed, return_face_ids=True)
    p, fid = p.cpu().numpy(), fid.cpu().numpy()
    assert np.array_equal(p.view(np.int64), ep.barycentric(v, f, fid, seed).view(np.int64))
    rp, rfid = ep.sample_points(v, f, n, seed)
    assert np.array_equal(fid, rfid) and np.array_equal(p.view(np.int64), rp.view(np.int64))
    assert (ep.face_areas(v, f)[fid] > 0).all()


def test_sampling_distribution_and_seeds():
    from scipy.stats import chisquare

    from nrw.evaluation import sample_points_uniformly

    v, f = _mesh(2, n_faces=1500)
    areas = ep.face_areas(v, f)
    n = 3_000_000
    _, fid = sample_points_uniformly(v, f, n, seed=123, return_face_ids=True)
    cnt = np.bincount(fid.cpu().numpy(), minlength=len(f))
    pos = areas > 0
    assert (cnt[~pos] == 0).all()
    exp = areas[pos] / areas[pos].sum() * n
    assert chisquare(cnt[pos], exp).pvalue > 1e-3
    a = sample_points_uniformly(v, f, 1000, seed=5)
    b = sample_points_uniformly(v, f, 1000, seed=5)
    c = sample_points_uniformly(v, f, 1000, seed=6)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert torch.equal(sample_points_uniformly(v, f, 400, seed=5), a[:400])          # depends on (seed, s) only


def test_sampling_rejects_bad_meshes():
    from nrw._lib import NrwError
    from nrw.evaluation import sample_points_uniformly

    v, f = _mesh(3, zero=False)
    bad = f.copy()
    bad[100, 2] = len(v)
    with pytest.raises(NrwError, match="outside"):
        sample_points_uniformly(v, bad, 10)
    with pytest.raises(NrwError, match="area"):
        sample_points_uniformly(v, np.array([[1, 1, 2], [3, 3, 3]]), 10)
    with pytest.raises(NrwError, match="faces"):
        sample_points_uniformly(v, f[:, :2], 10)
    vv = v.copy()
    vv[0, 0] = np.nan
    with pytest.raises(NrwError, match="finite"):
        sample_points_uniformly(vv, f, 10)


BBX = [[-1.0, -0.5, -0.8], [1.2, 0.9, 0.6]]


def test_crops_match_oracle():
    from nrw.evaluation import _box_mask, bbx_crop, point_crop

    rng = np.random.default_rng(8)
    pts = rng.uniform(-1.5, 1.5, (200000, 3))
    assert np.array_equal(bbx_crop(pts, BBX), ep.bbx_crop(pts, BBX))
    assert torch.equal(bbx_crop(torch.from_numpy(pts).cuda(), BBX).cpu(), torch.from_numpy(ep.bbx_crop(pts, BBX)))
    assert np.array_equal(_box_mask(torch.from_numpy(pts).cuda(), BBX).cpu().numpy(), ep.box_mask(pts, BBX))
    sfm = rng.uniform(-1.3, 1.4, (5000, 3))
    for voxel in (0.02, 0.1, 0.35):
        src = rng.uniform(-1.3, 1.4, (50000, 3))
        got = point_crop(src, sfm, voxel, BBX)
        exp = ep.point_crop(src, sfm, voxel, BBX)
        assert 0 < len(exp) < len(src) and np.array_equal(got, exp)
        assert torch.equal(point_crop(torch.from_numpy(src).cuda(), sfm, voxel, BBX).cpu(), torch.from_numpy(exp))


# ---- end to end ---------------------------------------------------------------------------------------------------------
THRESHOLDS = [0.01 * k for k in range(1, 21)]                            # 20 thresholds


def _write_scene(d, seed=0, n_gt=1500, n_pred=2000, with_sfm=True):
    from nrw.mesh import write_ply

    rng = np.random.default_rng(seed)
    lo, hi = np.array(BBX[0]), np.array(BBX[1])
    gt, pred = surface_scene(rng, n_gt, n_pred, lo - 0.1, hi + 0.1, noise=0.02)
    os.makedirs(d, exist_ok=True)
    write_ply(os.path.join(d, "gt.ply"), gt)
    write_ply(os.path.join(d, "pred.ply"), pred)
    cfg = {"eval_bbx": BBX, "sfm2gt": np.eye(4).tolist()}
    if with_sfm:
        xyz, err, tl = sfm_points(rng, 4000, lo, hi)
        os.makedirs(os.path.join(d, "sfm"), exist_ok=True)
        write_points3d(os.path.join(d, "sfm", "points3D.bin"), xyz, err, tl)
        cfg.update(sfm_path=os.path.join(d, "sfm"), eval_tl=10, eval_error=2.0, eval_voxel=0.15)
    return gt, pred, cfg


class _Trimesh:
    """stand-in for the trimesh calls of eval_utils.trimesh_load: load() serves in-memory arrays, export() writes nothing"""

    def __init__(self, arrays):
        self.arrays = arrays

    def load(self, path):
        return types.SimpleNamespace(vertices=self.arrays[path])

    @staticmethod
    def PointCloud(v):
        return types.SimpleNamespace(export=lambda path: None)


@pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")
@pytest.mark.parametrize("with_sfm", [False, True])
def test_eval_mesh_matches_reference(tmp_path, monkeypatch, with_sfm):
    from nrw.evaluation import eval_mesh

    ref = ep.load_eval()
    eu = ref.eval_utils
    d = str(tmp_path)
    gt, pred, cfg = _write_scene(d, seed=1 + with_sfm, with_sfm=with_sfm)
    # the two reference branches agree here: identity sfm2gt, and no point on (or rounding onto) the box boundary
    for p in (gt, pred):
        assert np.array_equal(ep.bbx_crop(p, BBX), p[ep.box_mask(p, BBX)])
        lo, hi = np.array(BBX[0]), np.array(BBX[1])
        assert np.abs(p - lo).min() > 1e-9 and np.abs(p - hi).min() > 1e-9
    g, q = gt[ep.box_mask(gt, BBX)], pred[ep.box_mask(pred, BBX)]
    if with_sfm:
        sfm = ep.load_eval().eval_utils.filtered_sfm(cfg["sfm_path"], np.eye(4), cfg["eval_tl"], cfg["eval_error"])
        g, q = ep.point_crop(g, sfm, cfg["eval_voxel"], BBX), ep.point_crop(q, sfm, cfg["eval_voxel"], BBX)
    d1, _ = ep.nn_brute(q, g)
    d2, _ = ep.nn_brute(g, q)
    for t in THRESHOLDS:
        gap = min(np.abs(d1 - t).min(), np.abs(d2 - t).min())
        assert gap > np.spacing(t), t                     # no distance within one ulp of a threshold

    monkeypatch.setattr(eu, "trimesh", _Trimesh({f"{d}/ref/pred.ply": pred, f"{d}/gt.ply": gt}))
    monkeypatch.setattr(eu.spc_ops, "points_to_morton", ep.morton16, raising=False)
    os.makedirs(f"{d}/ref")
    r = ref.eval_mesh.eval_mesh(f"{d}/ref/pred.ply", f"{d}/gt.ply", dict(cfg), False, threshold=list(THRESHOLDS), use_o3d=False,
                                save_name="x")
    o = eval_mesh(f"{d}/pred.ply", f"{d}/gt.ply", dict(cfg), False, threshold=list(THRESHOLDS), save_name="x")
    assert set(r) == set(o)
    for k in ("prec", "recal", "fscore"):
        assert float(r[k]) == o[k]
    for k in ("dist1", "dist2"):
        assert abs(o[k] / float(r[k]) - 1) < 1e-12
    jr = json.load(open(f"{d}/ref/eval_x/metrics.json"))
    jo = json.load(open(f"{d}/eval_x/metrics.json"))
    assert jr == jo and 0 < min(jo["precs"]) < 1 and 0 < min(jo["recals"]) < 1
    for t in THRESHOLDS:
        mr = json.load(open(f"{d}/ref/eval_x/visualize/{t:.2f}/metrics.json"))
        mo = json.load(open(f"{d}/eval_x/visualize/{t:.2f}/metrics.json"))
        assert set(mr) == set(mo)
        for k in mr:
            assert abs(mo[k] - mr[k]) <= 1e-12 * abs(mr[k])
    names = {"down_gt.ply", "down_pred_in_gt.ply"} | ({"sfm_points.ply", "pred_filtered.ply", "target_filtered.ply"} if with_sfm else set())
    assert names <= set(os.listdir(f"{d}/eval_x"))


def test_eval_mesh_on_marching_cubes_sphere(tmp_path):
    from nrw.evaluation import eval_mesh
    from nrw.mesh import marching_cubes, write_ply

    dim, R = 96, 0.8
    lin = torch.linspace(-1, 1, dim, device="cuda", dtype=torch.float64)
    x, y, z = torch.meshgrid(lin, lin, lin, indexing="ij")
    vol = (torch.sqrt(x * x + y * y + z * z) - R).float()
    v, f, _ = marching_cubes(vol)
    voxel = 2.0 / (dim - 1)
    verts = v.double().cpu().numpy() * voxel - 1.0
    write_ply(str(tmp_path / "mesh.ply"), verts, f.cpu().numpy())
    g = torch.Generator().manual_seed(0)
    gt = _sphere(g, 200000, R).numpy()
    write_ply(str(tmp_path / "gt.ply"), gt)
    cfg = {"eval_bbx": [[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]], "sfm2gt": np.eye(4).tolist()}
    ts = [voxel / 4, 2 * voxel, 3 * voxel]
    m = eval_mesh(str(tmp_path / "mesh.ply"), str(tmp_path / "gt.ply"), cfg, True, threshold=ts, save_name="m")
    j = json.load(open(tmp_path / "eval_m" / "metrics.json"))
    assert m["dist1"] < voxel and m["dist2"] < voxel
    assert j["fscores"][1] == 1.0 and j["fscores"][2] == 1.0
    down = __import__("nrw.mesh", fromlist=["read_ply"]).read_ply(str(tmp_path / "eval_m" / "down_pred_in_gt.ply"))
    assert len(down["vertices"]) == 10 * len(gt)


def test_cli_writes_reference_layout(tmp_path):
    import yaml

    d = str(tmp_path)
    _, _, cfg = _write_scene(d, seed=7)
    sfm = cfg.pop("sfm_path")
    for k in ("eval_tl", "eval_error", "eval_voxel"):
        cfg.pop(k)
    with open(f"{d}/config.yaml", "w") as fh:
        yaml.safe_dump(cfg, fh)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    cmd = [sys.executable, "-s", "-m", "nrw.evaluation", "--file_pred", f"{d}/pred.ply", "--file_trgt", f"{d}/gt.ply",
           "--scene_config_path", f"{d}/config.yaml", "--threshold", "0.01,0.2,0.01", "--save_name", "cli",
           "--sfm_path", sfm, "--track_lenth", "10", "--reproj_error", "2", "--voxel_size", "0.15"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = f"{d}/eval_cli"
    j = json.load(open(f"{out}/metrics.json"))
    assert set(j) == {"thresholds", "fscores", "precs", "recals"}
    assert j["thresholds"] == [float(t) for t in np.arange(0.01, 0.2, 0.01)]
    assert {"down_gt.ply", "down_pred_in_gt.ply", "sfm_points.ply", "pred_filtered.ply", "target_filtered.ply", "visualize"} <= set(os.listdir(out))
    for t in j["thresholds"]:
        m = json.load(open(f"{out}/visualize/{t:.2f}/metrics.json"))
        assert set(m) == {"dist1", "dist2", "prec", "recal", "fscore"}


def test_eval_mesh_raises_on_empty_and_non_finite(tmp_path):
    from nrw._lib import NrwError
    from nrw.evaluation import eval_mesh, nn_correspondance
    from nrw.mesh import write_ply

    d = str(tmp_path)
    write_ply(f"{d}/gt.ply", np.random.default_rng(0).random((100, 3)) + 5.0)        # all outside the box
    write_ply(f"{d}/pred.ply", np.random.default_rng(1).random((100, 3)))
    cfg = {"eval_bbx": BBX, "sfm2gt": np.eye(4).tolist()}
    with pytest.raises(NrwError, match="ground-truth"):
        eval_mesh(f"{d}/pred.ply", f"{d}/gt.ply", cfg, False)
    bad = np.random.default_rng(2).random((10, 3))
    bad[3, 1] = np.inf
    with pytest.raises(NrwError, match="finite"):
        nn_correspondance(bad, bad)
    assert nn_correspondance(bad[:0], bad) == ([], [])
