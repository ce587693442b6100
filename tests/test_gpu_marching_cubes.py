"""GPU: masked marching cubes (csrc/mcubes.cu, nrw.mesh.marching_cubes) against the numpy restatement oracle/mc_port.py
bit for bit, mesh topology at sizes the oracle cannot reach, and the drop-in extract_mesh (dense, sparse, two ranks,
the reference's own NeuconWSystem call sites)."""
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

from conftest import ROOT
from oracle import mc_port, ref_import
from util_nrw import build_system, synth

pytestmark = pytest.mark.gpu


def _mc(vol, level=0.0, mask=None):
    from nrw.mesh import marching_cubes

    return marching_cubes(vol, level, mask)


def _smooth(shape, seed, sigma=2.0):
    x = gaussian_filter(np.random.default_rng(seed).standard_normal(shape), sigma)
    return (x / x.std()).astype(np.float32)


def _sparse_mask(shape, seed):
    """the mask sparse_sdf_volume returns (8-corner erosion of the evaluated points), for a random point set"""
    from nrw.mesh import _scatter_volume

    g = torch.Generator().manual_seed(seed)
    n = int(np.prod(shape))
    keep = torch.nonzero(torch.rand(n, generator=g) < 0.9).reshape(-1)
    ind = torch.stack(torch.unravel_index(keep, shape), -1).cuda()
    _, m = _scatter_volume(ind, torch.zeros(len(keep), device="cuda"), max(shape))       # a cube; cropped below
    m = m[:shape[0], :shape[1], :shape[2]]
    return m.contiguous()


def _compare(vol_np, level, mask):
    v, f, n = _mc(torch.from_numpy(vol_np).cuda(), level, mask)
    rv, rf, rn = mc_port.marching_cubes(vol_np, level, None if mask is None else mask.cpu().numpy())
    assert v.shape == rv.shape and f.shape == rf.shape
    assert np.array_equal(f.cpu().numpy(), rf)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), rv.view(np.uint32))
    if len(rn):
        assert float(np.abs(n.cpu().numpy() - rn).max()) <= 1e-6
    assert torch.isfinite(v).all() and torch.isfinite(n).all()
    return v, f, n


@pytest.mark.parametrize("shape", [(2, 2, 2), (3, 5, 7), (33, 64, 65), (97, 97, 97)])
@pytest.mark.parametrize("level", [0.0, 0.3])
@pytest.mark.parametrize("mask_kind", ["none", "random", "sparse"])
def test_matches_oracle(shape, level, mask_kind):
    vol = _smooth(shape, seed=sum(shape), sigma=1.0 if min(shape) < 8 else 3.0)
    mask = None
    if mask_kind == "random":
        mask = torch.from_numpy(np.random.default_rng(7).random(shape) < 0.7).cuda()
    elif mask_kind == "sparse":
        mask = _sparse_mask(shape, 3)
    v, f, _ = _compare(vol, level, mask)
    if min(shape) > 8 and mask is None:
        assert f.shape[0] > 100


def test_ties_and_non_finite_values():
    rng = np.random.default_rng(5)
    ints = rng.integers(-2, 3, (21, 18, 23)).astype(np.float32)            # many values exactly at the level
    for level in (0.0, 1.0):
        _compare(ints, level, None)
    bad = _smooth((30, 31, 29), 9)
    idx = rng.integers(0, bad.size, 200)
    bad.reshape(-1)[idx[:70]] = np.nan
    bad.reshape(-1)[idx[70:140]] = np.inf
    bad.reshape(-1)[idx[140:]] = -np.inf
    _compare(bad, 0.0, None)
    _compare(bad, 0.0, torch.from_numpy(rng.random(bad.shape) < 0.8).cuda())
    for const in (1.0, -1.0):                                              # no crossing / everything below
        v, f, n = _mc(torch.full((17, 9, 12), const, device="cuda"))
        assert v.shape == (0, 3) and f.shape == (0, 3) and n.shape == (0, 3)


def _sphere_t(n, R, c):
    a = torch.arange(n, device="cuda", dtype=torch.float32)
    d2 = (a - c[0])[:, None, None] ** 2 + (a - c[1])[None, :, None] ** 2 + (a - c[2])[None, None, :] ** 2
    return d2.sqrt_().sub_(R)


def _topology(f, nv):
    """(closed and consistently oriented, Euler characteristic) on the device"""
    f = f.to(torch.int64)
    a = torch.cat([f[:, 0], f[:, 1], f[:, 2]])
    b = torch.cat([f[:, 1], f[:, 2], f[:, 0]])
    fwd = torch.sort(a * nv + b).values
    uniq = bool((fwd[1:] != fwd[:-1]).all())
    rev = b * nv + a
    pos = torch.searchsorted(fwd, rev).clamp_(max=fwd.numel() - 1)
    closed = bool((fwd[pos] == rev).all())
    n_edges = fwd.numel() // 2
    return uniq and closed, nv - n_edges + f.shape[0]


def test_large_sphere_closed_and_accurate():
    c = (127.3, 128.1, 126.6)
    vol = _sphere_t(256, 100.0, c)
    v, f, n = _mc(vol)
    ok, chi = _topology(f, v.shape[0])
    assert ok and chi == 2
    cc = torch.tensor(c, device="cuda")
    radial = (v - cc) / (v - cc).norm(dim=1, keepdim=True)
    assert float((n * radial).sum(1).min()) >= 0.999
    p0, p1, p2 = (v[f[:, i].long()].double() for i in range(3))
    enclosed = float((p0 * torch.cross(p1, p2, dim=1)).sum()) / 6
    assert abs(enclosed / (4 / 3 * np.pi * 100.0 ** 3) - 1) < 0.005
    v2, f2, n2 = _mc(vol)                                                  # determinism
    assert torch.equal(v, v2) and torch.equal(f, f2) and torch.equal(n, n2)


def test_sphere_896_needs_64_bit_edge_ids():
    vol = _sphere_t(896, 400.0, (447.6, 447.2, 448.3))
    v, f, _ = _mc(vol)
    below = vol < 0
    del vol
    crossings = sum(int((below.narrow(ax, 0, 895) != below.narrow(ax, 1, 895)).sum()) for ax in range(3))
    del below
    assert v.shape[0] == crossings
    ok, chi = _topology(f, v.shape[0])
    assert ok and chi == 2


def _surface_params():
    """synthetic parameters whose SDF (positive everywhere in [-1,1]^3) is shifted down so that its zero level set is a
    closed surface inside the box"""
    P = synth.make_params(seed=0)
    P["neuconw.sdf_net.lin8.bias"][0] -= 0.3
    return P


@pytest.fixture(scope="module")
def renderer():
    return build_system(_surface_params(), synth.PathConfig(), precision="bf16x3", backend=0)["renderer"]


def test_extract_mesh_dense_matches_oracle_and_colours(renderer, tmp_path):
    from nrw.mesh import extract_mesh, read_ply, sdf_volume

    so, sr = [0.1, -0.2, 0.3], 2.0
    emb = torch.randn(1, synth.PathConfig().n_a, generator=torch.Generator().manual_seed(1)).cuda()
    mesh = extract_mesh(96, 65536, sr, so, origin=[0.05, 0.0, -0.02], radius=0.9, with_color=True, embedding_a=emb,
                        renderer=renderer)
    vol, vol_origin, voxel = sdf_volume(renderer, 96, origin=[0.05, 0.0, -0.02], radius=0.9)
    rv, rf, rn = mc_port.marching_cubes(vol.cpu().numpy(), 0.0)
    vt = rv * voxel + vol_origin
    assert len(rf) > 1000
    assert np.array_equal(mesh.faces, rf) and np.array_equal(mesh.vertices, vt * sr + np.array(so))
    assert float(np.abs(mesh.vertex_normals - rn).max()) <= 1e-6
    pts = torch.from_numpy(vt).float().cuda().reshape(-1, 1, 3)
    d = torch.zeros_like(pts)
    d[..., 2] = 1
    with torch.no_grad():
        rgb = renderer.rgb(pts, d, emb.repeat(pts.shape[0], 1).reshape(-1, 1, emb.shape[1])).cpu().numpy()
    want = np.clip(np.round(rgb * 255), 0, 255)
    diff = np.abs(mesh.vertex_colors.astype(np.int64) - want)
    near_half = np.abs(rgb * 255 - np.floor(rgb * 255) - 0.5) < 255e-6             # rgb within 1e-6 of a rounding tie
    assert (diff[~near_half] == 0).all() and diff.max() <= 1
    p = str(tmp_path / "dense.ply")
    mesh.export(p)
    r = read_ply(p)
    assert np.array_equal(r["faces"], mesh.faces) and np.array_equal(r["colors"], mesh.vertex_colors)
    assert np.array_equal(r["vertices"], mesh.vertices.astype(np.float32))


def test_extract_mesh_sparse_both_formats(renderer):
    from nrw.mesh import extract_mesh, gen_grid_spc, marching_cubes, sparse_sdf_volume
    from nrw.synthetic import sphere_shell_points

    renderer.scene_config = {"sfm2gt": np.eye(4).tolist(), "eval_bbx": [[-1.0] * 3, [1.0] * 3]}
    renderer.sfm_points, renderer.voxel_size = sphere_shell_points(0.5, 0.03, 4000, seed=1).numpy(), 0.12
    renderer.octree_data = renderer.get_octree(0)
    grid = gen_grid_spc(renderer, int(renderer.octree_data["level"]) + 2)
    up = grid["up_times"]
    leaves = grid["leaves"].cpu().to(torch.int64)
    k = torch.arange(up)
    kern = torch.stack(torch.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    ind_up = (leaves[:, None, :] * up + kern[None]).reshape(-1, 3)
    ref_fmt = {"sparse_vol": ind_up * grid["voxel_size"] + grid["vol_origin"], "voxel_size": grid["voxel_size"],
               "dim": grid["dim"], "vol_origin": grid["vol_origin"].numpy()}          # tools/extract_mesh.py:89-101
    so, sr = renderer.origin.float().numpy().tolist(), float(renderer.radius)
    m1 = extract_mesh(0, 1 << 18, sr, so, sparse_data=grid, renderer=renderer)
    m2 = extract_mesh(0, 1 << 18, sr, so, sparse_data=ref_fmt, renderer=renderer)
    assert len(m1.faces) > 1000
    assert np.array_equal(m1.faces, m2.faces) and np.array_equal(m1.vertices, m2.vertices)
    assert np.array_equal(m1.vertex_normals, m2.vertex_normals)
    # no vertex on an edge with an unevaluated end (the sparse volume is 1 there)
    vol, mask = sparse_sdf_volume(renderer, grid)
    ev = torch.zeros_like(mask)
    ev[ind_up[:, 0], ind_up[:, 1], ind_up[:, 2]] = True
    v, f, _ = marching_cubes(vol, 0.0, mask)
    lo = v.floor().long()
    ax = (v != v.floor()).int().argmax(1)
    hi = lo.clone()
    hi[torch.arange(len(v)), ax] += 1
    assert bool(ev[lo[:, 0], lo[:, 1], lo[:, 2]].all()) and bool(ev[hi[:, 0], hi[:, 1], hi[:, 2]].all())


_WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.path.join({root!r}, "neuralrecon-w_b200")); sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
from util_nrw import build_system, synth
from test_gpu_marching_cubes import _surface_params
from nrw.mesh import extract_mesh
rank = int(os.environ["RANK"])
dist.init_process_group("gloo", rank=rank, world_size=2)
r = build_system(_surface_params(), synth.PathConfig(), precision="bf16x3", backend=0)["renderer"]
emb = torch.full((1, synth.PathConfig().n_a), 0.1, device="cuda")
m = extract_mesh(40, 7777, 1.5, [0.0, 0.1, 0.0], with_color=True, embedding_a=emb, chunk_rgb=333, renderer=r)
if rank == 0:
    np.savez({out!r}, v=m.vertices, f=m.faces, n=m.vertex_normals, c=m.vertex_colors)
else:
    assert m is None
dist.barrier()
dist.destroy_process_group()
"""


def test_extract_mesh_two_ranks(renderer, tmp_path):
    from nrw.mesh import extract_mesh

    out = str(tmp_path / "mesh.npz")
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(root=ROOT, out=out))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29533", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    logs = [p.communicate(timeout=600)[0].decode() for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(logs)[-3000:]
    got = np.load(out)
    assert len(got["f"]) > 100
    emb = torch.full((1, synth.PathConfig().n_a), 0.1, device="cuda")
    m = extract_mesh(40, 7777, 1.5, [0.0, 0.1, 0.0], with_color=True, embedding_a=emb, chunk_rgb=333, renderer=renderer)
    assert np.array_equal(got["v"], m.vertices) and np.array_equal(got["f"], m.faces)
    assert np.array_equal(got["n"], m.vertex_normals) and np.array_equal(got["c"], m.vertex_colors)


@pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")
def test_reference_system_call_sites(tmp_path):
    """neuconw_system.py:468-475 (validation_step) and tools/extract_mesh.py:154-158 call forms on the reference's own
    NeuconWSystem with the documented patch, extract_mesh included."""
    import argparse

    import nrw
    import nrw.generate_voxel as ngv
    import nrw.mesh
    import yaml
    from nrw.mesh import read_ply

    m = ref_import.load_system()
    ns = m.ns
    ns.NeuconW, ns.NeRF, ns.NeuconWRenderer = nrw.NeuconW, nrw.NeRF, nrw.NeuconWRenderer
    ns.convert_to_dense, ns.gen_octree, ns.octree_to_spc = ngv.convert_to_dense, ngv.gen_octree, ngv.octree_to_spc
    ns.extract_mesh = nrw.mesh.extract_mesh
    scene = dict(origin=[0.0, 0.0, 0.0], radius=1.0, sfm2gt=np.eye(4).tolist(), eval_bbx=[[-1.0] * 3, [1.0] * 3],
                 eval_bbx_detail=[[-0.6] * 3, [0.6] * 3], voxel_size=0.1, min_track_length=0)
    with open(tmp_path / "config.yaml", "w") as fh:
        yaml.safe_dump(scene, fh)
    config = m.get_cfg_defaults()
    config.merge_from_file(os.path.join(m.config_dir, "train_brandenburg_gate.yaml"))
    config.DATASET.ROOT_DIR = str(tmp_path)
    config.NEUCONW.N_VOCAB = 64
    hparams = argparse.Namespace(num_gpus=1, test_batch_size=128, exp_name="mesh", num_epochs=1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sysm = m.NeuconWSystem(hparams, config, None)
    sysm.to("cuda")
    mesh = ns.extract_mesh(dim=128, chunk=16384, scene_radius=sysm.scene_config["radius"],
                           scene_origin=sysm.scene_config["origin"], with_color=False, renderer=sysm.renderer)
    p1 = str(tmp_path / "00000000.ply")
    mesh.export(p1)
    r1 = read_ply(p1)
    assert len(r1["faces"]) > 1000 and r1["colors"] is None and np.array_equal(r1["faces"], mesh.faces)
    emb = sysm.embedding_a((torch.ones(1, device="cuda") * 11).long())
    mesh2 = ns.extract_mesh(64, 16384, scene["radius"], scene["origin"], origin=[0.0, 0.0, 0.0], radius=1.0, with_color=True,
                            embedding_a=emb, chunk_rgb=1024, sparse_data=None, renderer=sysm.renderer)
    p2 = str(tmp_path / "extracted_mesh_res_64_radius_1.0_colored.ply")
    mesh2.export(p2)
    r2 = read_ply(p2)
    assert len(r2["faces"]) > 100 and r2["colors"].shape == (len(mesh2.vertices), 3)
    assert np.array_equal(r2["colors"], mesh2.vertex_colors)
