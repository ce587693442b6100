"""CPU checks of the marching-cubes case tables (csrc/gen_mc_tables.py), the numpy restatement oracle/mc_port.py, the
PLY writer and the argument checks of the three nrw_mc_* exports (no device needed)."""
import numpy as np
import pytest
from scipy.ndimage import gaussian_filter

from oracle import mc_port as mc

gen = mc.gen


def sphere(n, R, c):
    g = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).astype(np.float64)
    return (np.linalg.norm(g - np.array(c), axis=-1) - R).astype(np.float32)


def edge_counts(f):
    """(undirected edge -> face count, directed edges are unique)"""
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
    directed_unique = len(np.unique(e, axis=0)) == len(e)
    u, cnt = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    return u, cnt, directed_unique


def euler(v, f):
    u, _, _ = edge_counts(f)
    return len(v) - len(u) + len(f)


def enclosed_volume(v, f):
    a, b, c = (v[f[:, i]].astype(np.float64) for i in range(3))
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6)


def test_committed_table_header_is_generated():
    with open(gen.HEADER_PATH) as fh:
        assert fh.read() == gen.header()


@pytest.mark.parametrize("case", range(256))
def test_case_table(case):
    tris = gen.case_triangles(case)
    used = sorted({e for t in tris for e in t})
    assert used == gen.crossing_edges(case)                          # every crossing edge and no other
    assert all(len(set(t)) == 3 for t in tris)                       # no degenerate triangle
    count, mask, table = mc.TRI_COUNT, mc.EDGE_MASK, mc.TRI_TABLE
    assert count[case] == len(tris) and mask[case] == sum(1 << e for e in used)
    assert [tuple(int(x) for x in r) for r in table[case, :len(tris)]] == tris
    # directed boundary of the triangles == the face rule's directed segments, face by face
    directed = {}
    for t in tris:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            if (b, a) in directed:
                del directed[(b, a)]
            else:
                directed[(a, b)] = True
    segs = gen.face_segments(case)
    assert set(directed) == {(p, q) for p, q, _ in segs}
    for fi, (_, _, fedges) in enumerate(gen.FACES):
        on_face = {(p, q) for (p, q) in directed if p in fedges and q in fedges}
        assert on_face == {(p, q) for p, q, f in segs if f == fi}


def _fields():
    yield "sphere", sphere(48, 20.0, (23.3, 24.1, 22.7)), 2
    # torus: major radius 12, minor 5
    g = np.stack(np.meshgrid(*[np.arange(48)] * 3, indexing="ij"), -1).astype(np.float64) - np.array([23.6, 23.2, 24.1])
    q = np.stack([np.hypot(g[..., 0], g[..., 1]) - 12.0, g[..., 2]], -1)
    yield "torus", (np.linalg.norm(q, axis=-1) - 5.0).astype(np.float32), 0
    two = np.minimum(sphere(48, 9.0, (12.2, 13.1, 12.7)), sphere(48, 8.0, (33.4, 32.9, 34.2)))
    yield "two_spheres", two, 4
    for seed in range(12):
        x = gaussian_filter(np.random.default_rng(seed).standard_normal((36, 36, 36)), 3)
        x = (x / x.std()).astype(np.float32)
        x[[0, -1]] = 1
        x[:, [0, -1]] = 1
        x[:, :, [0, -1]] = 1
        yield f"random{seed}", x, None


@pytest.mark.parametrize("name,vol,chi", list(_fields()), ids=[f[0] for f in _fields()])
def test_oracle_closed_oriented_mesh(name, vol, chi):
    v, f, n = mc.marching_cubes(vol, 0.0)
    assert len(f) > 0 and f.dtype == np.int32 and v.dtype == np.float32
    _, cnt, directed_unique = edge_counts(f)
    assert (cnt == 2).all() and directed_unique                     # closed, consistently oriented
    if chi is not None:
        assert euler(v, f) == chi
    assert np.isfinite(v).all() and np.isfinite(n).all()
    if name == "sphere":
        c = np.array([23.3, 24.1, 22.7])
        vol_ = enclosed_volume(v, f)
        assert abs(vol_ / (4 / 3 * np.pi * 20.0 ** 3) - 1) < 0.01
        r = np.linalg.norm(v - c, axis=1)
        assert np.abs(r - 20.0).max() < 0.05
        assert (np.einsum("ij,ij->i", n, (v - c) / r[:, None]) > 0.999).all()
    if name in ("torus", "two_spheres"):
        assert enclosed_volume(v, f) > 0


@pytest.mark.parametrize("seed", range(4))
def test_oracle_mask_boundary_lies_on_unmeshed_cells(seed):
    rng = np.random.default_rng(100 + seed)
    vol = sphere(24, 8.0, (11.3, 12.1, 11.6)) if seed % 2 else gaussian_filter(rng.standard_normal((24, 24, 24)), 2).astype(np.float32)
    mask = rng.random(vol.shape) < 0.8
    v, f, _, vid = mc.marching_cubes_ids(vol, 0.0, mask)
    _, meshed = mc.cell_state(vol, 0.0, mask)
    u, cnt, directed_unique = edge_counts(f)
    assert directed_unique and cnt.max() <= 2
    n_checked = 0
    for a, b in u[cnt == 1]:
        ga, gb = vid[a], vid[b]
        pa = np.array(np.unravel_index(ga // 3, vol.shape)); pb = np.array(np.unravel_index(gb // 3, vol.shape))
        aa, ab = ga % 3, gb % 3
        # the cube face holding both lattice edges: normal to both edges' axes (perpendicular edges), or the other axis
        # along which the two edges line up (parallel edges)
        perp = 3 - aa - ab if aa != ab else [t for t in range(3) if t != aa and pa[t] == pb[t]][0]
        assert pa[perp] == pb[perp]
        x = pa[perp]
        lo = np.minimum(pa, pb)
        cells = []
        for side in (x - 1, x):
            c = lo.copy()
            c[perp] = side
            inside = all(0 <= c[t] < vol.shape[t] - 1 for t in range(3))
            cells.append(bool(meshed[tuple(c)]) if inside else False)
        assert not all(cells), (a, b)
        n_checked += 1
    assert n_checked > 0


def test_ply_round_trip(tmp_path):
    from nrw.mesh import Mesh, read_ply

    rng = np.random.default_rng(0)
    v = rng.standard_normal((50, 3))
    f = rng.integers(0, 50, (80, 3))
    n = rng.standard_normal((50, 3)).astype(np.float32)
    c = rng.integers(0, 256, (50, 3)).astype(np.uint8)
    for colors in (None, c):
        p = str(tmp_path / "m.ply")
        Mesh(v, f, n, colors).export(p)
        r = read_ply(p)
        assert np.array_equal(r["vertices"], v.astype(np.float32)) and np.array_equal(r["normals"], n)
        assert np.array_equal(r["faces"], f)
        assert (r["colors"] is None) if colors is None else np.array_equal(r["colors"], c)
    with pytest.raises(Exception):
        Mesh(v, f, n).export(str(tmp_path / "m.obj"))


def test_mc_exports_reject_bad_arguments():
    from nrw import _lib

    L = _lib.lib()
    assert L.nrw_mc_scratch_bytes(1, 4, 4) < 0 and b"nrw_mc_scratch_bytes" in L.nrw_last_error()
    assert 0 < L.nrw_mc_scratch_bytes(1024, 1024, 1024) <= 1.1 * 2 ** 30
    fake = 1 << 20                                                   # never dereferenced: the checks come first
    assert L.nrw_mc_count(None, 4, 4, 4, 0.0, None, fake, fake, None) != 0 and b"mc_count" in L.nrw_last_error()
    assert L.nrw_mc_count(fake, 4, 1, 4, 0.0, None, fake, fake, None) != 0 and b">= 2" in L.nrw_last_error()
    assert L.nrw_mc_count(fake, 4, 4, 4, 0.0, None, fake + 16, fake, None) != 0 and b"aligned" in L.nrw_last_error()
    assert L.nrw_mc_count(fake, 4, 4, 4, 0.0, None, fake, None, None) != 0 and b"counts" in L.nrw_last_error()
    assert L.nrw_mc_emit(fake, 4, 4, 4, 0.0, None, None, 1, 1, fake, fake, fake, None) != 0 and b"mc_emit" in L.nrw_last_error()
    assert L.nrw_mc_emit(fake, 4, 4, 4, 0.0, None, fake, 1 << 31, 1, fake, fake, fake, None) != 0
    assert b"n_verts" in L.nrw_last_error()
    assert L.nrw_mc_emit(fake, 4, 4, 4, 0.0, None, fake, 3, 1, None, fake, fake, None) != 0 and b"null" in L.nrw_last_error()
