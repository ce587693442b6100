"""Numpy restatement of the masked marching cubes of csrc/mcubes.cu (TEST INFRASTRUCTURE).

Same case tables (imported from csrc/gen_mc_tables.py), same vertex and face order, same float32 arithmetic:
  * cell (i,j,k) is meshed when it lies inside the volume, its 8 corners are finite and (with a mask) mask[i+1,j+1,k+1];
  * vertices are the crossing edges of meshed cells in ascending global edge id 3*lin(lower corner) + axis,
    lin(i,j,k) = (i*d1 + j)*d2 + k;  position = lower corner + t along the axis, t = (level - v_a) / (v_b - v_a);
  * faces come in cell order lin(i,j,k), table order within a cell;
  * normal = normalised lerp(t) of the lattice gradient at the two edge ends: np.gradient (central differences inside,
    one-sided at the border), where a neighbour that is not finite counts as outside the array and a component with
    neither neighbour available is 0; a zero (or non-finite) gradient gives a zero normal."""
import importlib.util
import os

import numpy as np

_GEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neuralrecon-w_b200", "csrc", "gen_mc_tables.py")
_spec = importlib.util.spec_from_file_location("gen_mc_tables", _GEN)
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)

TRI_COUNT, EDGE_MASK, TRI_TABLE = gen.tables()
CO = gen.CORNER_OFFSETS
EDGE_AXIS, EDGE_LOWER = gen.EDGE_AXIS, gen.EDGE_LOWER


def cell_state(vol, level=0.0, mask=None):
    """(case uint8 [d0-1,d1-1,d2-1], meshed bool [same])."""
    v = np.asarray(vol, dtype=np.float32)
    d0, d1, d2 = v.shape
    below = v < np.float32(level)
    fin = np.isfinite(v)
    case = np.zeros((d0 - 1, d1 - 1, d2 - 1), dtype=np.int64)
    meshed = np.ones(case.shape, dtype=bool)
    for n in range(8):
        a, b, c = CO[n]
        sl = (slice(a, a + d0 - 1), slice(b, b + d1 - 1), slice(c, c + d2 - 1))
        case |= below[sl].astype(np.int64) << n
        meshed &= fin[sl]
    if mask is not None:
        meshed &= np.asarray(mask).astype(bool)[1:, 1:, 1:]
    return case.astype(np.uint8), meshed


def gradient(vol):
    """Lattice gradient [3, d0, d1, d2] float32 (np.gradient semantics, non-finite neighbours as outside)."""
    v = np.asarray(vol, dtype=np.float32)
    fin = np.isfinite(v)
    out = np.zeros((3,) + v.shape, dtype=np.float32)
    for ax in range(3):
        vm = np.moveaxis(v, ax, 0)
        fm = np.moveaxis(fin, ax, 0)
        has_lo = np.zeros(vm.shape, dtype=bool)
        has_hi = np.zeros(vm.shape, dtype=bool)
        has_lo[1:] = fm[:-1]
        has_hi[:-1] = fm[1:]
        lo = np.zeros_like(vm)
        hi = np.zeros_like(vm)
        lo[1:] = vm[:-1]
        hi[:-1] = vm[1:]
        with np.errstate(invalid="ignore", over="ignore"):
            central = (hi - lo) * np.float32(0.5)
            fwd = hi - vm
            bwd = vm - lo
        g = np.where(has_lo & has_hi, central, np.where(has_hi, fwd, np.where(has_lo, bwd, np.float32(0))))
        out[ax] = np.moveaxis(g.astype(np.float32), 0, ax)
    return out


def marching_cubes(vol, level=0.0, mask=None):
    """-> verts float32 [V,3] (index coordinates), faces int32 [F,3], normals float32 [V,3]."""
    return marching_cubes_ids(vol, level, mask)[:3]


def marching_cubes_ids(vol, level=0.0, mask=None):
    """marching_cubes plus the global edge id of every vertex (int64 [V])."""
    v = np.ascontiguousarray(vol, dtype=np.float32)
    d0, d1, d2 = v.shape
    assert min(v.shape) >= 2
    lvl = np.float32(level)
    case, meshed = cell_state(v, level, mask)
    ntri = np.where(meshed, TRI_COUNT[case], 0).astype(np.int64)
    ci, cj, ck = np.nonzero(ntri)                                  # C order == ascending lin
    cc = case[ci, cj, ck]

    def gid(e, i, j, k):
        lo = EDGE_LOWER[e]
        return 3 * (((i + lo[..., 0]) * d1 + (j + lo[..., 1])) * d2 + (k + lo[..., 2])) + EDGE_AXIS[e]

    # vertices: every crossing edge of a meshed cell (the table uses exactly those)
    mi, mj, mk = np.nonzero(meshed & (case != 0) & (case != 255))
    mc = case[mi, mj, mk].astype(np.int64)
    ids = [gid(np.full(mi.shape, e), mi, mj, mk)[(EDGE_MASK[mc] >> e) & 1 == 1] for e in range(12)]
    vid = np.unique(np.concatenate(ids)) if ids else np.zeros(0, np.int64)
    # faces: cell order, table order within the cell
    rep = ntri[ci, cj, ck]
    cell = np.repeat(np.arange(ci.shape[0]), rep)
    slot = np.arange(cell.shape[0]) - np.repeat(np.cumsum(rep) - rep, rep)
    edges = TRI_TABLE[cc[cell], slot].astype(np.int64)            # [F,3]
    fid = gid(edges, ci[cell][:, None], cj[cell][:, None], ck[cell][:, None])
    faces = np.searchsorted(vid, fid).astype(np.int32).reshape(-1, 3)
    # positions and normals
    lin, axis = vid // 3, vid % 3
    p = np.stack(np.unravel_index(lin, v.shape), -1)
    stride = np.array([d1 * d2, d2, 1], dtype=np.int64)
    flat = v.reshape(-1)
    va, vb = flat[lin], flat[lin + stride[axis]]
    t = ((lvl - va) / (vb - va)).astype(np.float32)
    verts = p.astype(np.float32)
    r = np.arange(vid.shape[0])
    verts[r, axis] = verts[r, axis] + t
    G = gradient(v).reshape(3, -1)
    ga, gb = G[:, lin].T, G[:, lin + stride[axis]].T
    g = (ga + t[:, None] * (gb - ga)).astype(np.float32)
    nrm = np.sqrt(g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1] + g[:, 2] * g[:, 2]).astype(np.float32)
    ok = (nrm > 0) & np.isfinite(nrm)
    normals = np.zeros_like(g)
    normals[ok] = g[ok] / nrm[ok, None]
    return verts.reshape(-1, 3), faces, normals.reshape(-1, 3), vid
