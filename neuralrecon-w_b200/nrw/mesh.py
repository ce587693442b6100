"""Device-resident SDF-grid evaluation for mesh extraction (SURVEY.md 8f-1; BASELINE config 5).

Mirrors the SDF half of utils/visualization.py::extract_mesh (lines 36-107) and tools/extract_mesh.py::gen_grid_spc
(lines 60-102).  The reference builds the query lattice on the CPU, ships every chunk to the GPU, copies every SDF
chunk back (`.cpu()` per chunk), all-gathers and scatters into a dense volume on the host.  Here the lattice points are
GENERATED on the device chunk by chunk (nrw_grid_points_dense / nrw_grid_points_sparse) straight into the SDF query
(nrw_sdf_query), ranks take the contiguous slices of get_local_split (utils/visualization.py:27-35) and one
all_gather joins them; the dense volume, the validity mask and the scatter stay on the GPU.  `sdf_volume` /
`sparse_sdf_volume` return exactly the arrays the reference hands to skimage.measure.marching_cubes.

`marching_cubes` is this library's own masked marching cubes on the device (csrc/mcubes.cu states its rules; it does not
reproduce skimage's triangulation), and `extract_mesh` is a drop-in for utils/visualization.py::extract_mesh that returns
a `Mesh` whose `export(path)` writes binary PLY, so neither skimage nor trimesh is needed."""
import os
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from ._lib import NrwError, check, ptr, stream_ptr


def _f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def _local_range(n, world, rank):
    """get_local_split (utils/visualization.py:27-35): pad to a multiple of world, contiguous slice per rank.
    Returns (start, stop_unpadded, slice_length)."""
    per = n // world if n % world == 0 else n // world + 1
    a = rank * per
    return a, min(n, a + per), per


def _gather_slices(local, per, n, world):
    """all_gather of equal-length slices (utils/visualization.py:81-88) -> first n entries, on every rank."""
    if world == 1:
        return local[:n]
    if local.shape[0] < per:                  # this rank's slice reaches into the zero padding
        local = torch.cat([local, torch.zeros(per - local.shape[0], dtype=local.dtype, device=local.device)])
    parts = [torch.empty(per, dtype=local.dtype, device=local.device) for _ in range(world)]
    dist.all_gather(parts, local.contiguous())                   # NCCL over NVLink in training; the reference's collective
    return torch.cat(parts, 0)[:n]


def sdf_volume(renderer, dim, origin=(0.0, 0.0, 0.0), radius=1.0, chunk=1 << 20):
    """Dense branch of extract_mesh (sparse_data=None): SDF on the dim^3 lattice of
    torch.linspace(origin[c]-radius, origin[c]+radius, dim), returned as a float32 CUDA tensor [dim,dim,dim]
    (= `sdf.reshape((dim,dim,dim))` of utils/visualization.py:96), plus (vol_origin, voxel_size)."""
    L = _lib.lib()
    eng = renderer.engine
    dev = next(renderer.neuconw.parameters()).device
    if dev.type != "cuda":
        raise NrwError("sdf_volume: the networks must live on a CUDA device")
    o64 = np.array(origin, dtype=np.float64)
    lo, hi = (o64 - radius).astype(np.float32), (o64 + radius).astype(np.float32)
    n = int(dim) ** 3
    world, rank = _world()
    a, b, per = _local_range(n, world, rank)
    local = torch.empty(max(b - a, 0), dtype=torch.float32, device=dev)
    pts = torch.empty(min(chunk, max(b - a, 1)), 3, dtype=torch.float32, device=dev)
    eng.ensure(dev, 1, 2, 0, chunk_hint=pts.shape[0])
    eng.pack(dev)
    with torch.no_grad():
        for i in range(a, b, pts.shape[0]):
            m = min(pts.shape[0], b - i)
            check(L.nrw_grid_points_dense(int(dim), _f3(lo), _f3(hi), i, m, ptr(pts), stream_ptr()), "nrw_grid_points_dense")
            check(L.nrw_sdf_query(eng.ctx, ptr(pts), m, C.c_void_p(local.data_ptr() + (i - a) * 4), stream_ptr()), "nrw_sdf_query")
    sdf = _gather_slices(local, per, n, world)
    return sdf.reshape(dim, dim, dim), (o64 - radius), 2 * radius / (dim - 1)


def gen_grid_spc(renderer, eval_level, device=0):
    """tools/extract_mesh.py:60-102 without materialising the candidate list: returns the description of the
    up-sampled sparse lattice {leaves int16 [m,3] (lexicographic), up_times, voxel_size, dim, vol_origin}."""
    if renderer.octree_data is None:
        renderer.octree_data = renderer.get_octree(device)
    od = renderer.octree_data
    spc = od["spc_data"]
    L0 = int(od["level"])
    pyr = spc["pyramid"]
    leaves = spc["points"][int(pyr[1, L0]):int(pyr[1, L0 + 1])].to(torch.int64)
    key = (leaves[:, 0] * (1 << L0) + leaves[:, 1]) * (1 << L0) + leaves[:, 2]
    leaves = leaves[torch.argsort(key)].to(torch.int16).contiguous()          # torch.nonzero(dense) order
    up_times = 2 ** (int(eval_level) - L0)
    if up_times < 1:
        raise NrwError(f"gen_grid_spc: eval_level {eval_level} below the octree level {L0}")
    scale = od["scale"]
    return {"leaves": leaves, "up_times": up_times, "voxel_size": 2 / (2 ** int(eval_level)) * scale,
            "dim": int((2 ** L0) * up_times), "vol_origin": od["scene_origin"].float().cpu() - scale}


def sparse_candidates(renderer, grid, chunk=1 << 20, threshold=None, sdf_fn=None, want_sdf=True):
    """SDF of every candidate of an up-sampled sparse lattice (gen_grid_spc / surface_selection), chunked:
    points generated on the device, SDF through nrw_sdf_query (or `sdf_fn(xyz_training)` in tests), ranks split and
    all-gather as the reference does (neuconw_system.py:236-258).  With `threshold` the stable compaction
    xyz_sfm[sdf <= threshold] (neuconw_system.py:259) runs chunk by chunk on the device as well.
    Returns dict(sdf [n] or None, kept_xyz_sfm [m,3] or None, n)."""
    L = _lib.lib()
    eng = renderer.engine
    leaves = grid["leaves"]
    dev = leaves.device
    up = int(grid["up_times"])
    n = int(leaves.shape[0]) * up ** 3
    voxel = float(np.float32(grid["voxel_size"]))
    vol_origin = [float(x) for x in grid["vol_origin"]]
    scene_origin = [float(x) for x in torch.as_tensor(renderer.origin).float().cpu()]
    radius = float(renderer.radius)
    world, rank = _world()
    a, b, per = _local_range(n, world, rank)
    local = torch.empty(max(b - a, 0), dtype=torch.float32, device=dev)
    c = min(chunk, max(b - a, 1))
    xt = torch.empty(c, 3, dtype=torch.float32, device=dev)
    if sdf_fn is None:
        eng.ensure(dev, 1, 2, 0, chunk_hint=c)
        eng.pack(dev)
    with torch.no_grad():
        for i in range(a, b, c):
            m = min(c, b - i)
            check(L.nrw_grid_points_sparse(ptr(leaves), leaves.shape[0], up, voxel, _f3(vol_origin), _f3(scene_origin), radius,
                                           i, m, None, ptr(xt), stream_ptr()), "nrw_grid_points_sparse")
            if sdf_fn is None:
                check(L.nrw_sdf_query(eng.ctx, ptr(xt), m, C.c_void_p(local.data_ptr() + (i - a) * 4), stream_ptr()), "nrw_sdf_query")
            else:
                local[i - a:i - a + m] = sdf_fn(xt[:m]).reshape(-1)
    sdf = _gather_slices(local, per, n, world)
    kept = None
    if threshold is not None:
        # capacity: every candidate for small lattices, an exact count first for large ones
        total = n if n <= (1 << 24) else int((sdf <= threshold).sum())
        cap = torch.empty(max(total, 1), 3, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        xs = torch.empty(c, 3, dtype=torch.float32, device=dev)
        sb = L.nrw_compact_scratch_bytes(c)
        scratch = torch.empty(sb + 256, dtype=torch.uint8, device=dev)
        sp = (scratch.data_ptr() + 255) // 256 * 256
        for i in range(0, n, c):
            m = min(c, n - i)
            check(L.nrw_grid_points_sparse(ptr(leaves), leaves.shape[0], up, voxel, _f3(vol_origin), _f3(scene_origin), radius,
                                           i, m, ptr(xs), ptr(xt), stream_ptr()), "nrw_grid_points_sparse")
            check(L.nrw_threshold_compact(C.c_void_p(sdf.data_ptr() + i * 4), ptr(xs), m, float(threshold), ptr(cap), ptr(count),
                                          C.c_void_p(sp), stream_ptr()), "nrw_threshold_compact")
        kept = cap[:int(count)]
    return {"sdf": sdf if want_sdf else None, "kept_xyz_sfm": kept, "n": n}


def sparse_sdf_volume(renderer, grid, chunk=1 << 20, sdf_fn=None):
    """Sparse branch of extract_mesh (utils/visualization.py:53-66,98-116): returns (sdf_dense [dim]^3 float32 CUDA, ones
    outside the lattice; mask_dense bool CUDA - a cell is valid iff all 8 of its corners are lattice points)."""
    res = sparse_candidates(renderer, grid, chunk=chunk, sdf_fn=sdf_fn)
    leaves, up, dim = grid["leaves"].to(torch.int64), int(grid["up_times"]), int(grid["dim"])
    k = torch.arange(up, device=leaves.device)
    kern = torch.stack(torch.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    ind = (leaves[:, None, :] * up + kern[None, :, :]).reshape(-1, 3)          # ind = round((xyz - vol_origin)/voxel)
    return _scatter_volume(ind, res["sdf"], dim)


def _scatter_volume(ind, sdf, dim):
    """utils/visualization.py:98-116: SDF values at lattice indices ind [n,3] -> (dense volume, ones elsewhere; mask)."""
    dev = ind.device
    sdf_dense = torch.ones(dim, dim, dim, dtype=torch.float32, device=dev)
    sdf_dense[ind[:, 0], ind[:, 1], ind[:, 2]] = sdf
    m = torch.zeros(dim, dim, dim, dtype=torch.bool, device=dev)
    m[ind[:, 0], ind[:, 1], ind[:, 2]] = True
    # a marching-cubes cell (i, j, k) uses the corners (i - a, j - b, k - c), a, b, c in {0, 1} (wrap-around as torch.roll)
    valid = m.clone()
    for shift in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)):
        valid &= torch.roll(m, shifts=shift, dims=(0, 1, 2))
    return sdf_dense, valid


def marching_cubes(volume, level=0.0, mask=None):
    """Masked marching cubes of a CUDA fp32 volume [d0,d1,d2] (csrc/mcubes.cu): -> (verts fp32 [V,3] in index
    coordinates, faces int32 [F,3], normals fp32 [V,3]), CUDA tensors.  With `mask` (bool or uint8, same shape) cell
    (i,j,k) is meshed only when mask[i+1,j+1,k+1] is set, so `marching_cubes(*sparse_sdf_volume(r, grid))` works as is.
    One host read (the two counts) between the count and emit passes."""
    L = _lib.lib()
    if not (torch.is_tensor(volume) and volume.is_cuda and volume.dim() == 3):
        raise NrwError("marching_cubes: volume must be a 3-D CUDA tensor")
    if min(volume.shape) < 2:
        raise NrwError(f"marching_cubes: every dimension must be >= 2 (got {tuple(volume.shape)})")
    vol = volume.to(torch.float32).contiguous()
    d0, d1, d2 = (int(x) for x in vol.shape)
    m = None
    if mask is not None:
        if tuple(mask.shape) != tuple(vol.shape) or mask.device != vol.device:
            raise NrwError("marching_cubes: mask must have the volume's shape and device")
        m = (mask != 0).to(torch.uint8).contiguous()
    sb = L.nrw_mc_scratch_bytes(d0, d1, d2)
    if sb < 0:
        check(sb, "nrw_mc_scratch_bytes")
    scratch = torch.empty(sb + 256, dtype=torch.uint8, device=vol.device)
    sp = C.c_void_p((scratch.data_ptr() + 255) // 256 * 256)
    counts = torch.empty(2, dtype=torch.int64, device=vol.device)
    lvl = float(level)
    check(L.nrw_mc_count(ptr(vol), d0, d1, d2, lvl, ptr(m), sp, ptr(counts), stream_ptr()), "nrw_mc_count")
    nv, nf = counts.tolist()
    verts = torch.empty(nv, 3, dtype=torch.float32, device=vol.device)
    normals = torch.empty(nv, 3, dtype=torch.float32, device=vol.device)
    faces = torch.empty(nf, 3, dtype=torch.int32, device=vol.device)
    check(L.nrw_mc_emit(ptr(vol), d0, d1, d2, lvl, ptr(m), sp, nv, nf, ptr(verts), ptr(normals), ptr(faces), stream_ptr()),
          "nrw_mc_emit")
    return verts, faces, normals


class Mesh:
    """The slice of trimesh.Trimesh that extract_mesh's callers use: vertices float64 [V,3], faces int64 [F,3],
    vertex_normals float32 [V,3], vertex_colors uint8 [V,3] or None (numpy), and export(path)."""

    def __init__(self, vertices, faces, vertex_normals, vertex_colors=None):
        self.vertices = np.asarray(vertices)
        self.faces = np.asarray(faces, dtype=np.int64)
        self.vertex_normals = np.asarray(vertex_normals)
        self.vertex_colors = None if vertex_colors is None else np.asarray(vertex_colors, dtype=np.uint8)

    def export(self, path):
        """Binary little-endian PLY: vertex x y z nx ny nz (float32) [red green blue (uchar)], face list uchar int."""
        if os.path.splitext(str(path))[1].lower() != ".ply":
            raise NrwError(f"Mesh.export: only .ply is supported (got {path})")
        write_ply(path, self.vertices, self.faces, self.vertex_normals, self.vertex_colors)


def write_ply(path, vertices, faces=None, normals=None, colors=None):
    """Binary little-endian PLY: vertex x y z [nx ny nz] (float32) [red green blue (uchar)], and with `faces` a face list
    uchar int.  faces=None and normals=None write a point cloud."""
    n = len(vertices)
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if normals is not None else [])
    fields = [(name, "<f4") for name in names]
    if colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    v = np.empty(n, dtype=fields)
    for c, name in enumerate("xyz"):
        v[name] = vertices[:, c]
        if normals is not None:
            v["n" + name] = normals[:, c]
    if colors is not None:
        for c, name in enumerate(("red", "green", "blue")):
            v[name] = colors[:, c]
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    head += [f"property float {name}" for name in names]
    if colors is not None:
        head += [f"property uchar {name}" for name in ("red", "green", "blue")]
    if faces is not None:
        fc = np.empty(len(faces), dtype=[("n", "u1"), ("i", "<i4", (3,))])
        fc["n"] = 3
        fc["i"] = faces
        head += [f"element face {len(faces)}", "property list uchar int vertex_indices"]
    head += ["end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(v.tobytes())
        if faces is not None:
            fh.write(fc.tobytes())


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def _ply_header(data):
    """-> (format, [(element name, count, [(property name, type) or (name, ("list", count type, item type))])], body offset)"""
    if not data.startswith(b"ply"):
        raise NrwError("read_ply: not a PLY file")
    end = data.find(b"end_header")
    if end < 0:
        raise NrwError("read_ply: no end_header")
    body = data.index(b"\n", end) + 1
    fmt, elems = None, []
    for line in data[:end].decode("ascii", "replace").splitlines():
        t = line.split()
        if not t or t[0] in ("ply", "comment", "obj_info"):
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elems.append((t[1], int(t[2]), []))
        elif t[0] == "property" and elems:
            try:
                if t[1] == "list":
                    elems[-1][2].append((t[4], ("list", _PLY_TYPES[t[2]], _PLY_TYPES[t[3]])))
                else:
                    elems[-1][2].append((t[2], _PLY_TYPES[t[1]]))
            except KeyError as e:
                raise NrwError(f"read_ply: unknown property type in {line!r}") from e
    if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
        raise NrwError(f"read_ply: unsupported format {fmt}")
    return fmt, elems, body


def read_ply(path):
    """PLY reader for meshes and point clouds: ascii, binary little- and big-endian; any scalar vertex property type; an
    optional triangle face list with any integer count and index types (other polygons raise NrwError).  Returns a dict of
    numpy arrays: vertices [V,3] (x, y, z in their stored type), normals [V,3] or None, colors uint8 [V,3] or None,
    faces int64 [F,3] (empty without a face element)."""
    with open(path, "rb") as fh:
        data = fh.read()
    fmt, elems, pos = _ply_header(data)
    bo = "<" if fmt == "binary_little_endian" else ">"
    tokens = data[pos:].split() if fmt == "ascii" else None
    tok = 0
    vert, faces = None, np.zeros((0, 3), np.int64)
    for name, count, props in elems:
        lists = [p for p in props if isinstance(p[1], tuple)]
        if fmt == "ascii":
            rows = []
            for _ in range(count):
                row = {}
                for pname, ptype in props:
                    if isinstance(ptype, tuple):
                        k = int(tokens[tok])
                        row[pname] = tokens[tok + 1:tok + 1 + k]
                        tok += 1 + k
                    else:
                        row[pname] = tokens[tok]
                        tok += 1
                rows.append(row)
            if name == "face":
                if len(lists) != 1 or any(len(r[lists[0][0]]) != 3 for r in rows):
                    raise NrwError("read_ply: only triangle faces are supported")
                faces = np.array([[int(x) for x in r[lists[0][0]]] for r in rows], np.int64).reshape(-1, 3)
            elif name == "vertex":
                vert = {p: np.array([float(r[p]) for r in rows]).astype(t) for p, t in props if not isinstance(t, tuple)}
            continue
        if name == "face" and len(lists) == 1:
            cnt_t, idx_t = lists[0][1][1], lists[0][1][2]
            # read as if every face were a triangle; the first count that is not 3 sits at its true offset
            fields = []
            for p, t in props:
                if isinstance(t, tuple):
                    fields += [(p + "__n", bo + cnt_t), (p, bo + idx_t, (3,))]
                else:
                    fields.append((p, bo + t))
            dt = np.dtype(fields)
            if pos + dt.itemsize * count > len(data):
                raise NrwError("read_ply: file shorter than its face element (or polygons that are not triangles)")
            fc = np.frombuffer(data, dtype=dt, count=count, offset=pos)
            if (fc[lists[0][0] + "__n"] != 3).any():
                raise NrwError("read_ply: only triangle faces are supported")
            faces = fc[lists[0][0]].astype(np.int64).reshape(-1, 3)
            pos += dt.itemsize * count
            continue
        if lists:
            raise NrwError(f"read_ply: list properties are only supported in the face element (element {name})")
        dt = np.dtype([(p, bo + t) for p, t in props])
        if pos + dt.itemsize * count > len(data):
            raise NrwError(f"read_ply: file shorter than its {name} element")
        arr = np.frombuffer(data, dtype=dt, count=count, offset=pos)
        pos += dt.itemsize * count
        if name == "vertex":
            vert = {p: arr[p].astype(arr[p].dtype.newbyteorder("=")) for p, _ in props}
    if vert is None or not all(c in vert for c in "xyz"):
        raise NrwError("read_ply: no vertex element with x, y, z")

    def stack(names):
        return np.stack([vert[n] for n in names], 1) if all(n in vert for n in names) else None

    colors = stack(("red", "green", "blue"))
    return {"vertices": stack(("x", "y", "z")), "normals": stack(("nx", "ny", "nz")), "faces": faces,
            "colors": None if colors is None else colors.astype(np.uint8)}


def _sdf_at(renderer, xyz, chunk):
    """renderer.sdf at training-coordinate points xyz [n,3] (CUDA), rank slices + all_gather as the reference."""
    n = xyz.shape[0]
    world, rank = _world()
    a, b, per = _local_range(n, world, rank)
    local = torch.empty(max(b - a, 0), dtype=torch.float32, device=xyz.device)
    with torch.no_grad():
        for i in range(a, b, chunk):
            m = min(chunk, b - i)
            local[i - a:i - a + m] = renderer.sdf(xyz[i:i + m].reshape(-1, 1, 3)).reshape(-1)
    return _gather_slices(local, per, n, world)


def extract_mesh(dim, chunk, scene_radius, scene_origin, origin=None, radius=1.0, with_color=False, embedding_a=None,
                 chunk_rgb=256, sparse_data=None, renderer=None):
    """Drop-in for utils/visualization.py::extract_mesh (same signature): SDF volume, marching cubes and vertex colours
    on the GPU; rank 0 returns a `Mesh` (world coordinates), other ranks None.  `sparse_data` is either the reference's
    dict (sparse_vol [n,3] SfM points, voxel_size, dim, vol_origin) or the one gen_grid_spc returns (leaves, ...).
    Colours: renderer.rgb at the training-coordinate vertices, direction (0,0,1), stored as uint8 clamp(round(255 rgb))."""
    if origin is None:
        origin = [0, 0, 0]
    dev = next(renderer.neuconw.parameters()).device
    if sparse_data is None:
        vol, vol_origin, voxel_size = sdf_volume(renderer, dim, origin=origin, radius=radius, chunk=chunk)
        mask = None
        to_train = lambda v: v * voxel_size + vol_origin                       # float32 * float -> float32, + float64
        to_world = lambda v: v * scene_radius + np.array(scene_origin)
    else:
        # utils/visualization.py:57-65: training-coordinate origin and voxel size of the sparse lattice
        vol_origin_sfm = torch.from_numpy(np.array(sparse_data["vol_origin"])).float()
        so = torch.from_numpy(np.array(scene_origin)).float()
        vol_origin = ((vol_origin_sfm - so) / scene_radius).numpy()
        voxel_size = sparse_data["voxel_size"] / scene_radius
        if "leaves" in sparse_data:
            vol, mask = sparse_sdf_volume(renderer, sparse_data, chunk=chunk)
        else:
            sv = torch.as_tensor(sparse_data["sparse_vol"]).float()
            ind = torch.round((sv - vol_origin_sfm) / sparse_data["voxel_size"]).long().to(dev)
            xyz = ((sv - so) / scene_radius).to(dev)
            vol, mask = _scatter_volume(ind, _sdf_at(renderer, xyz, chunk), int(sparse_data["dim"]))
        so_np = so.numpy()
        to_train = lambda v: v * voxel_size + vol_origin                       # float32 throughout
        to_world = lambda v: v * scene_radius + so_np
    verts, faces, normals = marching_cubes(vol, 0.0, mask)
    verts_t = to_train(verts.cpu().numpy())
    verts_w = to_world(verts_t)
    colors = None
    if with_color:
        world, rank = _world()
        n = verts_t.shape[0]
        a, b, per = _local_range(n, world, rank)
        pts = torch.from_numpy(np.ascontiguousarray(verts_t)).float().to(dev)
        emb = embedding_a.detach().reshape(1, -1).to(dev)
        local = torch.empty(max(b - a, 0), 3, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for i in range(a, b, chunk_rgb):
                m = min(chunk_rgb, b - i)
                d = torch.zeros(m, 1, 3, dtype=torch.float32, device=dev)
                d[:, :, 2] = 1
                local[i - a:i - a + m] = renderer.rgb(pts[i:i + m].reshape(-1, 1, 3), d, emb.repeat(m, 1).reshape(m, 1, -1))
        rgb = _gather_slices(local.reshape(-1), per * 3, n * 3, world).reshape(n, 3)
        colors = torch.round(rgb * 255).clamp(0, 255).to(torch.uint8).cpu().numpy()
    if _world()[1] != 0:
        return None
    return Mesh(verts_w, faces.cpu().numpy(), normals.cpu().numpy(), colors)
