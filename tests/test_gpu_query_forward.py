"""GPU: the forward values of the standalone network queries (NeuconW.sdf, the gradient query, NeuconW.forward,
NeRF.forward and the indoor NeRF without the appearance head) against the port evaluated in fp64, on every path the SDF
query dispatches to, and their independence of how the points are batched.

Reference: oracle/neuconw_port.py sdf_forward, the normal as the autograd gradient of the SDF, color_forward and
nerf_forward, and util_indoor.nerf_forward_noapp (test_gpu_query_backward.ref_outputs), in fp64 and in fp32 as the
anchor of the tolerance rule.

Paths of a forward-only SDF query (engine.cu sdf_query / sdf_chunk_forward) with chunks of CHUNK = 1024 rows:
  fused chain (sdf_fused_kernel, no chunks)     tensor cores, 2 planes (bf16x3, mixed): every n
  per-layer chain, head fused into layer 7's    tensor cores, 1 or 3 planes (bf16, bf16x6), and 2 planes with
    epilogue (FWD_HEAD + sdf_head_sum)          NRW_SDF_FUSED=0: every chunk, of any number of rows
  per-layer chain, sdf_head_kernel on the       CUDA cores (bf16x6_simt): every chunk
    planes of u_8
The gradient and forward queries run the per-layer chain with sdf_head_kernel and the normal chain (GATE_FWD,
sdf_normal_kernel) on every backend.  SIZES put one chunk on either side of the 128-row tile and of 256 rows (where
the tensor-core chain used to switch a short chunk to sdf_head_kernel), and two whole chunks before a ragged tail of
200 and of 300 rows; the SDF query also runs BIG rows (many fused-chain CTAs, a ragged last 64-row tile).

Parameters: util_network_bwd.make_params("surface"), whose SDF crosses zero at |x| ~ 0.5 .. 0.7.
Inputs (edge_inputs): points up to |x| = 1.2 per coordinate (PE6 arguments up to 38 rad), every 4th row of the first
1024 on the SDF's zero level set; NeRF points [p/r, 1/r] with r log-uniform in [1, 1e4] (PE10 arguments up to 512
rad, 1/r down to 1e-4); unit view directions; codes from N(0, 1), every 16th row with entries of +/-5.

Tolerance (util_network_bwd's rule): the error of an output is tensor_err (sdf, density) or ray_err per row (normals,
rgb) against fp64; it passes at max(ANCHOR_FACTOR x the fp32 evaluation's error, the mode's floor).  wgmma's fp32
accumulation does not round to nearest (test_gpu_network_bwd.py), so on the tensor cores the SDF value and the normal
carry a bias of ~20x the fp32 reference's error even with three planes: the floors below were measured on an H100
(700 W), the worst over SIZES (and BIG), with the measured worst in brackets.
  bf16x6 on the CUDA cores   sdf 2e-6 (8.8e-7)  normals 1e-5 (4.9e-6)    rgb 1e-5 (5.2e-6)   density 1e-6 (3.3e-7)
  bf16x6 on the tensor cores sdf 5e-5 (2.4e-5)  normals 2.5e-4 (1.1e-4)  rgb 4e-5 (1.7e-5)   density 5e-6 (2.2e-6)
  bf16x3, mixed, per-layer   sdf 4e-5 (1.6e-5)  normals 2.5e-4 (1.1e-4)  rgb 3e-4 (1.3e-4)   density 2e-5 (8.1e-6)
(rgb: the worst of the colour net and the NeRF, the indoor NeRF's in every mode).  The SDF and the density are judged
against max|ref| + 1 (SCALAR_UNIT): a batch of a few rows on the zero level set has no scale of its own.
bf16 (one plane) is reported only: every output finite and at cosine >= 0.99 to fp64.

Batch invariance: 300 fixed rows give bit-identical outputs (torch.equal) in every mode and query whether queried
alone, at the start of a 2 x 1024 + 200 batch, at its end (the 200-row ragged tail) or at the end of a 2 x 1024 + 300
batch (include/nrw.h: results do not depend on how the caller batches the points); and nrw_sample's z_vals in bf16 do
not depend on whether its SDF query leaves a ragged chunk of under 256 rows.

Appearance width: NeuconW.forward and NeRF.forward at n_a in {1, 47, 96} under the same rule, and at n_a = 47 the
backward of both (the code gradient and static_linear_0's weights) under test_gpu_query_backward's rule."""
import functools
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import test_gpu_query_backward as qb
import util_network_bwd as un
from conftest import ROOT
from util_nrw import port, synth

pytestmark = pytest.mark.gpu
CHUNK = 1024
SIZES = (1, 127, 255, 256, 257, 300, 2 * CHUNK + 200, 2 * CHUNK + 300)
BIG = 70001
N_A = qb.N_A
VARIANT = "surface"      # the synthetic parameters with an SDF that has a zero level set (util_network_bwd)
# the outputs judged per query (the gradient query also returns the SDF)
OUTPUTS = dict(sdf=("sdf",), gradient=("sdf", "normals"), forward=("rgb", "sdf", "normals"), nerf=("density", "rgb"),
               nerf_indoor=("density", "rgb"))
ROW_VECTORS = ("normals", "rgb")
SCALAR_UNIT = 1.0        # sdf and density errors are relative to max|ref| + SCALAR_UNIT
# mode: (precision, GEMM backend); PER_LAYER runs in a subprocess with NRW_SDF_FUSED=0
MODES = {"bf16x6_simt": ("bf16x6", 1), "bf16x6_tc": ("bf16x6", 0), "bf16x3_tc": ("bf16x3", 0), "mixed_tc": ("mixed", 0)}
REPORTED = {"bf16_tc": ("bf16", 0)}
PER_LAYER = "bf16x3_per_layer"
ALL_MODES = {**MODES, **REPORTED, PER_LAYER: ("bf16x3", 0)}
# mode: {output: floor} (docstring)
FLOORS = {
    "bf16x6_simt": dict(sdf=2e-6, normals=1e-5, rgb=1e-5, density=1e-6),
    "bf16x6_tc": dict(sdf=5e-5, normals=2.5e-4, rgb=4e-5, density=5e-6),
    "bf16x3_tc": dict(sdf=4e-5, normals=2.5e-4, rgb=3e-4, density=2e-5),
    "mixed_tc": dict(sdf=4e-5, normals=2.5e-4, rgb=3e-4, density=2e-5),
}
FLOORS[PER_LAYER] = FLOORS["bf16x3_tc"]
COSINE_MIN = 0.99


# ------------------------------------------------------------------------------------------------------ inputs
@functools.lru_cache(maxsize=None)
def level_set_points(seed, n_a=N_A, k=CHUNK // 4):
    """k points on the zero level set of the SDF (fp64 bisection along rays from the origin), as fp32."""
    Q = {key: v.double() for key, v in qb.params(False, n_a, VARIANT).items() if key.startswith("neuconw.sdf_net.")}
    g = torch.Generator().manual_seed(seed)
    u = F.normalize(torch.randn(k, 3, generator=g, dtype=torch.float64), dim=-1)
    f = lambda r: port.sdf_forward(Q, u * r[:, None])[:, 0]
    with torch.no_grad():
        grid = torch.linspace(0.05, 1.2, 24, dtype=torch.float64)
        vals = torch.stack([f(torch.full((k,), float(r), dtype=torch.float64)) for r in grid], -1)
        change = (vals[:, :-1] * vals[:, 1:] <= 0)
        assert change.any(-1).all(), "the synthetic SDF has no zero crossing on some ray"
        j = change.float().argmax(-1)
        lo, hi, flo = grid[j], grid[j + 1], vals.gather(1, j[:, None])[:, 0]
        for _ in range(40):
            mid = 0.5 * (lo + hi)
            fm = f(mid)
            left = (fm * flo) <= 0
            hi, lo, flo = torch.where(left, mid, hi), torch.where(left, lo, mid), torch.where(left, flo, fm)
    return (u * (0.5 * (lo + hi))[:, None]).float()


@functools.lru_cache(maxsize=None)
def edge_inputs(n, seed=21, n_a=N_A):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 1.2
    on = torch.arange(0, min(n, CHUNK), 4)
    pts[on] = level_set_points(seed, n_a)[:len(on)]
    dirs = F.normalize(torch.randn(n, 3, generator=g), dim=-1)
    a = torch.randn(n, n_a, generator=g)
    loud = torch.arange(5, max(n, 5), 16)
    a[loud] = 5.0 * torch.sign(torch.randn(len(loud), n_a, generator=g))
    u = F.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
    r = 10.0 ** (4.0 * torch.rand(n, 1, generator=g, dtype=torch.float64))
    r[0::97], r[1::97] = 1.0, 1e4
    p = u * r
    pts4 = torch.cat([p / r, 1.0 / r], -1).float()
    return dict(pts=pts, dirs=dirs, a=a, pts4=pts4)


# ------------------------------------------------------------------------------------------------------ reference
@functools.lru_cache(maxsize=None)
def reference(query, n, dtype, n_a=N_A):
    """{output: value} of the port in `dtype` on edge_inputs(n)."""
    P = qb.params(query == "nerf_indoor", n_a, VARIANT)
    Q = {k: v.to(dtype) for k, v in un.net_params(P).items()}
    inp = edge_inputs(n, n_a=n_a)
    if query == "sdf":                 # no normal: BIG rows
        with torch.no_grad():
            return dict(sdf=port.sdf_forward(Q, inp["pts"].to(dtype))[:, 0])
    x = {k: v.to(dtype).clone().requires_grad_(k == "pts") for k, v in inp.items()}
    out = qb.ref_outputs(query, Q, x)
    return {k: out[k].detach() for k in OUTPUTS[query]}


def sizes_of(query):
    return SIZES + ((BIG,) if query == "sdf" else ())


# ------------------------------------------------------------------------------------------------------ CUDA
@functools.lru_cache(maxsize=None)
def modules(precision, backend, indoor=False, n_a=N_A):
    """(neuconw, nerf, engine) over chunks of CHUNK rows, kept until the module's tests end (release_engines; the
    modules hold the engine weakly)."""
    _, neuconw, nerf, eng = qb.make_modules(precision, backend, indoor=indoor, chunk_rows=CHUNK, n_a=n_a, variant=VARIANT)
    return neuconw, nerf, eng


@pytest.fixture(scope="module", autouse=True)
def release_engines():
    """frees every cached engine's packed weights and workspace when this module's tests are done."""
    yield
    modules.cache_clear()
    torch.cuda.empty_cache()


def run_query(mods, query, inp):
    """{output: CPU tensor} of the inference call of `query` on inp."""
    neuconw, nerf, eng = mods
    x = {k: v.cuda() for k, v in inp.items()}
    n = x["pts"].shape[0]
    with torch.no_grad():
        if query == "sdf":
            out = dict(sdf=neuconw.sdf(x["pts"]).reshape(-1))
        elif query == "gradient":
            _, sdf, nrm = eng.neuconw_forward(x["pts"], None, None, want_rgb=False)
            out = dict(sdf=sdf, normals=nrm)
        elif query == "forward":
            rgb, _, sdf, nrm = neuconw(torch.cat([x["pts"], x["dirs"], x["a"]], -1).view(1, n, -1))
            out = dict(rgb=rgb.reshape(n, 3), sdf=sdf.reshape(n), normals=nrm.reshape(n, 3))
        else:
            dens, rgb = nerf(x["pts4"], x["dirs"], x["a"])
            out = dict(density=dens.reshape(n), rgb=rgb)
    return {k: v.cpu() for k, v in out.items()}


def slice_inputs(inp, rows):
    return {k: v[rows] for k, v in inp.items()}


def cat_inputs(*parts):
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def invariance_batches():
    """(name, inputs, rows of the 300 fixed rows in them) per placement."""
    fixed, fill = edge_inputs(300, seed=31), edge_inputs(2 * CHUNK, seed=32)
    n_lead = 2 * CHUNK + 200 - 300
    return [("alone", fixed, slice(0, 300)),
            ("start of 2x1024+200", cat_inputs(fixed, slice_inputs(fill, slice(0, n_lead))), slice(0, 300)),
            ("ragged 200-row tail of 2x1024+200", cat_inputs(slice_inputs(fill, slice(0, n_lead)), fixed),
             slice(n_lead, n_lead + 300)),
            ("300-row tail of 2x1024+300", cat_inputs(fill, fixed), slice(2 * CHUNK, 2 * CHUNK + 300))]


def mode_outputs(mode, queries):
    """{("fp64", query, n): outputs, ("inv", query, placement): outputs of the fixed rows} of one mode."""
    prec, backend = ALL_MODES[mode]
    res = {}
    for query in queries:
        mods = modules(prec, backend, indoor=query == "nerf_indoor")
        for n in sizes_of(query):
            res[("fp64", query, n)] = run_query(mods, query, edge_inputs(n))
        for name, inp, rows in invariance_batches():
            res[("inv", query, name)] = {k: v[rows] for k, v in run_query(mods, query, inp).items()}
    return res


@functools.lru_cache(maxsize=None)
def per_layer_outputs():
    """mode_outputs of the SDF query with NRW_SDF_FUSED=0, in a process of its own (the switch is read once)."""
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "per_layer.pt")
        code = ("import sys, torch; sys.path[:0] = ['tests', '.', 'neuralrecon-w_b200']\n"
                "import test_gpu_query_forward as t\n"
                f"torch.save(t.mode_outputs({PER_LAYER!r}, ('sdf',)), {path!r})\n")
        r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, NRW_SDF_FUSED="0"),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        return torch.load(path)


@functools.lru_cache(maxsize=None)
def outputs(mode, query):
    if mode == PER_LAYER:
        return per_layer_outputs()
    return mode_outputs(mode, (query,))


# ------------------------------------------------------------------------------------------------------ judging
def output_err(k, x, ref):
    if k in ROW_VECTORS:
        return un.ray_err(x, ref)
    return un.tensor_err(x, ref, torch.full_like(ref, SCALAR_UNIT / un.FLOOR_REL))


def judge(mode, query, k, x, n, n_a=N_A):
    """(error, fp32 anchor error, bound) of output k of the query at n rows."""
    r64, r32 = reference(query, n, torch.float64, n_a)[k], reference(query, n, torch.float32, n_a)[k]
    x = x.reshape(r64.shape)
    e, a = output_err(k, x, r64), output_err(k, r32, r64)
    return e, a, max(un.ANCHOR_FACTOR * a, FLOORS[mode][k])


PAIRS = [(m, q) for m in MODES for q in OUTPUTS] + [(PER_LAYER, "sdf")]


@pytest.mark.parametrize("mode, query", PAIRS)
def test_query_forward_vs_fp64(mode, query):
    res = outputs(mode, query)
    fails, worst = [], {}
    for n in sizes_of(query):
        for k, x in res[("fp64", query, n)].items():
            e, a, bound = judge(mode, query, k, x, n)
            print(f"[query-fwd] {query} {mode} n={n} {k}: error {e:.3e} (fp32 {a:.3e}, bound {bound:.3e})")
            worst[k] = max(worst.get(k, (0.0, 0)), (e, n))
            if not e <= bound:
                fails.append((n, k, e, a, bound))
    for k, (e, n) in worst.items():
        print(f"[query-fwd] {query} {mode} worst {k} error {e:.3e} (n={n})")
    assert not fails, fails


@pytest.mark.parametrize("query", list(OUTPUTS))
def test_query_forward_bf16_is_close(query):
    """one plane: reported, and held to finite outputs at cosine >= COSINE_MIN to fp64."""
    res = outputs("bf16_tc", query)
    for n in sizes_of(query):
        for k, x in res[("fp64", query, n)].items():
            r64 = reference(query, n, torch.float64)[k]
            assert torch.isfinite(x).all(), (n, k)
            cos = un.cosine(x, r64)
            e = output_err(k, x.reshape(r64.shape), r64)
            print(f"[query-fwd] {query} bf16_tc n={n} {k}: error {e:.3e}, cosine {cos:.6f}")
            if n > 1 or k in ROW_VECTORS:      # the cosine of one scalar is its sign
                assert cos >= COSINE_MIN, (n, k, cos)


@pytest.mark.parametrize("mode, query", [(m, q) for m in [*MODES, *REPORTED] for q in OUTPUTS] + [(PER_LAYER, "sdf")])
def test_query_batch_invariance(mode, query):
    """the normal chain's GATE_FWD epilogue finishes a 32-row group that reaches past the chunk's last row on the generic
    path (epi_chunk16) and a full group on the specialised one: both must form the gate alike."""
    res = outputs(mode, query)
    names = [name for name, _, _ in invariance_batches()]
    alone = res[("inv", query, names[0])]
    diffs = []
    for name in names[1:]:
        for k, x in res[("inv", query, name)].items():
            if not torch.equal(x, alone[k]):
                bad = (x != alone[k]).reshape(x.shape[0], -1).any(-1)
                diffs.append((name, k, int(bad.sum()), float((x - alone[k]).abs().max())))
    for d in diffs:
        print(f"[query-fwd] {query} {mode} batch dependence: {d[0]} {d[1]}: {d[2]} rows differ, max |diff| {d[3]:.3e}")
    assert not diffs, diffs


def test_sampler_does_not_depend_on_the_chunking():
    """nrw_sample in bf16: 35 rays x 64 coarse samples = 2 x 1024 + 192 rows, so with chunks of 1024 rows the first SDF
    query ends in a 192-row chunk; the z_vals equal those of one 4096-row chunk.  Every ray runs from 3 units away
    through the unit sphere at a point inside the SDF's zero level set (VARIANT), so the importance rounds of every
    ray, the three in the short chunk included, follow the SDF across its surface."""
    from nrw.engine import make_sampler_cfg

    R, n_s = 35, 64
    g = torch.Generator().manual_seed(23)
    u = F.normalize(torch.randn(R, 3, generator=g, dtype=torch.float64), dim=-1)
    o = -3.0 * u
    d = F.normalize(0.2 * (2.0 * torch.rand(R, 3, generator=g, dtype=torch.float64) - 1.0) - o, dim=-1)
    b = (o * d).sum(-1, keepdim=True)
    disc = (b * b - (o * o).sum(-1, keepdim=True) + 1.0).sqrt()
    o, d, near, far = (t.float().contiguous().cuda() for t in (o, d, -b - disc, -b + disc))
    scfg = make_sampler_cfg(n_s, 64, 4, 0, 3, 0, False)
    z = []
    for chunk in (CHUNK, 4096):
        _, neuconw, _, eng = qb.make_modules("bf16", 0, chunk_rows=chunk, variant=VARIANT)
        with torch.no_grad():
            z.append(eng.sample(scfg, o, d, near, far)[0].cpu())
            sdf = neuconw.sdf((o[:, None, :] + d[:, None, :] * z[-1].cuda()[..., None]).reshape(-1, 3)).reshape(R, -1)
        assert eng.bound[3] == chunk and (R * n_s) % CHUNK < 256 < R * n_s
        assert ((sdf[:, :-1] * sdf[:, 1:]) < 0).any(-1).all(), "a ray misses the surface"
    bad = (z[0] != z[1]).any(-1)
    assert torch.equal(z[0], z[1]), (f"{int(bad.sum())} of {R} rays differ, max |dz| {float((z[0] - z[1]).abs().max()):.3e}")


# ------------------------------------------------------------------------------------------------------ code width
@pytest.mark.parametrize("n_a", [1, 47, 96])
@pytest.mark.parametrize("mode", ["bf16x6_simt", "bf16x3_tc"])
@pytest.mark.parametrize("query", ["forward", "nerf"])
def test_code_width_forward_vs_fp64(query, mode, n_a):
    mods = modules(*MODES[mode], n_a=n_a)
    n = 2 * CHUNK + 200
    res = run_query(mods, query, edge_inputs(n, n_a=n_a))
    fails = []
    for k, x in res.items():
        e, a, bound = judge(mode, query, k, x, n, n_a)
        print(f"[query-fwd] {query} {mode} n_a={n_a} {k}: error {e:.3e} (fp32 {a:.3e}, bound {bound:.3e})")
        if not e <= bound:
            fails.append((k, e, a, bound))
    assert not fails, fails


@pytest.mark.parametrize("mode", ["bf16x6_simt", "bf16x3_tc"])
@pytest.mark.parametrize("query", ["forward", "nerf"])
def test_code_width_backward_vs_fp64(query, mode):
    """n_a = 47: every gradient, the code's and static_linear_0's weights among them (test_gpu_query_backward's rule)."""
    qb.check_backward(query, mode, qb.reference_case(query, n_a=47), n_a=47)
