"""GPU: the standalone network queries are differentiable (nrw_neuconw_backward / nrw_nerf_backward through
nrw/engine.py's _NeuconWQueryFn / _NeRFQueryFn).

Against fp64 autograd of the port (oracle/neuconw_port.py sdf_forward, color_forward, nerf_forward; the normal as the
autograd gradient of the SDF with create_graph, so the points stay differentiable through it) for NeuconW.sdf,
NeuconW.gradient, NeuconW.forward, NeRF.forward and the indoor NeRF without the appearance head, with the upstream
gradient on one output at a time and then on all of them.  Rows whose colour-net or NeRF ReLU pre-activation lies near a
kink get zero upstream in the streams that cross that ReLU (util_network_bwd's margins).

Tolerance: util_network_bwd's rule.  A parameter tensor passes at max(4 x the error of the fp32 evaluation of the
reference, the mode's floor of test_gpu_network_bwd.py); an input gradient (points, view directions, codes) is judged per
row, with a floor per mode measured on an H100 (700 W) over the queries and stream sets below:
  bf16x6 on the CUDA cores  input floor 1e-4 (measured 3.4e-5, the points of NeuConW.forward under the normals)
  bf16x3 on the tensor cores input floor 5e-4 (measured 2.4e-4, the points of NeuconW.gradient)
  mixed on the tensor cores  input floor 5e-2 (measured 3.1e-2, the NeRF's 4-D points under rgb), view directions of
                             the colour net 3e-1 (measured 1.5e-1 in the worst of 300 rows): their gradient sums 27 plain
                             bf16 view-encoding columns weighted by frequencies up to 8, and rows where those cancel keep
                             the absolute error of the large terms
Gradients that the reference gives as exact zeros (parameters the query does not read) must come out as 0.0."""
import pytest
import torch
import torch.nn.functional as F

import util_indoor as ui
import util_network_bwd as un
from util_nrw import COLOR_CONFIG, SDF_CONFIG, build_system, cuda_train_step, port, rel_err, synth

pytestmark = pytest.mark.gpu
N_A = un.N_A
N = 300            # rows of the comparisons: less than one chunk, a ragged last 128-row tile
# mode: (precision, GEMM backend, parameter floor, input floor)
MODES = {
    "bf16x6_simt": ("bf16x6", 1, 2e-5, 1e-4),
    "bf16x3_tc": ("bf16x3", 0, 2e-4, 5e-4),
    "mixed_tc": ("mixed", 0, 3e-2, 5e-2),
}
MIXED_DIRS_FLOOR = 3e-1     # the colour net's view directions in 'mixed' (docstring)
# query: (network, outputs, inputs)
QUERIES = {
    "sdf": ("neuconw", ("sdf",), ("pts",)),
    "gradient": ("neuconw", ("normals",), ("pts",)),
    "forward": ("neuconw", ("rgb", "sdf", "normals"), ("pts", "dirs", "a")),
    "nerf": ("nerf", ("density", "rgb"), ("pts4", "dirs", "a")),
    "nerf_indoor": ("nerf", ("density", "rgb"), ("pts4", "dirs")),
}
ATOMIC = 2e-4      # fp32 atomics reorder only


def stream_sets(query):
    outs = QUERIES[query][1]
    return [(k,) for k in outs] + ([outs] if len(outs) > 1 else [])


def make_inputs(n, seed=3, n_a=N_A):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 0.8
    dirs = F.normalize(torch.randn(n, 3, generator=g), dim=-1)
    a = torch.randn(n, n_a, generator=g)
    p = F.normalize(torch.randn(n, 3, generator=g), dim=-1) * (1.0 + 3.0 * torch.rand(n, 1, generator=g))
    r = p.norm(dim=-1, keepdim=True)
    return dict(pts=pts, dirs=dirs, a=a, pts4=torch.cat([p / r, 1.0 / r], -1))


def params(indoor=False, n_a=N_A, variant=None):
    P = un.make_params(variant, n_a)
    return {k: v for k, v in P.items() if not k.startswith(ui.APP)} if indoor else P


def make_modules(precision, backend, indoor=False, chunk_rows=None, n_a=N_A, variant=None):
    """NeuconW and NeRF carrying the synthetic parameters, with their Engine (held by the caller: modules keep a weak
    reference)."""
    import nrw
    from nrw.engine import Engine

    P = params(indoor, n_a, variant)
    neuconw = nrw.NeuconW(SDF_CONFIG, COLOR_CONFIG, dict(init_val=0.3), in_channels_a=n_a, encode_a=True)
    nerf = nrw.NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4],
                    encode_appearance=not indoor, in_channels_a=n_a, in_channels_dir=27, use_viewdirs=True)
    neuconw.load_state_dict({k[len("neuconw."):]: v for k, v in P.items() if k.startswith("neuconw.")})
    nerf.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")})
    neuconw, nerf = neuconw.cuda(), nerf.cuda()
    eng = Engine(neuconw, nerf, n_vocab=un.N_VOCAB, n_a=n_a, precision=precision, backend=backend, chunk_rows=chunk_rows)
    return P, neuconw, nerf, eng


# ------------------------------------------------------------------------------------------------------ reference
def ref_outputs(query, Q, x):
    """the query's outputs as differentiable functions of the parameters Q and the inputs x (dicts of leaves)."""
    if QUERIES[query][0] == "nerf":
        fwd = ui.nerf_forward_noapp if query == "nerf_indoor" else port.nerf_forward
        dens, rgb = fwd(Q, x["pts4"], x["dirs"], x.get("a"))
        return dict(density=dens, rgb=rgb)
    h = port.sdf_forward(Q, x["pts"])
    (nrm,) = torch.autograd.grad(h[:, 0].sum(), x["pts"], create_graph=True)
    out = dict(sdf=h[:, 0], normals=nrm)
    if query == "forward":
        out["rgb"] = port.color_forward(Q, x["pts"], nrm, x["dirs"], h[:, 1:], x["a"])
    return out


def kink_rows(query, P, inp):
    """rows within util_network_bwd's margin of a ReLU kink of the colour net or the NeRF (fp64)."""
    Q = {k: v.double() for k, v in un.net_params(P).items()}
    x = {k: v.double() for k, v in inp.items()}
    with torch.no_grad():
        if query == "forward":
            pts = x["pts"].clone().requires_grad_(True)
            with torch.enable_grad():
                h = port.sdf_forward(Q, pts)
                (nrm,) = torch.autograd.grad(h[:, 0].sum(), pts)
            pres = un._color_preacts(Q, x["pts"], nrm, x["dirs"], h[:, 1:].detach(), x["a"])
            return un._near_kink(pres, un.kink_deltas(pres, False))
        if query == "nerf":
            pres = un._nerf_preacts(Q, x["pts4"], x["dirs"], x["a"])
            return un._near_kink(pres, un.kink_deltas(pres, True))
        if query == "nerf_indoor":     # the eight point layers, then views_linears.0
            pe = port.posenc(x["pts4"], 10)
            h, pres = pe, []
            for i in range(8):
                pres.append(F.linear(h, Q[f"nerf.pts_linears.{i}.weight"], Q[f"nerf.pts_linears.{i}.bias"]))
                h = F.relu(pres[-1])
                if i == 4:
                    h = torch.cat([pe, h], -1)
            feat = F.linear(h, Q["nerf.feature_linear.weight"], Q["nerf.feature_linear.bias"])
            pres.append(F.linear(torch.cat([feat, port.posenc(x["dirs"], 4)], -1), Q["nerf.views_linears.0.weight"],
                                 Q["nerf.views_linears.0.bias"]))
            return un._near_kink(pres, un.kink_deltas(pres, True))
    return torch.zeros(inp["pts"].shape[0], dtype=torch.bool)


def make_ups(query, P, inp, seed=9):
    g = torch.Generator().manual_seed(seed)
    n = inp["pts"].shape[0]
    keep = (~kink_rows(query, P, inp)).float()[:, None]
    shapes = dict(sdf=(n,), normals=(n, 3), rgb=(n, 3), density=(n, 1))
    ups = {k: torch.randn(shapes[k], generator=g) for k in QUERIES[query][1]}
    for k in ("rgb", "density"):
        if k in ups and (k == "rgb" or QUERIES[query][0] == "nerf"):
            ups[k] = ups[k] * keep
    return ups


def reference(query, P, inp, ups, dtype):
    """{stream set: {name: gradient}} over the network's parameters and the query's inputs."""
    net = QUERIES[query][0]
    Q = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in un.net_params(P).items()
         if k.startswith(net + ".")}
    x = {k: inp[k].to(dtype).clone().requires_grad_(True) for k in ("pts", "dirs", "a", "pts4")}
    out = ref_outputs(query, Q, x)
    names = list(Q) + list(QUERIES[query][2])
    leaves = list(Q.values()) + [x[k] for k in QUERIES[query][2]]
    res = {}
    for st in stream_sets(query):
        loss = sum((out[k] * ups[k].to(dtype).reshape(out[k].shape)).sum() for k in st)
        gs = torch.autograd.grad(loss, leaves, retain_graph=True, allow_unused=True)
        res[st] = {nm: (torch.zeros_like(t) if gv is None else gv).detach() for nm, t, gv in zip(names, leaves, gs)}
    return res


# ------------------------------------------------------------------------------------------------------ CUDA
def run_query(query, neuconw, nerf, inp, need=None):
    """the query on the modules with fresh leaf inputs requiring grad (those in `need`, default the query's inputs)."""
    need = QUERIES[query][2] if need is None else need
    x = {k: v.cuda().clone().requires_grad_(k in need) for k, v in inp.items()}
    if query == "sdf":
        return x, dict(sdf=neuconw.sdf(x["pts"]).reshape(-1))
    if query == "gradient":
        return x, dict(normals=neuconw.gradient(x["pts"]))
    if query == "forward":
        n = x["pts"].shape[0]
        rgb, _, sdf, nrm = neuconw(torch.cat([x["pts"], x["dirs"], x["a"]], -1).view(1, n, -1))
        return x, dict(rgb=rgb.reshape(n, 3), sdf=sdf.reshape(n), normals=nrm.reshape(n, 3))
    dens, rgb = nerf(x["pts4"], x["dirs"], x["a"])
    return x, dict(density=dens, rgb=rgb)


def cuda_grads(query, neuconw, nerf, inp, ups, st):
    """{name: gradient} (CPU) of sum_{k in st} <ups_k, out_k> for the network's parameters and the query's inputs."""
    net = QUERIES[query][0]
    mod = neuconw if net == "neuconw" else nerf
    mod.zero_grad(set_to_none=True)
    x, out = run_query(query, neuconw, nerf, inp)
    loss = sum((out[k] * ups[k].cuda().reshape(out[k].shape)).sum() for k in st)
    loss.backward()
    res = {f"{net}.{k}": (torch.zeros_like(p) if p.grad is None else p.grad).detach().cpu()
           for k, p in mod.named_parameters()}
    for k in QUERIES[query][2]:
        res[k] = x[k].grad.detach().cpu()
    return res


def reference_case(query, n_a=N_A):
    """(P, inputs, upstream, fp64 gradients, fp32 gradients) of the comparison at N rows."""
    P = params(query == "nerf_indoor", n_a)
    inp = make_inputs(N, n_a=n_a)
    ups = make_ups(query, P, inp)
    return P, inp, ups, reference(query, P, inp, ups, torch.float64), reference(query, P, inp, ups, torch.float32)


@pytest.fixture(scope="module")
def refs():
    cache = {}

    def get(query):
        if query not in cache:
            cache[query] = reference_case(query)
        return cache[query]

    return get


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("query", list(QUERIES))
def test_query_backward_vs_fp64(query, mode, refs):
    check_backward(query, mode, refs(query))


def check_backward(query, mode, case, n_a=N_A):
    """every parameter and input gradient of the query in `mode` against case's fp64 gradients under the rule above."""
    P, inp, ups, g64, g32 = case
    prec, backend, pfloor, ifloor = MODES[mode]
    _, neuconw, nerf, eng = make_modules(prec, backend, indoor=query == "nerf_indoor", n_a=n_a)
    sets = stream_sets(query)
    full = g64[sets[-1]]
    fails, worst = [], {}
    for st in sets:
        got = cuda_grads(query, neuconw, nerf, inp, ups, st)
        tag = "+".join(st)
        for k, r64 in g64[st].items():
            x = got[k].reshape(r64.shape)
            assert torch.isfinite(x).all(), (tag, k)
            if not full[k].any():                      # not read by this query: exact zeros
                if x.any():
                    fails.append((tag, k, "expected exact zeros"))
                continue
            is_input = k in QUERIES[query][2]
            err = un.ray_err if is_input else un.tensor_err
            e = err(x, r64, scale=full[k]) if is_input else err(x, r64, full[k])
            a = err(g32[st][k], r64, scale=full[k]) if is_input else err(g32[st][k], r64, full[k])
            floor = ifloor if is_input else pfloor
            if mode == "mixed_tc" and query == "forward" and k == "dirs":
                floor = MIXED_DIRS_FLOOR
            bound = max(un.ANCHOR_FACTOR * a, floor)
            kind = "input" if is_input else "param"
            worst[kind] = max(worst.get(kind, (0.0, "")), (e, f"{tag}.{k}"))
            if not e <= bound:
                fails.append((tag, k, e, a, bound))
    for kind, (e, where) in sorted(worst.items()):
        print(f"[query-bwd] {query} {mode} n_a={n_a} worst {kind} error {e:.3e} ({where})")
    assert not fails, fails[:20]


# ------------------------------------------------------------------------------------------------------ contract
@pytest.fixture(scope="module")
def tc_modules():
    return make_modules("bf16x3", 0)


@pytest.mark.parametrize("query", ["sdf", "gradient", "forward", "nerf"])
def test_outputs_equal_the_inference_call(query, tc_modules):
    _, neuconw, nerf, _ = tc_modules
    inp = make_inputs(N, seed=4)
    x, out = run_query(query, neuconw, nerf, inp)
    assert all(v.grad_fn is not None for v in out.values())
    with torch.no_grad():
        _, ref = run_query(query, neuconw, nerf, inp, need=())
    for k in out:
        assert torch.equal(out[k].detach(), ref[k]), k


@pytest.mark.parametrize("query", ["sdf", "forward", "nerf"])
def test_no_input_requiring_grad_gives_inference_outputs(query, tc_modules):
    _, neuconw, nerf, _ = tc_modules
    assert torch.is_grad_enabled() and all(p.requires_grad for p in neuconw.parameters())
    _, out = run_query(query, neuconw, nerf, make_inputs(64), need=())
    assert all(v.grad_fn is None and not v.requires_grad for v in out.values())


def test_gradient_marks_its_input(tc_modules):
    _, neuconw, _, _ = tc_modules
    x = make_inputs(64)["pts"].cuda()
    nrm = neuconw.gradient(x)
    assert x.requires_grad and nrm.grad_fn is not None
    with torch.no_grad():
        assert neuconw.gradient(make_inputs(64)["pts"].cuda()).grad_fn is None


def test_code_gets_no_gradient_without_the_appearance_head():
    _, neuconw, nerf, eng = make_modules("bf16x3", 0, indoor=True)
    inp = make_inputs(64)
    x = {k: v.cuda().requires_grad_(True) for k, v in inp.items()}
    dens, rgb = nerf(x["pts4"], x["dirs"], x["a"])
    (dens.sum() + rgb.sum()).backward()
    assert x["a"].grad is None
    assert x["pts4"].grad is not None and x["dirs"].grad.abs().sum() > 0


@pytest.mark.parametrize("query", ["sdf", "gradient", "nerf"])
def test_differentiating_the_backward_raises(query, tc_modules):
    """create_graph=True through a query's backward raises (the gradient of its result would silently be zero)."""
    _, neuconw, nerf, _ = tc_modules
    x, out = run_query(query, neuconw, nerf, make_inputs(64))
    inp = x["pts4" if query == "nerf" else "pts"]
    loss = sum((v ** 2).sum() for v in out.values())
    with pytest.raises(RuntimeError, match="once-differentiable"):
        torch.autograd.grad(loss, inp, create_graph=True)


def test_retain_graph_gives_equal_gradients(tc_modules):
    _, neuconw, _, _ = tc_modules
    x = make_inputs(N)["pts"].cuda().requires_grad_(True)
    nrm = neuconw.gradient(x)
    loss = ((nrm.norm(dim=-1) - 1) ** 2).mean()
    params = [p for p in neuconw.parameters() if p.requires_grad]
    g1 = torch.autograd.grad(loss, [x] + params, retain_graph=True, allow_unused=True)
    g2 = torch.autograd.grad(loss, [x] + params, allow_unused=True)
    for a, b in zip(g1, g2):
        if a is not None:
            assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < ATOMIC


@pytest.mark.parametrize("query", ["gradient", "forward", "nerf"])
def test_chunked_query_matches_one_chunk(query):
    """n = 2500 rows over chunks of 1024 (two whole chunks and a ragged 452-row tail) against one chunk."""
    inp = make_inputs(2500, seed=6)
    P = params()
    ups = make_ups(query, P, inp)
    res = []
    for chunk in (1024, None):
        _, neuconw, nerf, eng = make_modules("bf16x3", 0, chunk_rows=chunk)
        got = cuda_grads(query, neuconw, nerf, inp, ups, QUERIES[query][1])
        assert eng.bound[3] == 1024 if chunk else eng.bound[3] >= 2500
        res.append(got)
    for k in res[0]:
        if k in QUERIES[query][2]:
            e = un.ray_err(res[0][k], res[1][k], scale=res[1][k])
        else:
            e = rel_err(res[0][k].numpy(), res[1][k].numpy())
        assert e < ATOMIC, (k, e)


# ------------------------------------------------------------------------------------------------------ interleaving
CFG = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)


def _system():
    P = synth.make_params(seed=0)
    return build_system(P, CFG, precision="bf16x3", backend=0, chunk_rows=2048)


def _eikonal_grads(s, x):
    s["neuconw"].zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    loss = ((s["neuconw"].gradient(x).norm(dim=-1) - 1) ** 2).mean()
    return x, loss


def _flat_grads(mod):
    return torch.cat([p.grad.reshape(-1) for p in mod.parameters() if p.grad is not None]).cpu()


def test_query_between_a_render_and_its_backward():
    """render forward, then a query with its backward, then the render's backward: the render's gradient equals a run
    without the query."""
    s = _system()
    r = s["renderer"]
    b = {k: v.cuda() for k, v in synth.make_rays(300, CFG, seed=1).items()}
    bg = torch.zeros(1, 3, device="cuda")
    x0 = make_inputs(2048, seed=8)["pts"].cuda()

    def render_grads(query):
        for m in (s["neuconw"], s["nerf"], s["emb"]):
            m.zero_grad(set_to_none=True)
        res = r.render(b["rays"], b["ts"], b["label"], perturb_overwrite=0, background_rgb=bg, cos_anneal_ratio=0.5)
        if query:
            x, loss = _eikonal_grads(s, x0)
            torch.autograd.grad(loss, [x] + list(s["neuconw"].parameters()), allow_unused=True)
        (res["color"].sum() + res["gradient_error"].sum()).backward()
        return r.engine.last_flat_grad.clone(), s["emb"].weight.grad.clone()

    g_ref, e_ref = render_grads(False)
    g_q, e_q = render_grads(True)
    assert rel_err(g_q.cpu().numpy(), g_ref.cpu().numpy()) < ATOMIC
    assert rel_err(e_q.cpu().numpy(), e_ref.cpu().numpy()) < ATOMIC


def test_training_step_between_a_query_and_its_backward():
    """query forward, a training step, then the query's backward: the query's gradients are those of an uninterrupted
    query; and the query's backward after the step leaves the bound workspace as it was."""
    s = _system()
    batch = synth.make_rays(256, CFG, seed=3)
    x0 = make_inputs(4096, seed=9)["pts"].cuda()
    cuda_train_step(s, CFG, batch)
    eng = s["renderer"].engine
    x, loss = _eikonal_grads(s, x0)
    loss.backward()
    ref_x, ref_p = x.grad.cpu(), _flat_grads(s["neuconw"])
    slots, bound, ws_bytes = eng.slots, eng.bound, eng.workspace.numel()
    x, loss = _eikonal_grads(s, x0)
    cuda_train_step(s, CFG, batch)
    s["neuconw"].zero_grad(set_to_none=True)
    loss.backward()
    assert eng.bound == bound and eng.slots == slots and eng.workspace.numel() == ws_bytes
    assert un.ray_err(x.grad.cpu(), ref_x, scale=ref_x) < ATOMIC
    assert rel_err(_flat_grads(s["neuconw"]).numpy(), ref_p.numpy()) < ATOMIC


# ------------------------------------------------------------------------------------------------------ drop-in
def test_eikonal_loss_matches_the_reference_neuconw():
    """((neuconw.gradient(x).norm(dim=-1) - 1)**2).mean() on the reference's own NeuconW with the same weights gives the
    same parameter gradients within the bf16x3 floor."""
    from oracle import ref_import

    if not ref_import.available():
        pytest.skip("no reference copy (oracle/_ref) on this box")
    ref = ref_import.load()
    P = params()
    m = ref.NeuconW(sdfNet_config=SDF_CONFIG, colorNet_config=COLOR_CONFIG, SNet_config=dict(init_val=0.3),
                    in_channels_a=N_A, encode_a=True).double()
    m.load_state_dict({k[len("neuconw."):]: v.double() for k, v in P.items() if k.startswith("neuconw.")})
    x = make_inputs(N, seed=10)["pts"]
    ((m.gradient(x.double()).norm(dim=-1) - 1) ** 2).mean().backward()
    want = {"neuconw." + k: p.grad for k, p in m.named_parameters() if p.grad is not None and p.grad.any()}
    _, neuconw, _, eng = make_modules("bf16x3", 0)
    xc = x.cuda()
    ((neuconw.gradient(xc).norm(dim=-1) - 1) ** 2).mean().backward()
    got = {"neuconw." + k: p.grad.cpu() for k, p in neuconw.named_parameters()}
    assert want
    for k, r in want.items():
        e = un.tensor_err(got[k], r, r)
        print(f"[query-bwd] drop-in eikonal {k}: {e:.3e}")
        assert e <= MODES["bf16x3_tc"][2], (k, e)
