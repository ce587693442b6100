"""Stage-level harness for the network half of the backward (csrc/engine.cu network_backward, nrw_network_backward).

The five per-sample upstream gradients of the compositing stage (d_sdf, d_normals, d_rgb, d_bg_alpha, d_bg_rgb) are
INJECTED, so neither the sampler's discontinuities nor the compositor's cancellations enter a comparison: z_vals are
inputs, and the port's networks (oracle/neuconw_port.py: sdf_forward, sdf_gradient, color_forward,
render_core_outside), evaluated in fp64, are an exact reference of the same operation.

  make_case       seeded rays, z_vals, z_out, sample_dist, a_emb and a parameter variant; rows that lie near a ReLU
                  kink get zero upstream gradient in the streams that cross that ReLU (kink_masks)
  reference       forward outputs and autograd gradients of L = sum <upstream, output> for every parameter by name and
                  for a_emb, per stream set (each stream alone, then all together)
  cuda_network    nrw_render_forward, then nrw_network_backward once per stream set
  tensor_err      the tolerance rule below

Tolerance rule, per parameter tensor:  err = max|x - ref64| / (max|ref64| + 1e-3 max|full64|), where full64 is the
same tensor under all five streams.  grad_a_emb and the forward outputs use the same rule per ray (util_composite's
ray_err).  A tensor passes at max(4 x the error of the fp32 evaluation of the reference, floor).  Parameters listed by
structural_zeros must come out as exact zeros and are not judged by the rule."""
import ctypes as C
import os
from contextlib import contextmanager

import numpy as np
import torch
import torch.nn.functional as F

from util_composite import ANCHOR_FACTOR, FLOOR_REL, judge, ray_err  # noqa: F401  (re-exported for the tests)
from util_nrw import COLOR_CONFIG, SDF_CONFIG, port, synth

STREAMS = ("sdf", "normals", "rgb", "bg_alpha", "bg_rgb")
BG_STREAMS = ("bg_alpha", "bg_rgb")
FWD_KEYS = ("sv_sdf", "gradients", "sv_rgb", "sv_bg_alpha", "sv_bg_rgb")
N_A = 48
N_VOCAB = 5000
# Rows whose ReLU pre-activation lies within KINK_DELTA x rms(layer) of zero get zero upstream gradient in the streams
# that cross that ReLU: with zero upstream such a row contributes exactly nothing on either side, so a forward that
# lands on the other side of a kink cannot show up as a gradient error.  Each margin is >= 10x the largest relative
# pre-activation error of an fp32 evaluation (test_network_bwd_cpu.py).  The kernels' own pre-activations are not read
# back; what stands in for them is that both bf16x6 modes produce the ReLU nets' outputs (sv_rgb, sv_bg_alpha,
# sv_bg_rgb) within 2x the fp32 reference's error on an H100.  The NeRF's eight point layers take a 2^9-frequency
# encoding of the point, so fp32 rounding of the point alone moves their pre-activations by up to ~9e-5 rms: they get
# KINK_DELTA_PTS (the colour net and the appearance layers: ~3e-6).
KINK_DELTA = 1e-4
KINK_DELTA_PTS = 1e-3
# NeRF density threshold of torch's softplus (and of pointwise.cu head_kernel / head_bwd mode 2)
SOFTPLUS_THRESHOLD = 20.0

# name: (R, S, n_outside, chunk_rows, recompute, variant, geometry seed)
#   one_ray    one chunk of 28 rows, less than one 128-row tile, no background
#   ragged     SDF chunks of 1008 + 28 rows, NeRF chunks of 1024 + 160 rows; every chunk keeps its own slot
#   c2_counts  the C2 sample count (64 + 64) with 4 outside, T = 132
#   recompute  ragged with one slot per network (NRW_RECOMPUTE=1): chunk 0 is recomputed inside the backward
#   dense_bg   nerf.alpha_linear.bias shifted so that densities fall on both sides of the softplus threshold
CASES = {
    "one_ray": (1, 28, 0, None, False, None, 11),
    "ragged": (37, 28, 4, 1024, False, None, 12),
    "c2_counts": (24, 128, 4, None, False, None, 13),
    "recompute": (37, 28, 4, 1024, True, None, 12),
    "dense_bg": (24, 28, 4, None, False, "dense_bg", 14),
}
DENSE_BG_SHIFT = 20.03    # added to nerf.alpha_linear.bias: about half the densities exceed 20 (test_network_bwd_cpu.py)
# subtracted from the SDF's bias: the synthetic SDF is >= 0.065 in [-1.2, 1.2]^3, and 0.3 below it has a zero level set
# at |x| ~ 0.5 .. 0.7
SURFACE_SHIFT = 0.3


def geometry(name):
    """(R, S, n_outside, variant, seed): what the inputs and hence the reference depend on."""
    R, S, n_o, _, _, variant, seed = CASES[name]
    return R, S, n_o, variant, seed


def streams_of(case):
    return STREAMS if case["n_outside"] > 0 else STREAMS[:3]


def stream_sets(case):
    """each stream alone, then all of them together (the last entry: `full`)."""
    st = streams_of(case)
    return [(k,) for k in st] + [st]


# --------------------------------------------------------------------------------------------------- parameters
def make_params(variant=None, n_a=N_A):
    P = synth.make_params(seed=0, n_vocab=N_VOCAB, n_a=n_a)
    if variant == "dense_bg":
        P["nerf.alpha_linear.bias"] = P["nerf.alpha_linear.bias"] + DENSE_BG_SHIFT
    elif variant == "surface":
        P["neuconw.sdf_net.lin8.bias"] = P["neuconw.sdf_net.lin8.bias"] - SURFACE_SHIFT * (torch.arange(513) == 0)
    else:
        assert variant is None, variant
    return P


def net_params(P):
    """the parameters the networks read (embedding_a.weight reaches them as the a_emb input)."""
    return {k: v for k, v in P.items() if not k.startswith("embedding_a.")}


# --------------------------------------------------------------------------------------------------- cases
def make_case(R, S, n_outside, variant, seed):
    """Rays from ~3 units away through the unit sphere; z_vals sorted uniform draws between the sphere's near and far
    hits (the SDF net's surface |x| ~ 0.5 lies in between), z_out behind far as the sampler spaces them, per-ray
    sample_dist and appearance codes."""
    g = torch.Generator().manual_seed(int(seed))
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    theta, phi = rnd(R) * 2 * np.pi, rnd(R) * np.pi * 0.8 + 0.1 * np.pi
    dirn = torch.stack([torch.sin(phi) * torch.cos(theta), torch.sin(phi) * torch.sin(theta), torch.cos(phi)], -1)
    o = -3.0 * dirn
    target = 0.4 * (2.0 * rnd(R, 3) - 1.0)
    d = target - o
    d = d / d.norm(dim=-1, keepdim=True)
    # unit-sphere hits of o + t d
    b = (o * d).sum(-1)
    disc = (b * b - (o * o).sum(-1) + 1.0).clamp_min(1e-3).sqrt()
    near, far = -b - disc, -b + disc
    z = near[:, None] + (far - near)[:, None] * torch.sort(rnd(R, S), -1)[0]
    sample_dist = ((far - near) / S)[:, None]
    if n_outside > 0:
        lin = torch.linspace(1e-3, 1.0 - 1.0 / (n_outside + 1.0), n_outside, dtype=torch.float64)
        mids = 0.5 * (lin[1:] + lin[:-1])
        upper, lower = torch.cat([mids, lin[-1:]]), torch.cat([lin[:1], mids])
        zo = lower[None, :] + (upper - lower)[None, :] * rnd(R, n_outside)
        z_out = far[:, None] / torch.flip(zo, dims=[-1]) + 1.0 / S
    else:
        z_out = torch.zeros(R, 0, dtype=torch.float64)
    a_emb = torch.randn(R, N_A, generator=g)
    f = lambda t: t.float().contiguous()
    case = dict(R=R, S=S, n_outside=n_outside, T=S + n_outside, variant=variant, seed=seed, o=f(o), d=f(d),
                z_vals=f(z), z_out=f(z_out), sample_dist=f(sample_dist), a_emb=a_emb.contiguous())
    case["P"] = make_params(variant)
    case["mask_rgb"], case["mask_bg"] = kink_masks(case)
    case["ups"] = make_ups(case)
    return case


def make_named_case(name):
    return make_case(*geometry(name))


def z_feed(case):
    """the merged NeRF sample positions, as the reference renderer forms them."""
    return torch.sort(torch.cat([case["z_vals"], case["z_out"]], -1), dim=-1)[0]


def _points(o, d, z, sample_dist):
    """render_core's mid points: flat pts [R*S,3], dirs [R*S,3]."""
    R, S = z.shape
    dists = torch.cat([z[..., 1:] - z[..., :-1], sample_dist.expand(R, 1)], -1)
    mid = z + dists * 0.5
    pts = (o[:, None, :] + d[:, None, :] * mid[..., :, None]).reshape(-1, 3)
    return pts, d[:, None, :].expand(R, S, 3).reshape(-1, 3)


def _color_preacts(Q, pts, nrm, dirs, feat, a, pre="neuconw.color_net."):
    """pre-activations of the colour net's six ReLUs (color_forward's layers in order)."""
    xf = F.linear(feat, Q[pre + "xyz_encoding_final.weight"], Q[pre + "xyz_encoding_final.bias"])
    h = torch.cat([xf, port.posenc(dirs, 4), a], 1)
    out = []
    for s in range(2):
        q = f"{pre}static_encoding.static_linear_{s}."
        out.append(F.linear(h, Q[q + "weight"], Q[q + "bias"]))
        h = F.relu(out[-1])
    x = torch.cat([pts, nrm, h], -1)
    for l in range(4):
        out.append(F.linear(x, port.wn_weight(Q, f"{pre}lin{l}."), Q[f"{pre}lin{l}.bias"]))
        x = F.relu(out[-1])
    return out


def _nerf_preacts(Q, pts4, dirs, a, pre="nerf."):
    """pre-activations of the NeRF's eight point-layer and four appearance-layer ReLUs (nerf_forward's order)."""
    pe = port.posenc(pts4, 10)
    h, out = pe, []
    for i in range(8):
        out.append(F.linear(h, Q[f"{pre}pts_linears.{i}.weight"], Q[f"{pre}pts_linears.{i}.bias"]))
        h = F.relu(out[-1])
        if i == 4:
            h = torch.cat([pe, h], -1)
    feat = F.linear(h, Q[pre + "feature_linear.weight"], Q[pre + "feature_linear.bias"])
    h = torch.cat([feat, port.posenc(dirs, 4), a], -1)
    for s in range(4):
        q = f"{pre}apperence_encoding.static_linear_{s}."
        out.append(F.linear(h, Q[q + "weight"], Q[q + "bias"]))
        h = F.relu(out[-1])
    return out


def _nerf_inputs(o, d, zf, sample_dist, a_emb):
    """render_core_outside's pts4, dirs and per-row appearance codes, plus its dists."""
    R, T = zf.shape
    dists = torch.cat([zf[..., 1:] - zf[..., :-1], sample_dist.expand(R, 1)], -1)
    mid = zf + dists * 0.5
    pts = o[:, None, :] + d[:, None, :] * mid[..., :, None]
    r = torch.linalg.norm(pts, ord=2, dim=-1, keepdim=True).clip(1.0, 1e10)
    pts4 = torch.cat([pts / r, 1.0 / r], -1).reshape(-1, 4)
    dirs = d[:, None, :].expand(R, T, 3).reshape(-1, 3)
    a = a_emb[:, None, :].expand(R, T, a_emb.shape[-1]).reshape(R * T, -1)
    return pts4, dirs, a, dists


def preacts(case, dtype=torch.float64):
    """(colour-net ReLU pre-activations [R*S, n] per layer, NeRF ReLU pre-activations [R*T, n] per layer)."""
    Q = {k: v.to(dtype) for k, v in net_params(case["P"]).items()}
    cv = lambda t: t.to(dtype)
    o, d, z, sd, a_emb = cv(case["o"]), cv(case["d"]), cv(case["z_vals"]), cv(case["sample_dist"]), cv(case["a_emb"])
    R, S = z.shape
    pts, dirs = _points(o, d, z, sd)
    with torch.no_grad():
        feat = port.sdf_forward(Q, pts)[:, 1:]
    nrm = port.sdf_gradient(Q, pts, create_graph=False).detach()
    a = a_emb[:, None, :].expand(R, S, N_A).reshape(R * S, -1)
    with torch.no_grad():
        pc = _color_preacts(Q, pts, nrm, dirs, feat, a)
        pn = []
        if case["n_outside"] > 0:
            pts4, ndirs, na, _ = _nerf_inputs(o, d, cv(z_feed(case)), sd, a_emb)
            pn = _nerf_preacts(Q, pts4, ndirs, na)
    return pc, pn


def kink_deltas(pres, nerf):
    """the margin of each layer in preacts' order."""
    return [KINK_DELTA_PTS if nerf and i < 8 else KINK_DELTA for i in range(len(pres))]


def _near_kink(pres, deltas):
    bad = torch.zeros(pres[0].shape[0], dtype=torch.bool)
    for z, delta in zip(pres, deltas):
        bad |= (z.abs() < delta * z.pow(2).mean().sqrt()).any(-1)
    return bad


def kink_masks(case):
    """(colour rows [R,S], NeRF rows [R,T]) within the layer's margin x rms(layer) of a ReLU kink in some layer (fp64)."""
    pc, pn = preacts(case)
    R, S, T = case["R"], case["S"], case["T"]
    mc = _near_kink(pc, kink_deltas(pc, False)).reshape(R, S)
    mn = _near_kink(pn, kink_deltas(pn, True)).reshape(R, T) if pn else torch.zeros(R, T, dtype=torch.bool)
    return mc, mn


def density(case, dtype=torch.float64):
    """the NeRF's pre-softplus density per row [R,T]."""
    Q = {k: v.to(dtype) for k, v in net_params(case["P"]).items()}
    cv = lambda t: t.to(dtype)
    pts4, dirs, a, _ = _nerf_inputs(cv(case["o"]), cv(case["d"]), cv(z_feed(case)), cv(case["sample_dist"]),
                                    cv(case["a_emb"]))
    with torch.no_grad():
        return port.nerf_forward(Q, pts4, dirs, a)[0].reshape(case["R"], case["T"])


def make_ups(case):
    """one seeded upstream gradient per stream (fp32), zero on the kink-masked rows of the streams crossing a ReLU."""
    g = torch.Generator().manual_seed(int(case["seed"]) + 7)
    R, S, T = case["R"], case["S"], case["T"]
    ups = dict(sdf=torch.randn(R, S, generator=g), normals=torch.randn(R, S, 3, generator=g),
               rgb=torch.randn(R, S, 3, generator=g) * (~case["mask_rgb"]).float()[..., None])
    if case["n_outside"] > 0:
        keep = (~case["mask_bg"]).float()
        ups["bg_alpha"] = torch.randn(R, T, generator=g) * keep
        ups["bg_rgb"] = torch.randn(R, T, 3, generator=g) * keep[..., None]
    return ups


# --------------------------------------------------------------------------------------------------- reference
def forward_graph(case, dtype, Q=None, a_emb=None):
    """the five network outputs in `dtype` as differentiable functions of Q (name -> leaf) and a_emb [R,n_a]."""
    cv = lambda t: t.to(dtype)
    o, d, z, sd = cv(case["o"]), cv(case["d"]), cv(case["z_vals"]), cv(case["sample_dist"])
    R, S = z.shape
    pts, dirs = _points(o, d, z, sd)
    a = a_emb[:, None, :].expand(R, S, N_A).reshape(R * S, -1)
    out = port.sdf_forward(Q, pts)
    nrm = port.sdf_gradient(Q, pts, create_graph=True)
    rgb = port.color_forward(Q, pts, nrm, dirs, out[:, 1:], a)
    res = dict(sdf=out[:, 0].reshape(R, S), normals=nrm.reshape(R, S, 3), rgb=rgb.reshape(R, S, 3))
    if case["n_outside"] > 0:
        res["bg_alpha"], res["bg_rgb"] = port.render_core_outside(Q, o, d, cv(z_feed(case)), sd, a_emb)
    return res


def leaves(case, dtype):
    Q = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in net_params(case["P"]).items()}
    a = case["a_emb"].detach().to(dtype).clone().requires_grad_(True)
    return Q, a


def reference(case, dtype, sets=None):
    """(forward dict keyed by FWD_KEYS, [gradient dict per stream set]); a gradient dict maps every parameter name and
    "a_emb" to the autograd gradient of sum_{k in set} <ups_k, out_k> (zeros where the output does not depend on it)."""
    sets = stream_sets(case) if sets is None else sets
    Q, a = leaves(case, dtype)
    out = forward_graph(case, dtype, Q, a)
    fwd = dict(sv_sdf=out["sdf"], gradients=out["normals"], sv_rgb=out["rgb"])
    if case["n_outside"] > 0:
        fwd.update(sv_bg_alpha=out["bg_alpha"], sv_bg_rgb=out["bg_rgb"])
    fwd = {k: v.detach() for k, v in fwd.items()}
    names = list(Q) + ["a_emb"]
    tensors = list(Q.values()) + [a]
    grads = []
    for st in sets:
        loss = sum((out[k] * case["ups"][k].to(dtype)).sum() for k in st)
        gs = torch.autograd.grad(loss, tensors, retain_graph=True, allow_unused=True)
        grads.append({n: (torch.zeros_like(t) if gv is None else gv).detach() for n, t, gv in zip(names, tensors, gs)})
    return fwd, grads


def loss_value(case, sets, Q, a):
    """sum_{k in sets} <ups_k, out_k> in fp64 at parameters Q and codes a (no graph kept)."""
    with torch.no_grad():
        out = forward_graph(case, torch.float64, Q, a)
        return float(sum((out[k] * case["ups"][k].double()).sum() for k in sets))


# --------------------------------------------------------------------------------------------------- structural zeros
DEAD = ("neuconw.xyz_encoding_final.", "nerf.views_linears.", "neuconw.deviation_network.variance")
LIN8 = "neuconw.sdf_net.lin8."
NERF_RGB = ("nerf.feature_linear.", "nerf.apperence_encoding.", "nerf.rgb_linear.")


def structural_zeros(case, st):
    """{name: rows} of the gradients that are exactly zero under the stream set st: rows = None for the whole tensor,
    else a slice of its first dimension.  "a_emb" stands for the appearance-code gradient."""
    names = list(net_params(case["P"])) + ["a_emb"]
    st = set(st)
    zero = {}

    def add(prefixes, rows=None):
        for n in names:
            if n.startswith(prefixes) and zero.get(n, 0) is not None:
                zero[n] = rows

    add(DEAD)
    if case["n_outside"] == 0 or not st & set(BG_STREAMS):
        add(("nerf.",))
    if not st & {"sdf", "normals", "rgb"}:
        add(("neuconw.",))
    # lin8 row 0 is the SDF, rows 1.. the feature that reaches nothing but the colour net; the SDF's own bias moves
    # neither the normal nor the feature
    if "rgb" not in st:
        add(("neuconw.color_net.",))
        add((LIN8,), slice(1, None))
        if "sdf" not in st:
            add((LIN8 + "bias",))
    elif "sdf" not in st:
        add((LIN8 + "bias",), slice(0, 1))
    if "bg_rgb" not in st:
        add(NERF_RGB)
    if "bg_alpha" not in st:
        add(("nerf.alpha_linear.",))
    if "rgb" not in st and "bg_rgb" not in st:
        add(("a_emb",))
    return zero


def zero_part(t, rows):
    return t if rows is None else t[rows]


def nonzero_part(t, rows):
    """the entries of t that structural_zeros does not cover (empty when it covers all)."""
    if rows is None:
        return t.new_zeros(0)
    keep = torch.ones(t.shape[0], dtype=torch.bool)
    keep[rows] = False
    return t[keep]


# --------------------------------------------------------------------------------------------------- CUDA
@contextmanager
def _env(key, value):
    old = os.environ.get(key)
    os.environ[key] = value
    try:
        yield
    finally:
        if old is None:
            del os.environ[key]
        else:
            os.environ[key] = old


def make_engine(case, precision, backend, chunk_rows=None, recompute=False):
    """an Engine over modules carrying the case's parameters, bound for a backward of the case's shape."""
    import nrw
    from nrw.engine import Engine

    P = case["P"]
    neuconw = nrw.NeuconW(SDF_CONFIG, COLOR_CONFIG, dict(init_val=0.3), in_channels_a=N_A, encode_a=True)
    nerf = nrw.NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4],
                    encode_appearance=True, in_channels_a=N_A, in_channels_dir=27, use_viewdirs=True)
    neuconw.load_state_dict({k[len("neuconw."):]: v for k, v in P.items() if k.startswith("neuconw.")})
    nerf.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")})
    dev = torch.device("cuda")
    neuconw, nerf = neuconw.to(dev), nerf.to(dev)
    eng = Engine(neuconw, nerf, n_vocab=N_VOCAB, n_a=N_A, precision=precision, backend=backend, chunk_rows=chunk_rows)
    eng._modules = (neuconw, nerf)                        # the engine holds only weak references to its modules
    with _env("NRW_RECOMPUTE", "1" if recompute else "0"):
        eng.ensure(dev, case["R"], case["T"], 1, S=case["S"])
    eng.pack(dev)
    return eng


def render_io(case):
    """device tensors of one render call: the case's inputs, every output NaN."""
    R, S, n_o, T = case["R"], case["S"], case["n_outside"], case["T"]
    nan = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")
    cu = lambda t: t.detach().float().contiguous().cuda()
    return dict(o=cu(case["o"]), d=cu(case["d"]), z_vals=cu(case["z_vals"]), z_out=cu(case["z_out"]),
                sample_dist=cu(case["sample_dist"].reshape(-1)), a_emb=cu(case["a_emb"]),
                inv_s=torch.full((1,), 20.0, device="cuda"), color=nan(R, 3), color_sphere=nan(R, 3),
                color_bg=nan(R, 3), cdf=nan(R, S), gradients=nan(R, S, 3), weights=nan(R, T), weights_sum=nan(R),
                inside_sphere=nan(R, S), depth=nan(R), normals=nan(R, 3), gradient_error=nan(1), sv_sdf=nan(R, S),
                sv_rgb=nan(R, S, 3), sv_bg_alpha=nan(R, T), sv_bg_rgb=nan(R, T, 3), sv_z_feed=nan(R, T),
                sv_relax_sum=nan(1))


def render_forward(eng, case, t):
    """nrw_render_forward stamped with a fresh generation, as _RenderFn does; returns the render cfg."""
    from nrw import _lib
    from nrw.engine import _io_struct, make_render_cfg

    rcfg = make_render_cfg(case["R"], case["S"], case["n_outside"], 0.3, None, True)
    eng.generation = getattr(eng, "generation", 0) + 1
    rcfg.reserved0 = eng.generation
    io = _io_struct(t)
    _lib.check(eng.L.nrw_render_forward(eng.ctx, C.byref(rcfg), C.byref(io), _lib.stream_ptr()), "nrw_render_forward")
    return rcfg, io


def upstream_tensors(case, st):
    """device upstream gradients: the set's streams from case["ups"], zeros for the others (the C ABI takes no NULL)."""
    out = {}
    for k in streams_of(case):
        u = case["ups"][k] if k in st else torch.zeros_like(case["ups"][k])
        out[k] = u.float().contiguous().cuda()
    return out


def network_backward(eng, case, rcfg, io, ups, grad_params, grad_a_emb):
    """nrw_network_backward's status (upstream dict may omit streams: NULL pointers)."""
    from nrw import _lib

    p = lambda k: _lib.ptr(ups.get(k))
    return eng.L.nrw_network_backward(eng.ctx, C.byref(rcfg), C.byref(io), p("sdf"), p("normals"), p("rgb"),
                                      p("bg_alpha"), p("bg_rgb"), _lib.ptr(grad_params), _lib.ptr(grad_a_emb),
                                      _lib.stream_ptr())


def unflatten(eng, flat, names):
    return {n: flat[eng.index[n][1]:eng.index[n][1] + eng.index[n][2]].view(eng.index[n][0]) for n in names}


def cuda_network(case, precision, backend, chunk_rows=None, recompute=False, sets=None, prefill=None):
    """For each stream set: nrw_render_forward (a fresh forward in the slots), then nrw_network_backward with exactly
    that set's upstream gradients.  grad_params starts as `prefill` (default zeros: it is accumulated into), grad_a_emb
    as NaN.  Returns (forward dict of the first render incl. sv_z_feed, [gradient dict per set], flat gradients) on the
    CPU; gradient dicts are keyed like the reference's."""
    from nrw import _lib

    sets = stream_sets(case) if sets is None else sets
    eng = make_engine(case, precision, backend, chunk_rows, recompute)
    names = list(net_params(case["P"]))
    fwd, grads, flats = None, [], []
    for st in sets:
        t = render_io(case)
        rcfg, io = render_forward(eng, case, t)
        ups = upstream_tensors(case, st)
        gp = torch.zeros(eng.total, dtype=torch.float32, device="cuda") if prefill is None else prefill.cuda().clone()
        ga = torch.full((case["R"], N_A), float("nan"), dtype=torch.float32, device="cuda")
        _lib.check(network_backward(eng, case, rcfg, io, ups, gp, ga), "nrw_network_backward")
        torch.cuda.synchronize()
        if fwd is None:
            keys = FWD_KEYS if case["n_outside"] > 0 else FWD_KEYS[:3]
            fwd = {k: t[k].cpu() for k in keys + ("sv_z_feed",)}
        flat = gp.cpu()
        res = unflatten(eng, flat, names)
        res["a_emb"] = ga.cpu()
        grads.append(res)
        flats.append(flat)
    return fwd, grads, flats, eng


# --------------------------------------------------------------------------------------------------- tolerance
def tensor_err(x, ref, full):
    """max|x - ref| / (max|ref| + FLOOR_REL max|full|) over the whole tensor; inf for a non-finite x."""
    return ray_err(torch.as_tensor(x).reshape(1, -1), torch.as_tensor(ref).reshape(1, -1),
                   scale=torch.as_tensor(full).reshape(1, -1))


def grad_err(key, x, ref, full):
    """the tolerance rule's error of one gradient: per ray for a_emb, per tensor for a parameter."""
    if key == "a_emb":
        return ray_err(x, ref, scale=full)
    return tensor_err(x, ref, full)


def cosine(x, ref):
    x, ref = torch.as_tensor(x).double().reshape(-1), torch.as_tensor(ref).double().reshape(-1)
    return float((x @ ref) / (x.norm() * ref.norm() + 1e-300))
