"""Stage-level harness for the NeuS compositing kernels (csrc/composite.cu, nrw_composite_forward / _backward).

Per-sample SDF, normals, colours and background alpha/colour are INJECTED, so no network is involved and the port's
render_core (oracle/neuconw_port.py), evaluated in fp64, is an exact reference of the same operation.

  make_case      seeded fp32 inputs mixing five kinds of rays, every sample a fixed margin away from the kernel's
                 discontinuities (sphere masks, the two ReLU kinks of iter_cos)
  reference      render_core on the injected tensors promoted to a dtype; forward dict + autograd gradients
  cuda_composite nrw_composite_forward, then nrw_composite_backward once per set of upstream gradients
  ray_err        per-ray error against the fp64 reference (the tolerance rule below)

Tolerance rule: an output's error is  max over rays of  max|x - ref64| / (max|ref64| + floor)  (per ray, see ray_err
for the floor).  A kernel output passes when that is <= 4 x the same error of the fp32 evaluation of the reference,
or <= 2e-6 (forward) / 2e-5 (backward), whichever is larger."""
import ctypes as C
import types
from contextlib import contextmanager

import numpy as np
import torch

from util_nrw import port

UPSTREAM = ("color", "color_sphere", "color_bg", "cdf", "gradients", "weights", "weights_sum", "depth", "normals",
            "gradient_error")
FWD_KEYS = ("color", "color_sphere", "color_bg", "cdf", "weights", "weights_sum", "depth", "normals", "gradient_error")
BWD_KEYS = ("d_sdf", "d_nrm", "d_rgb", "d_bg_alpha", "d_bg_rgb", "grad_inv_s")
LEAVES = ("sdf", "normals", "rgb", "bg_alpha", "bg_rgb", "inv_s")      # BWD_KEYS[i] is the gradient of LEAVES[i]
# Floor of the per-ray normaliser, relative to the ray's full gradient (all ten upstream gradients together).  On a
# ray that turns opaque behind its surface, the gradient under ONE upstream gradient (weights_sum, weights) is the
# residue of cancelling terms ~1e4 times larger (dA = g*T - (later g*w) / (1 - alpha + 1e-7)); any fp32 evaluation
# keeps ~1e-7 of those terms, so it is measured against 1e-3 of the ray's full gradient.
FLOOR_REL = 1e-3
FWD_FLOOR, BWD_FLOOR = 2e-6, 2e-5
ANCHOR_FACTOR = 4.0


def bwd_floor(case, upstream, key):
    """The backward floor is 2e-5 except for two measured exceptions (H100, worst over the case table):
      * grad_inv_s: one scalar summed over up to 3.8e5 samples, per lane, per warp, then atomically over rays, where
        torch sums pairwise; 1e-4 (measured 3.1e-5 for weights_sum alone at R = 300, S = 252);
      * d_sdf under a single upstream gradient at inv_s >= 1e3, the opaque-ray residue described at FLOOR_REL; 1e-3
        (measured 4.5e-4 for weights_sum alone at inv_s = 1e4, 3.1e-5 for color_sphere alone at inv_s = 1e3)."""
    if key == "grad_inv_s":
        return 1e-4
    if key == "d_sdf" and len(upstream) == 1 and float(case["inv_s"]) >= 1e3:
        return 1e-3
    return BWD_FLOOR
MARGIN = 1e-4             # distance of |p| from 1 and 1.2, and of tc = d.n from 0 and 1
N_KINDS = 5               # crossing, outside the unit sphere, increasing SDF, repeated z, relax shell
MAX_REDRAWS = 200


def cpl(T):
    """samples per lane of the kernel instance that runs T samples per ray (composite.cu: pick_cpl)."""
    return 5 if T <= 160 else (8 if T <= 256 else (16 if T <= 512 else 40))


# name: (R, S, n_outside, inv_s, cos_anneal_ratio, trim_sphere, background_rgb)
# background_rgb: None = NULL pointer, "zeros", or "color" (a non-zero colour)
CASES = {
    "c5_T28_bg": (37, 24, 4, 20.0, 0.3, 1, "zeros"),
    "c5_T28_nobg": (37, 28, 0, 1e3, 0.0, 1, None),
    "c5_T160_bg_notrim_sat": (300, 128, 32, 1e4, 1.0, 0, "color"),
    "c5_T160_nobg_R1": (1, 160, 0, 1.0, 0.3, 0, "color"),
    "c5_T160_bg_soft": (300, 156, 4, 1.0, 0.0, 1, "zeros"),
    "c8_T161_bg_notrim": (37, 157, 4, 20.0, 0.0, 0, "color"),
    "c8_T256_nobg_sat": (300, 256, 0, 1e4, 0.3, 1, "zeros"),
    "c8_T256_bg32": (37, 224, 32, 1e3, 1.0, 1, None),
    "c8_T161_nobg_R1": (1, 161, 0, 20.0, 1.0, 1, "color"),
    "c8_T256_bg_soft_notrim": (300, 252, 4, 1.0, 0.3, 0, None),
    "c16_T257_bg_notrim_sat": (37, 253, 4, 1e4, 0.3, 0, "zeros"),
    "c16_T512_nobg": (37, 512, 0, 20.0, 0.0, 1, "color"),
    "c16_T512_bg32": (300, 480, 32, 1e3, 0.3, 1, "color"),
    "c16_T257_nobg_R1_sat": (1, 257, 0, 1e4, 1.0, 0, None),
    "c40_T513_bg": (37, 509, 4, 20.0, 0.3, 1, "color"),
    "c40_T1056_bg32_sat": (37, 1024, 32, 1e4, 0.3, 1, "zeros"),      # the reference defaults: 512 + 512, 32 outside
    "c40_T1280_bg32_notrim": (300, 1248, 32, 1e3, 0.0, 0, "color"),
    "c40_T1280_nobg_soft": (37, 1280, 0, 1.0, 1.0, 1, None),
    "c40_T513_nobg_R1_sat": (1, 513, 0, 1e4, 0.0, 0, "zeros"),
    "c40_T1056_bg_notrim": (300, 1052, 4, 20.0, 1.0, 0, None),
}


def case_seed(name):
    return sorted(CASES).index(name) + 101


def make_named_case(name):
    R, S, n_o, inv_s, cos, trim, bgc = CASES[name]
    return make_case(R, S, n_o, inv_s, cos, trim, bgc, case_seed(name))


# --------------------------------------------------------------------------------------------------- cases
def _unit(v):
    return v / v.norm(dim=-1, keepdim=True)


def _mid_pn(o, d, z, sample_dist):
    """mid points and their radius, in fp64 (render_core's dists / mid / pts)."""
    o, d, z, sd = o.double(), d.double(), z.double(), sample_dist.double()
    dist = torch.cat([z[:, 1:] - z[:, :-1], sd.expand(z.shape[0], 1)], -1)
    mid = z + dist * 0.5
    pn = (o[:, None, :] + d[:, None, :] * mid[..., None]).norm(dim=-1)
    return dist, mid, pn


def _radius_ok(pn):
    return (((pn - 1.0).abs() >= MARGIN) & ((pn - 1.2).abs() >= MARGIN)).all(-1)


def _tc_ok(d, n):
    tc = (d.double()[:, None, :] * n.double()).sum(-1)
    return ((tc.abs() >= MARGIN) & ((tc - 1.0).abs() >= MARGIN))


def make_case(R, S, n_outside, inv_s, cos_anneal_ratio, trim_sphere, background_rgb, seed):
    """fp32 inputs of one compositing call.  Ray r is of kind (r + seed) % 5:
      0  crosses a surface inside the unit sphere, the SDF falling steeply through zero;
      1  lies entirely outside the unit sphere (and outside radius 1.2): `inside` and `relax` are 0 everywhere;
      2  the SDF increases along the ray: negative (alpha ~ 1, opaque) where the ray enters the sphere, then rising
         through zero at t0;
      3  like 0, with repeated z values (dist = 0) as the sampler's merge produces;
      4  passes between radius 1.0 and 1.2, so `relax` differs from `inside`.
    Rays whose samples come within MARGIN of |p| = 1 or 1.2 get new z values, samples whose tc = d.n comes within
    MARGIN of 0 or 1 get new normals; a ray still violating a margin after MAX_REDRAWS draws is marked in `ok`.

    Every ray carries one pinned sample at its surface crossing with both prev*inv_s and next*inv_s moderate
    (next*inv_s in [-2, 2], 2*h*inv_s in ~[1, 4] through its normal).  With inv_s = 1e4 every other sample has
    |x| >> 17, where fp32 sigmoid(x) rounds to 0 or 1 and P*(1 - P) vanishes; the pinned sample keeps each ray's
    SDF / normal / inv_s gradients above that flush-to-zero level.  The other samples are kept out of the two regimes
    where fp32 cannot resolve the reference's own derivatives (see the SDF block below).

    The lower clip of alpha needs no margin: iter_cos <= 0 and dist >= 0 give prev >= next, hence P >= N and
    alpha_raw = (P - N + 1e-5) / (P + 1e-5) >= 1e-5 / (P + 1e-5) > 0 for every sample (also in fp32, where sigmoid and
    rounding are monotone).  `margins` re-checks this (P >= N in fp64) along with the margins above."""
    g = torch.Generator().manual_seed(int(seed))
    T = S + n_outside
    kind = (torch.arange(R) + seed) % N_KINDS
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    theta = rnd(R) * 2 * np.pi
    lateral = torch.where(kind == 1, 1.5 + 0.0 * theta, torch.where(kind == 4, 1.1 + 0.0 * theta, 0.3 * rnd(R)))
    o = torch.stack([lateral * torch.cos(theta), lateral * torch.sin(theta), torch.full((R,), -3.0, dtype=torch.float64)], -1)
    spread = torch.where(kind == 1, 0.02, torch.where(kind == 4, 0.01, 0.08)).double()
    d = _unit(torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64) + spread[:, None] * (2.0 * rnd(R, 3) - 1.0))
    o, d = o.float(), d.float()
    zlo, zhi = 1.5, 4.5
    sample_dist = torch.full((R, 1), (zhi - zlo) / S, dtype=torch.float32)

    def draw_z(n):
        z = torch.sort(zlo + (zhi - zlo) * rnd(n, S), dim=-1)[0]
        dup = rnd(n, S) < 0.15
        dup[:, 0] = False
        return torch.where(dup, torch.roll(z, 1, -1), z).float()

    z = draw_z(R)
    z = torch.where((kind == 3)[:, None], z, torch.sort(zlo + (zhi - zlo) * rnd(R, S), dim=-1)[0].float())
    ok = torch.ones(R, dtype=torch.bool)
    for _ in range(MAX_REDRAWS):
        bad = ~_radius_ok(_mid_pn(o, d, z, sample_dist)[2])
        if not bad.any():
            break
        zn = draw_z(R)
        zp = torch.sort(zlo + (zhi - zlo) * rnd(R, S), dim=-1)[0].float()
        z = torch.where(bad[:, None], torch.where((kind == 3)[:, None], zn, zp), z)
    ok &= _radius_ok(_mid_pn(o, d, z, sample_dist)[2])

    # normals: |n| in ~[0.5, 1.5], tc = d.n spread over both ReLU kinks (0 and 1)
    def draw_n():
        a = (rnd(R, S, 1) * 2.6 - 1.3)
        return (a * d.double()[:, None, :] + 0.4 * rn(R, S, 3)).float()

    nrm = draw_n()
    for _ in range(MAX_REDRAWS):
        bad = ~_tc_ok(d, nrm)
        if not bad.any():
            break
        nrm = torch.where(bad[..., None], draw_n(), nrm)
    ok &= _tc_ok(d, nrm).all(-1)

    # SDF: linear through a crossing t0 along the ray (falling, or rising for kind 2) + small noise
    dist, mid, pn = _mid_pn(o, d, z, sample_dist)
    t0 = torch.where((kind == 0) | (kind == 3), 2.3 + 1.4 * rnd(R), 2.0 + 2.0 * rnd(R))
    slope = (1.0 + 2.0 * rnd(R)) * torch.where(kind == 2, -1.0, 1.0).double()
    sdf = slope[:, None] * (t0[:, None] - mid) + 0.005 * rn(R, S)
    c, inv_s = float(cos_anneal_ratio), float(inv_s)
    ic_of = lambda tc: -(torch.relu(-tc * 0.5 + 0.5) * (1.0 - c) + torch.relu(-tc) * c)
    rows = torch.arange(R)
    j = (mid - t0[:, None]).abs().argmin(-1)
    # pinned sample j: its normal is chosen so that 2 h inv_s (h = -iter_cos * dist / 2) is as close as the grid of
    # tc allows to a draw in [1, 4], and its SDF puts next * inv_s in [-2, 2]: prev and next are both moderate.
    grid = torch.linspace(-1.0, 1.0, 4001, dtype=torch.float64)
    grid = grid[(grid.abs() >= 10 * MARGIN) & ((grid - 1.0).abs() >= 10 * MARGIN)]
    want = 1.0 + 3.0 * rnd(R)
    k = (-ic_of(grid)[None, :] * dist[rows, j][:, None] * inv_s - want[:, None]).abs().argmin(-1)
    tcj = grid[k]
    dj = d.double()
    perp = _unit(torch.linalg.cross(dj, _unit(rn(R, 3))))
    nrm[rows, j] = (tcj[:, None] * dj + 0.5 * perp).float()
    tc = (d.double()[:, None, :] * nrm.double()).sum(-1)
    h = -ic_of(tc) * dist * 0.5                                      # prev = sdf + h, next = sdf - h
    sdf[rows, j] = h[rows, j] + (rnd(R) * 4.0 - 2.0) / inv_s
    # every other sample stays out of the two regimes where fp32 cannot resolve the reference's own derivatives
    # (a gradient there is rounding noise in ANY fp32 evaluation, so no tolerance anchored to fp32 could check it):
    #  * x = prev * inv_s or next * inv_s in [6, 20]: 1 - sigmoid(x) < 2.5e-3 is held to a few ulps of 1;
    #  * |prev * inv_s| < 25 with next * inv_s < -7: the quotient rule's dalpha/dP = N / (P + 1e-5)^2 is far below
    #    the rounding of its fp32 evaluation as 1/den - num/den^2.
    # Such samples are moved to prev * inv_s in [-35, -25] (fully opaque, no sensitivity left).
    xp, xn = (sdf + h) * inv_s, (sdf - h) * inv_s
    band = lambda x: (x >= 6.0) & (x <= 20.0)
    bad = band(xp) | band(xn) | ((xp.abs() < 25.0) & (xn < -7.0))
    bad[rows, j] = False
    sdf = torch.where(bad, -(25.0 + 10.0 * rnd(R, S)) / inv_s - h, sdf)
    sdf = sdf.float()
    rgb = torch.rand(R, S, 3, generator=g)
    # background alpha as the NeRF head makes it, 1 - exp(-sigma * dist) with sigma in [0, 1.5): the optical depth
    # before the unit sphere stays <= ~1, so the surface is still visible through the background (bg_transmittance)
    if n_outside > 0:
        bg_dist = torch.cat([dist, sample_dist.double().expand(R, n_outside)], -1)
        bg_alpha = (1.0 - torch.exp(-1.5 * rnd(R, T) * bg_dist)).float()
    else:
        bg_alpha = None
    bg_rgb = torch.rand(R, T, 3, generator=g) if n_outside > 0 else None
    if background_rgb is None:
        bgc = None
    elif background_rgb == "zeros":
        bgc = torch.zeros(1, 3)
    else:
        assert background_rgb == "color"
        bgc = torch.tensor([[0.25, 0.5, 0.75]])
    case = dict(R=R, S=S, n_outside=n_outside, T=T, cos_anneal_ratio=float(cos_anneal_ratio),
                trim_sphere=int(bool(trim_sphere)), background_rgb=bgc, o=o.contiguous(), d=d.contiguous(),
                z_vals=z.contiguous(), sample_dist=sample_dist, sdf=sdf.contiguous(), normals=nrm.contiguous(),
                rgb=rgb, bg_alpha=bg_alpha, bg_rgb=bg_rgb, inv_s=torch.tensor([[float(inv_s)]]), kind=kind, ok=ok,
                pinned=j)
    return case


def margins(case):
    """Per-margin booleans over all samples, evaluated in fp64 on the fp32 inputs (all True for a valid case)."""
    dist, mid, pn = _mid_pn(case["o"], case["d"], case["z_vals"], case["sample_dist"])
    tc = (case["d"].double()[:, None, :] * case["normals"].double()).sum(-1)
    c = case["cos_anneal_ratio"]
    ic = -(torch.relu(-tc * 0.5 + 0.5) * (1.0 - c) + torch.relu(-tc) * c)
    sdf, inv_s = case["sdf"].double(), float(case["inv_s"])
    P = torch.sigmoid((sdf - ic * dist * 0.5) * inv_s)
    N = torch.sigmoid((sdf + ic * dist * 0.5) * inv_s)
    return dict(radius_1=bool(((pn - 1.0).abs() >= MARGIN).all()), radius_1p2=bool(((pn - 1.2).abs() >= MARGIN).all()),
                tc_0=bool((tc.abs() >= MARGIN).all()), tc_1=bool(((tc - 1.0).abs() >= MARGIN).all()),
                alpha_raw_positive=bool((P >= N).all()) and bool((dist >= 0).all()))


def bg_transmittance(case):
    """merged transmittance at each ray's first sample inside the unit sphere (fp64; NaN for rays that never enter
    it): the share of the surface's weight the background leaves."""
    R, S = case["R"], case["S"]
    pn = _mid_pn(case["o"], case["d"], case["z_vals"], case["sample_dist"])[2]
    inside = pn < 1.0
    first = torch.where(inside.any(-1), inside.double().argmax(-1), torch.full((R,), -1))
    x = 1.0 - case["bg_alpha"][:, :S].double() + 1e-7
    before = torch.arange(S)[None, :] < first[:, None]
    t = torch.where(before, x, torch.ones_like(x)).prod(-1)
    return torch.where(first >= 0, t, torch.full_like(t, float("nan")))


def make_ups(case, seed=0):
    """one random upstream gradient per render output (fp32, shapes of render_core's outputs)."""
    g = torch.Generator().manual_seed(int(seed) + 7)
    R, S, T = case["R"], case["S"], case["T"]
    shapes = dict(color=(R, 3), color_sphere=(R, 3), color_bg=(R, 3), cdf=(R, S), gradients=(R, S, 3), weights=(R, T),
                  weights_sum=(R, 1), depth=(R,), normals=(R, 3), gradient_error=())
    return {k: torch.randn(shapes[k], generator=g) for k in UPSTREAM}


def upstream_sets():
    """the ten single upstream gradients, then all ten together."""
    return [(k,) for k in UPSTREAM] + [UPSTREAM]


# --------------------------------------------------------------------------------------------------- reference
@contextmanager
def injected(leaves):
    """replace the port's network by the injected (rgb, inv_s, sdf, normals) leaves; always restored."""
    saved = port.neuconw_forward
    try:
        port.neuconw_forward = lambda P_, pts_, dirs_, a_: (leaves["rgb"], leaves["inv_s"], leaves["sdf"],
                                                            leaves["normals"])
        yield
    finally:
        port.neuconw_forward = saved


def render_leaves(case, leaves, dtype):
    """render_core on leaf tensors: sdf [R*S,1], normals [R*S,3], rgb [R*S,3], bg_alpha [R,T], bg_rgb [R,T,3],
    inv_s [1,1] (bg_* None without a background)."""
    R = case["R"]
    cv = lambda t: t.to(dtype)
    cfg = types.SimpleNamespace(trim_sphere=bool(case["trim_sphere"]))
    bgc = None if case["background_rgb"] is None else cv(case["background_rgb"])
    with injected(leaves):
        return port.render_core(None, cfg, cv(case["o"]), cv(case["d"]), cv(case["z_vals"]), cv(case["sample_dist"]),
                                torch.zeros(R, 1, dtype=dtype), case["cos_anneal_ratio"], leaves["bg_alpha"],
                                leaves["bg_rgb"], bgc)


def make_leaves(case, dtype):
    R, S = case["R"], case["S"]
    lv = dict(sdf=case["sdf"].reshape(R * S, 1), normals=case["normals"].reshape(R * S, 3),
              rgb=case["rgb"].reshape(R * S, 3), bg_alpha=case["bg_alpha"], bg_rgb=case["bg_rgb"], inv_s=case["inv_s"])
    return {k: (None if v is None else v.detach().to(dtype).clone().requires_grad_(True)) for k, v in lv.items()}


def relax_count(case):
    pn = _mid_pn(case["o"], case["d"], case["z_vals"], case["sample_dist"])[2]
    return float((pn < 1.2).double().sum())


def reference(case, dtype, ups=None, sets=()):
    """render_core in `dtype` on the injected inputs.  Returns (forward dict, [gradient dict per upstream set]):
    for each tuple of UPSTREAM names in `sets`, autograd gradients of sum_k <out_k, ups_k> with respect to the six
    leaves, keyed by BWD_KEYS (d_bg_* are zeros without a background)."""
    R, S, T = case["R"], case["S"], case["T"]
    leaves = make_leaves(case, dtype)
    out = render_leaves(case, leaves, dtype)
    fwd = {k: out[k].detach() for k in FWD_KEYS + ("inside_sphere", "gradients")}
    shapes = dict(d_sdf=(R, S), d_nrm=(R, S, 3), d_rgb=(R, S, 3), d_bg_alpha=(R, T), d_bg_rgb=(R, T, 3), grad_inv_s=())
    grads = []
    for st in sets:
        terms = [(out[k] * ups[k].to(dtype)).sum() for k in st if out[k].requires_grad]
        res = {k: torch.zeros(shapes[k], dtype=dtype) for k in BWD_KEYS}
        if terms:
            names = [n for n in LEAVES if leaves[n] is not None]
            gs = torch.autograd.grad(sum(terms), [leaves[n] for n in names], retain_graph=True, allow_unused=True)
            for n, gv in zip(names, gs):
                if gv is not None:
                    key = BWD_KEYS[LEAVES.index(n)]
                    res[key] = gv.detach().reshape(shapes[key])
        grads.append(res)
    return fwd, grads


# --------------------------------------------------------------------------------------------------- CUDA
def cuda_composite(case, ups=None, sets=()):
    """nrw_composite_forward, then nrw_composite_backward once per upstream set with exactly those upstream gradients
    non-NULL.  Every output buffer starts as NaN, so an element the kernel does not write fails the comparison.
    Returns (forward dict, [backward dict per set]) on the CPU; forward also carries sv_relax_sum."""
    from nrw import _lib
    from nrw._lib import RenderGrads
    from nrw.engine import _io_struct, make_render_cfg

    L = _lib.lib()
    R, S, n_o, T = case["R"], case["S"], case["n_outside"], case["T"]
    bg = n_o > 0
    nan = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")
    cu = lambda t: None if t is None else t.detach().float().contiguous().cuda()
    t = dict(o=cu(case["o"]), d=cu(case["d"]), z_vals=cu(case["z_vals"]), z_out=nan(R, n_o),
             sample_dist=cu(case["sample_dist"].reshape(-1)), a_emb=nan(R, 48), inv_s=cu(case["inv_s"].reshape(1)),
             color=nan(R, 3), color_sphere=nan(R, 3), color_bg=nan(R, 3), cdf=nan(R, S), gradients=nan(R, S, 3),
             weights=nan(R, T), weights_sum=nan(R), inside_sphere=nan(R, S), depth=nan(R), normals=nan(R, 3),
             gradient_error=nan(1), sv_sdf=cu(case["sdf"]), sv_rgb=cu(case["rgb"]), sv_bg_alpha=cu(case["bg_alpha"]),
             sv_bg_rgb=cu(case["bg_rgb"]), sv_z_feed=nan(R, T), sv_relax_sum=nan(1))
    nrm = cu(case["normals"])
    bgc = cu(case["background_rgb"])
    rcfg = make_render_cfg(R, S, n_o, case["cos_anneal_ratio"], bgc, case["trim_sphere"])
    io = _io_struct(t)
    scratch = nan(2)
    _lib.check(L.nrw_composite_forward(C.byref(rcfg), C.byref(io), _lib.ptr(t["sv_sdf"]), _lib.ptr(nrm),
                                       _lib.ptr(t["sv_rgb"]), _lib.ptr(t["sv_bg_alpha"] if bg else None),
                                       _lib.ptr(t["sv_bg_rgb"] if bg else None), _lib.ptr(scratch), _lib.stream_ptr()),
               "nrw_composite_forward")
    torch.cuda.synchronize()
    fwd = {k: t[k].cpu() for k in FWD_KEYS + ("inside_sphere", "gradients", "sv_relax_sum")}
    bwds = []
    for st in sets:
        gr = RenderGrads()
        keep = {}
        for k in UPSTREAM:
            keep[k] = cu(ups[k].reshape(-1)) if k in st else None
            setattr(gr, "g_" + k, _lib.ptr(keep[k]))
        out = dict(d_sdf=nan(R, S), d_nrm=nan(R, S, 3), d_rgb=nan(R, S, 3), d_bg_alpha=nan(R, T), d_bg_rgb=nan(R, T, 3),
                   grad_inv_s=nan(1))
        gr.grad_params, gr.grad_a_emb, gr.grad_inv_s = None, None, _lib.ptr(out["grad_inv_s"])
        _lib.check(L.nrw_composite_backward(C.byref(rcfg), C.byref(io), C.byref(gr), _lib.ptr(nrm),
                                            _lib.ptr(out["d_sdf"]), _lib.ptr(out["d_nrm"]), _lib.ptr(out["d_rgb"]),
                                            _lib.ptr(out["d_bg_alpha"]), _lib.ptr(out["d_bg_rgb"]), _lib.stream_ptr()),
                   "nrw_composite_backward")
        torch.cuda.synchronize()
        res = {k: v.cpu() for k, v in out.items()}
        res["grad_inv_s"] = res["grad_inv_s"].reshape(())
        bwds.append(res)
    return fwd, bwds


# --------------------------------------------------------------------------------------------------- tolerance
def ray_err(x, ref, ok=None, scale=None, floor_rel=None):
    """max over rays of  max|x - ref| / (max|ref| + FLOOR_REL * max|scale| + 1e-30),  maxima taken over the ray.
    `scale` (default: ref) is the same output's fp64 value under all ten upstream gradients together, i.e. the
    ray's full gradient.  A 0-d tensor is one ray.  Non-finite x gives inf."""
    floor_rel = FLOOR_REL if floor_rel is None else floor_rel
    x = torch.as_tensor(x).double()
    ref = torch.as_tensor(ref).double().reshape(x.shape)
    scale = ref if scale is None else torch.as_tensor(scale).double().reshape(x.shape)
    if x.dim() == 0:
        x, ref, scale = x.reshape(1, 1), ref.reshape(1, 1), scale.reshape(1, 1)
    else:
        x, ref, scale = (t.reshape(t.shape[0], -1) for t in (x, ref, scale))
        if ok is not None:
            x, ref, scale = x[ok], ref[ok], scale[ok]
    if x.numel() == 0:
        return 0.0
    if not torch.isfinite(x).all():
        return float("inf")
    den = ref.abs().amax(-1) + floor_rel * scale.abs().amax(-1) + 1e-30
    return float(((x - ref).abs().amax(-1) / den).max())


def judge(x, ref64, ref32, floor, ok=None, scale=None, factor=ANCHOR_FACTOR):
    """(kernel error, fp32-reference error, bound, passed) under the tolerance rule."""
    e = ray_err(x, ref64, ok, scale)
    a = ray_err(ref32, ref64, ok, scale)
    bound = max(factor * a, floor)
    return e, a, bound, e <= bound
