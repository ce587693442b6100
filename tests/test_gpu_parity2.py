"""GPU parity, round-2 additions (VERDICT r1 weak #1-#3, #9):
  * a full train step at the BENCHMARKED sample counts (C2: 64 + 64, k = 4, 4 outside) vs the oracle port;
  * the perturbed-strata and the surface-guided fine-sampling goldens produced by the UNMODIFIED reference
    (tests/golden/small_perturb.npz, fine_c3.npz; octree trace results injected, oracle/make_golden.py);
  * stage-wise compositing (nrw_composite_forward / nrw_composite_backward) with injected per-sample inputs;
  * NeuconWRenderer.rgb / .sdf;
  * the measured searchsorted-index mismatch rate of the whole CUDA sampler vs the reference ops (reported).
Everything goes through the C ABI (ctypes) or the host mirror that calls it."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from util_nrw import build_system, cuda_train_step, port, rel_err, synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4


@pytest.fixture(scope="module")
def P():
    return synth.make_params(seed=0)


def _report(name, obj):
    """measured parity figures of this run -> gpurun_out/parity_report.json (copied to profiles/ by hand)."""
    d = os.path.join(ROOT, "gpurun_out")
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, "parity_report.json")
    cur = json.load(open(p)) if os.path.isfile(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, "w"), indent=1, sort_keys=True)
    print(f"[parity] {name}: {obj}")


def install_injected_hits(renderer, hits):
    """CUDA-side twin of oracle.make_golden.install_injected_hits: the octree TRACER (csrc/octree.cu) is replaced by
    the injected trace results; NeuconWRenderer.get_near_far_octree / get_near_far_sdf / sparse_sampler run as usual."""
    coarse, fine = {"tag": "coarse"}, {"tag": "fine", "voxel_size": hits["fine_voxel_sfm"]}

    def fake_trace(od, rays_o_sfm, rays_d):
        dev = rays_o_sfm.device
        if od is fine:
            return hits["surface"].to(dev), None
        assert od is coarse
        return hits["sfm_near"].to(dev), hits["sfm_far"].to(dev)

    renderer._octree_near_far = fake_trace
    renderer.octree_data, renderer.fine_octree_data = coarse, fine
    renderer.nerf_far_override = True
    renderer.voxel_size = hits["voxel_size"]


# ------------------------------------------------------------------------------------------------------------
def test_train_step_c2_sample_counts(P):
    """BASELINE C2 counts (64 coarse + 64 importance in 4 rounds + 4 outside -> S=128, T=132), brandenburg frame,
    perturbed strata with injected draws, R=64, bf16x3 tensor-core path vs the oracle port: 1e-4 on every dict key."""
    cfg = synth.PathConfig(perturb=1.0, **synth.BRANDENBURG)
    assert (cfg.n_samples, cfg.n_importance, cfg.up_sample_steps, cfg.n_outside) == (64, 64, 4, 4)
    R = 64
    batch = synth.make_rays(R, cfg, seed=13)
    noise = synth.make_perturb_noise(R, cfg.n_outside, seed=6)
    res_p, loss_p, grads_p = port.train_step(P, cfg, batch, perturb_overwrite=-1, noise=noise)
    s = build_system(P, cfg, precision="bf16x3", backend=0, chunk_rows=4096)
    res_c, loss_c, grads_c = cuda_train_step(s, cfg, batch, perturb_overwrite=-1, noise=noise)
    assert res_c["weights"].shape == (R, 132) and res_c["gradients"].shape == (R, 128, 3)
    errs = {}
    for k in res_p:
        a, b = res_c[k].numpy(), res_p[k].detach().numpy()
        assert a.shape == b.shape, k
        errs[k] = rel_err(a, b)
    _report("c2_counts_train_step_output_rel_err", {k: float(f"{v:.3g}") for k, v in errs.items()})
    for k, e in errs.items():
        assert e < RTOL, (k, e)
    assert np.array_equal(res_c["inside_sphere"].numpy(), res_p["inside_sphere"].numpy())
    assert abs(float(loss_c) - float(loss_p)) < RTOL * abs(float(loss_p))
    gmax = max(float(g.abs().max()) for g in grads_p.values())
    gerr = {}
    for k in grads_p:
        if float(grads_p[k].abs().max()) < 1e-4 * gmax:
            continue
        gerr[k] = rel_err(grads_c[k].numpy(), grads_p[k].numpy())
    _report("c2_counts_train_step_max_param_grad_rel_err", float(f"{max(gerr.values()):.3g}"))
    for k, e in gerr.items():
        assert e < 1e-2, (k, e)


@pytest.mark.parametrize("name", ["small_perturb", "fine_c3"])
def test_cuda_vs_reference_golden_perturb_and_fine(P, name):
    """CUDA path vs the UNMODIFIED reference's tensors: perturbed strata (the reference's two torch.rand draws after
    torch.manual_seed(seed) are reproduced on the CPU generator and injected) and, for fine_c3, SfM-octree near/far
    override + surface-guided sampling window + boundary samples (renderer.py:380-456, 546-566)."""
    from oracle.make_golden import CASES, FINE_CASES, grad_probe

    cfg, n_rays, pov, rseed = CASES[name]
    G = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    batch = synth.make_rays(n_rays, cfg, seed=11)
    torch.manual_seed(rseed)                       # renderer.py:499,506-508: rand([R,1]) then rand([R,n_outside])
    noise = (torch.rand([n_rays, 1]), torch.rand([n_rays, cfg.n_outside]))
    s = build_system(P, cfg, precision="bf16x3", backend=0, chunk_rows=2048)
    if name in FINE_CASES:
        install_injected_hits(s["renderer"], synth.make_injected_hits(batch, cfg))
    res_c, loss_c, grads_c = cuda_train_step(s, cfg, batch, perturb_overwrite=pov, noise=noise)
    ex = s["renderer"].last_extras
    # strata that do not depend on the network: fp32-exact up to 1 ulp of the torch evaluation
    assert rel_err(ex["z_vals_outside"].cpu().numpy(), G["z_vals_outside"]) < 1e-6
    assert rel_err(ex["sample_dist"].cpu().numpy(), G["sample_dist"]) < 1e-6
    z = ex["z_vals"].cpu().numpy()
    assert z.shape == G["z_vals"].shape
    assert np.all(z[:, 1:] >= z[:, :-1])
    # inverse-cdf sampling is discontinuous in the SDF: a ray whose importance sample moved to a neighbouring bin
    # (tensor-core SDF vs fp32 SDF, |delta| ~ 1e-6) is counted, reported and excluded from the per-ray comparison
    same = np.abs(z - G["z_vals"]).max(axis=1) <= 2e-5 * np.abs(G["z_vals"]).max()
    _report(f"golden_{name}_rays_with_flipped_bins", int((~same).sum()))
    assert same.sum() >= int(0.95 * n_rays), int(same.sum())
    per_ray = ("color", "color_sphere", "color_bg", "cdf_fine", "gradients", "mask_error", "weights", "weights_sum",
               "weights_max", "inside_sphere", "depth")
    for k in per_ray:
        a, b = res_c[k].numpy()[same], G["out." + k][same]
        assert rel_err(a, b) < RTOL, (k, rel_err(a, b))
    if same.all():
        for k, v in res_c.items():
            assert rel_err(v.numpy(), G["out." + k]) < RTOL, k
        assert abs(float(loss_c) - float(G["loss"])) < RTOL * abs(float(G["loss"]))
        gp = grad_probe(grads_c)
        big = max(float(np.abs(G[k]).max()) for k in G.files if k.startswith("gp."))
        for k, v in gp.items():
            if np.abs(G["gp." + k]).max() > 1e-3 * big:
                assert rel_err(v, G["gp." + k]) < 3e-3, k


# ------------------------------------------------------------------------------------------------------------
def test_sampler_index_mismatch_rate_reported(P):
    """Whole CUDA sampler (tensor-core SDF queries inside) at C2 counts vs the reference ops (oracle port, fp32 SDF):
    searchsorted indices of every up-sampling round.  Given IDENTICAL sdf inputs the CUDA round is bit-exact against
    the written-down restatement and that restatement has 0 mismatches against torch on the seeded cases
    (tests/test_sampler_oracle.py); what is measured here is the effect of the SDF's 1e-6 differences."""
    from nrw.engine import make_sampler_cfg

    cfg = synth.PathConfig(perturb=1.0, **synth.BRANDENBURG)
    R = 128
    batch = synth.make_rays(R, cfg, seed=21)
    noise = synth.make_perturb_noise(R, cfg.n_outside, seed=5)
    rays = batch["rays"]
    o = ((rays[:, 0:3] - torch.tensor(cfg.origin, dtype=torch.float64).float()) / cfg.radius).float()
    d = rays[:, 3:6]
    near, far = (rays[:, 6:7] / cfg.radius).float(), (rays[:, 7:8] / cfg.radius).float()
    trace = []
    with torch.no_grad():
        port.sparse_sampler(P, cfg, o, d, near, far, cfg.perturb, noise=noise, trace=trace)
    s = build_system(P, cfg, precision="bf16x3", backend=0, chunk_rows=4096)
    scfg = make_sampler_cfg(cfg.n_samples, cfg.n_importance, cfg.up_sample_steps, cfg.n_outside, cfg.s_val_base, 0, True)
    eng = s["renderer"].engine
    z, zo, sd, ti, to = eng.sample(scfg, o.cuda(), d.cuda().contiguous(), near.cuda(), far.cuda(), None, None,
                                   noise[0].cuda(), noise[1].cuda(), trace=True)
    k, n_new = cfg.up_sample_steps, cfg.n_importance // cfg.up_sample_steps
    ti = ti.cpu().numpy().reshape(k, R, n_new)
    mism = [int((ti[i] != trace[i]["inds"].numpy()).sum()) for i in range(k)]
    rate = sum(mism) / float(k * R * n_new)
    _report("c2_sampler_searchsorted_index_mismatch_vs_reference_ops", {"per_round": mism, "total": k * R * n_new, "rate": rate})
    assert rate < 2e-2
    assert rel_err(z.cpu().numpy(), trace[-1]["z_out"].numpy()) < 2e-3   # a flipped bin moves one sample by < one bin


# ------------------------------------------------------------------------------------------------------------
def _io(t):
    from nrw import _lib
    from nrw.engine import _io_struct

    return _io_struct(t)


def test_composite_stage_injected_inputs():
    """nrw_composite_forward / nrw_composite_backward (K4, renderer.py:365-378,570-783) with INJECTED per-sample
    sdf / normals / rgb / background alpha+rgb, against autograd through the port's render_core."""
    from nrw import _lib
    from nrw._lib import RenderGrads
    from nrw.engine import make_render_cfg

    L = _lib.lib()
    g = torch.Generator().manual_seed(4)
    R, S, n_o = 37, 24, 4
    T = S + n_o
    cfg = synth.PathConfig(n_outside=n_o)
    o = torch.tensor([0.0, 0.0, -3.0]).expand(R, 3).contiguous()
    d = torch.randn(R, 3, generator=g) * 0.12 + torch.tensor([0.0, 0.0, 1.0])
    d = (d / d.norm(dim=-1, keepdim=True)).contiguous()
    z = torch.sort(torch.rand(R, S, generator=g) * 2.0 + 2.0, dim=-1)[0].contiguous()
    sample_dist = torch.full((R, 1), 2.0 / S)
    mid = z + torch.cat([z[:, 1:] - z[:, :-1], sample_dist], -1) * 0.5
    pts = o[:, None] + d[:, None] * mid[..., None]
    sdf = (pts.norm(dim=-1) - 0.5 + 0.02 * torch.randn(R, S, generator=g)).reshape(-1, 1)
    nrm = pts / pts.norm(dim=-1, keepdim=True) + 0.1 * torch.randn(R, S, 3, generator=g)
    rgb = torch.rand(R * S, 3, generator=g)
    bg_alpha = torch.rand(R, T, generator=g) * 0.3
    bg_rgb = torch.rand(R, T, 3, generator=g)
    inv_s = torch.tensor([[20.0]])
    leaves = [t.clone().requires_grad_(True) for t in (sdf, nrm.reshape(-1, 3), rgb, bg_alpha, bg_rgb, inv_s)]
    saved = port.neuconw_forward
    try:
        port.neuconw_forward = lambda P_, pts_, dirs_, a_: (leaves[2], leaves[5], leaves[0], leaves[1])
        ret = port.render_core(None, cfg, o, d, z, sample_dist, torch.zeros(R, 48), 0.3, leaves[3], leaves[4],
                               torch.zeros(1, 3))
    finally:
        port.neuconw_forward = saved
    ups = {k: torch.randn(ret[k].shape, generator=g) for k in
           ("color", "color_sphere", "color_bg", "weights", "weights_sum", "depth", "normals", "gradient_error")}
    ups["cdf"] = torch.randn(R, S, generator=g) * 0.1
    obj = sum((ret[k] * ups[k]).sum() for k in ups)
    obj.backward()
    # ---- CUDA ----
    f = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device="cuda")
    c = lambda t: t.detach().float().contiguous().cuda()
    t = dict(o=c(o), d=c(d), z_vals=c(z), z_out=f(R, n_o), sample_dist=c(sample_dist.reshape(-1)), a_emb=f(R, 48),
             inv_s=c(inv_s.reshape(1)), color=f(R, 3), color_sphere=f(R, 3), color_bg=f(R, 3), cdf=f(R, S),
             gradients=f(R, S, 3), weights=f(R, T), weights_sum=f(R), inside_sphere=f(R, S), depth=f(R), normals=f(R, 3),
             gradient_error=f(1), sv_sdf=c(sdf.reshape(R, S)), sv_rgb=c(rgb.reshape(R, S, 3)), sv_bg_alpha=c(bg_alpha),
             sv_bg_rgb=c(bg_rgb), sv_z_feed=f(R, T), sv_relax_sum=f(1))
    nrm_c = c(nrm)
    rcfg = make_render_cfg(R, S, n_o, 0.3, torch.zeros(1, 3, device="cuda"), True)
    io = _io(t)
    scratch = f(4)
    _lib.check(L.nrw_composite_forward(C.byref(rcfg), C.byref(io), _lib.ptr(t["sv_sdf"]), _lib.ptr(nrm_c), _lib.ptr(t["sv_rgb"]),
                                       _lib.ptr(t["sv_bg_alpha"]), _lib.ptr(t["sv_bg_rgb"]), _lib.ptr(scratch),
                                       _lib.stream_ptr()), "nrw_composite_forward")
    torch.cuda.synchronize()
    for k_c, k_p in (("color", "color"), ("color_sphere", "color_sphere"), ("color_bg", "color_bg"), ("weights", "weights"),
                     ("depth", "depth"), ("normals", "normals"), ("cdf", "cdf"), ("inside_sphere", "inside_sphere")):
        assert rel_err(t[k_c].cpu().numpy(), ret[k_p].detach().numpy().reshape(t[k_c].shape)) < 2e-5, k_c
    assert rel_err(t["weights_sum"].cpu().numpy(), ret["weights_sum"].detach().numpy().reshape(-1)) < 2e-5
    assert abs(float(t["gradient_error"]) - float(ret["gradient_error"])) < 2e-5 * abs(float(ret["gradient_error"]))
    gr = RenderGrads()
    keep = {}
    for k_g, k_u in (("g_color", "color"), ("g_color_sphere", "color_sphere"), ("g_color_bg", "color_bg"), ("g_cdf", "cdf"),
                     ("g_weights", "weights"), ("g_weights_sum", "weights_sum"), ("g_depth", "depth"), ("g_normals", "normals"),
                     ("g_gradient_error", "gradient_error")):
        keep[k_g] = c(ups[k_u].reshape(-1))
        setattr(gr, k_g, _lib.ptr(keep[k_g]))
    gr.g_gradients = None
    g_invs, g_a, g_flat = f(1), f(R, 48), f(8)
    gr.grad_params, gr.grad_a_emb, gr.grad_inv_s = _lib.ptr(g_flat), _lib.ptr(g_a), _lib.ptr(g_invs)
    d_sdf, d_nrm, d_rgb, d_bga, d_bgc = f(R, S), f(R, S, 3), f(R, S, 3), f(R, T), f(R, T, 3)
    _lib.check(L.nrw_composite_backward(C.byref(rcfg), C.byref(io), C.byref(gr), _lib.ptr(nrm_c), _lib.ptr(d_sdf),
                                        _lib.ptr(d_nrm), _lib.ptr(d_rgb), _lib.ptr(d_bga), _lib.ptr(d_bgc),
                                        _lib.stream_ptr()), "nrw_composite_backward")
    torch.cuda.synchronize()
    want = dict(d_sdf=leaves[0].grad.reshape(R, S), d_nrm=leaves[1].grad.reshape(R, S, 3), d_rgb=leaves[2].grad.reshape(R, S, 3),
                d_bga=leaves[3].grad, d_bgc=leaves[4].grad)
    got = dict(d_sdf=d_sdf, d_nrm=d_nrm, d_rgb=d_rgb, d_bga=d_bga, d_bgc=d_bgc)
    for k in want:
        assert rel_err(got[k].cpu().numpy(), want[k].numpy()) < 1e-4, (k, rel_err(got[k].cpu().numpy(), want[k].numpy()))
    assert abs(float(g_invs) - float(leaves[5].grad)) < 1e-4 * abs(float(leaves[5].grad)) + 1e-7


def test_renderer_rgb_and_sdf(P):
    """NeuconWRenderer.sdf / .rgb (renderer.py:947-961) on arbitrary points vs the port's network ops."""
    cfg = synth.PathConfig()
    s = build_system(P, cfg, precision="bf16x3", backend=0, chunk_rows=2048)
    r = s["renderer"]
    g = torch.Generator().manual_seed(8)
    n = 777
    pts = (torch.rand(n, 1, 3, generator=g) * 2 - 1) * 0.8
    dirs = torch.randn(n, 1, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    a = torch.randn(n, 1, 48, generator=g)
    with torch.no_grad():
        sdf_c = r.sdf(pts.cuda()).cpu()
        rgb_c = r.rgb(pts.cuda(), dirs.cuda(), a.cuda()).cpu()
    Pg = {k: v.clone() for k, v in P.items()}
    rgb_p, _, sdf_p, _ = port.neuconw_forward(Pg, pts.reshape(-1, 3), dirs.reshape(-1, 3), a.reshape(n, 48))
    assert sdf_c.shape == (n, 1) and rgb_c.shape == (n, 3)
    assert rel_err(sdf_c.numpy().ravel(), sdf_p.detach().numpy().ravel()) < RTOL
    assert rel_err(rgb_c.numpy(), rgb_p.detach().numpy()) < RTOL
