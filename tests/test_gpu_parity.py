"""GPU parity tests: the CUDA path (through the C ABI) vs the CPU oracle port on identical seeded inputs,
vs the committed golden vectors of the unmodified reference, and size-independent properties at the
full BASELINE C2 shape.  Tolerance: 1e-4 relative (north-star) on rendered outputs."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from util_nrw import build_system, cuda_train_step, gemm_test, port, rel_err, synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4


@pytest.fixture(scope="module")
def P():
    return synth.make_params(seed=0)


# ------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("backend", [0, 1])
@pytest.mark.parametrize("shape", [(300, 512, 512), (1000, 64, 512), (777, 128, 640), (640, 256, 192), (129, 512, 64)])
def test_gemm_forward_form(backend, shape):
    M, N, K = shape
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(N, K, device="cuda") / np.sqrt(K)
    bias = torch.randn(N, device="cuda")
    ref = (A.double() @ B.double().T + bias.double()).float().cpu()
    for planes, tol in ((1, 6e-3), (2, 2e-5), (3, 2e-5)):
        D = gemm_test(backend, planes, 0, 1, A, B, bias, 0).cpu()
        assert rel_err(D, ref) < tol, (backend, shape, planes)


@pytest.mark.parametrize("backend", [0, 1])
@pytest.mark.parametrize("shape", [(5000, 512, 512, 4), (3000, 128, 640, 3), (2048, 256, 192, 1), (1000, 512, 64, 2),
                                   (4100, 256, 1024, 3), (3000, 512, 640, 2), (9000, 768, 512, 5)])
def test_gemm_weight_gradient_form(backend, shape):
    Ks, M, N, ks = shape
    torch.manual_seed(1)
    A = torch.randn(Ks, M, device="cuda")
    B = torch.randn(Ks, N, device="cuda") / np.sqrt(Ks)
    ref = (A.double().T @ B.double()).float().cpu()
    for planes, tol in ((1, 8e-3), (2, 5e-5), (3, 5e-5)):
        D = gemm_test(backend, planes, 1, ks, A, B, None, 0).cpu()
        assert rel_err(D, ref) < tol, (backend, shape, planes)


def test_gemm_epilogue_activations():
    torch.manual_seed(2)
    A = torch.randn(257, 128, device="cuda") * 0.1
    B = torch.randn(130, 128, device="cuda") * 0.1
    bias = torch.randn(130, device="cuda") * 0.01
    pre = (A.double() @ B.double().T + bias.double())
    refs = {1: torch.nn.functional.softplus(pre, beta=100), 2: torch.relu(pre), 3: torch.sigmoid(pre)}
    for act, ref in refs.items():
        for backend in (0, 1):
            D = gemm_test(backend, 3, 0, 1, A, B, bias, act).cpu()
            assert rel_err(D, ref.float().cpu()) < 2e-5, (act, backend)


# ------------------------------------------------------------------------------------------- MLPs
@pytest.mark.parametrize("precision,tol", [("bf16x3", RTOL), ("bf16x6", RTOL)])
def test_networks_forward(P, precision, tol):
    cfg = synth.PathConfig()
    s = build_system(P, cfg, precision=precision, backend=0, chunk_rows=4096)
    torch.manual_seed(1)
    n = 6000  # > one chunk, ragged tail
    x = (torch.rand(n, 3) * 2 - 1) * 0.9
    out = port.sdf_forward(P, x)
    g = port.sdf_gradient(P, x, create_graph=False)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    a = torch.randn(n, 48)
    rgb_ref = port.color_forward(P, x, g, dirs, out[:, 1:], a).detach()
    sdf = s["renderer"].sdf(x.cuda().reshape(-1, 1, 3)).cpu().reshape(-1)
    assert rel_err(sdf, out[:, 0].detach()) < tol
    xin = torch.cat([x, dirs, a], -1).reshape(n // 6, 6, 54).cuda()
    rgb, inv_s, sdf2, nrm = s["neuconw"](xin)
    assert rel_err(sdf2.cpu().reshape(-1), out[:, 0].detach()) < tol
    assert rel_err(nrm.cpu().reshape(-1, 3), g.detach()) < tol
    assert rel_err(rgb.cpu().reshape(-1, 3), rgb_ref) < tol
    assert abs(float(inv_s) - float(torch.exp(P["neuconw.deviation_network.variance"] * 10))) < 1e-4
    p4 = torch.randn(3000, 4) * 0.5
    rd, rr = port.nerf_forward(P, p4, dirs[:3000], a[:3000])
    dens, rgbn = s["nerf"](p4.cuda(), dirs[:3000].cuda(), a[:3000].cuda())
    assert rel_err(dens.cpu(), rd.detach()) < tol and rel_err(rgbn.cpu(), rr.detach()) < tol


def test_sdf_query_empty_and_tiny(P):
    s = build_system(P, synth.PathConfig(), precision="bf16x3", backend=0, chunk_rows=1024)
    assert s["renderer"].sdf(torch.zeros(0, 1, 3, device="cuda")).shape == (0, 1)
    x = torch.tensor([[[0.1, 0.2, 0.3]]], device="cuda")
    ref = port.sdf_value(P, x.cpu().reshape(1, 3)).detach()
    assert rel_err(s["renderer"].sdf(x).cpu(), ref) < RTOL


# ------------------------------------------------------------------------------------------- sampler
@pytest.mark.parametrize("case", ["det", "perturb"])
def test_sampler_vs_port(P, case):
    cfg = synth.C1 if case == "det" else synth.PathConfig(perturb=1.0, **synth.BRANDENBURG)
    R = 96
    s = build_system(P, cfg, precision="bf16x6", backend=0, chunk_rows=4096)
    batch = synth.make_rays(R, cfg, seed=21)
    noise = synth.make_perturb_noise(R, cfg.n_outside, seed=5) if case == "perturb" else None
    extras = {}
    with torch.no_grad():
        port.render(P, cfg, batch["rays"], batch["ts"], batch["label"], perturb_overwrite=-1 if noise else 0,
                    background_rgb=torch.zeros(1, 3), cos_anneal_ratio=0.5, noise=noise, extras=extras)
    r = s["renderer"]
    if noise is not None:
        r._noise_hook = lambda R_, n_, dev: (noise[0].to(dev), noise[1].to(dev))
    rays = batch["rays"].cuda()
    o = ((rays[:, 0:3] - r.origin.to("cuda").float()) / r.radius).float().contiguous()
    near, far = (rays[:, 6:7] / r.radius).float(), (rays[:, 7:8] / r.radius).float()
    with torch.no_grad():
        S, z, zo, sd, _, _ = r.sparse_sampler(o, rays[:, 3:6].contiguous(), near, far, cfg.perturb if noise else 0)
    z = z.cpu()
    assert z.shape == extras["z_vals"].shape
    assert torch.all(z[:, 1:] >= z[:, :-1])                       # sortedness
    # coarse/outside strata do not depend on the network: fp32-exact up to 1 ulp of the torch evaluation
    assert rel_err(zo.cpu(), extras["z_vals_outside"]) < 1e-6
    assert rel_err(sd.cpu(), extras["sample_dist"]) < 1e-6
    # importance samples go through the tensor-core SDF (documented: statistical agreement)
    assert rel_err(z, extras["z_vals"]) < 2e-5


# ------------------------------------------------------------------------------------------- end to end
def _check_step(P, cfg, R, precision, backend, out_tol, grad_tol, chunk_rows=2048, noise=None, pov=0):
    batch = synth.make_rays(R, cfg, seed=11)
    res_p, loss_p, grads_p = port.train_step(P, cfg, batch, perturb_overwrite=pov, noise=noise)
    s = build_system(P, cfg, precision=precision, backend=backend, chunk_rows=chunk_rows)
    res_c, loss_c, grads_c = cuda_train_step(s, cfg, batch, perturb_overwrite=pov, noise=noise)
    assert set(res_c) == set(res_p)
    for k in res_p:
        a, b = res_c[k].numpy(), res_p[k].detach().numpy()
        assert a.shape == b.shape, k
        assert rel_err(a, b) < out_tol, (k, rel_err(a, b))
    assert np.array_equal(res_c["inside_sphere"].numpy(), res_p["inside_sphere"].numpy())
    assert abs(float(loss_c) - float(loss_p)) < out_tol * abs(float(loss_p))
    gmax = max(float(g.abs().max()) for g in grads_p.values())
    for k in grads_p:
        if float(grads_p[k].abs().max()) < 1e-4 * gmax:      # gradients at the fp32 noise floor of the reference
            assert float((grads_c[k] - grads_p[k]).abs().max()) < 1e-6 * gmax + grad_tol * 1e-4 * gmax, k
            continue
        assert rel_err(grads_c[k].numpy(), grads_p[k].numpy()) < grad_tol, (k, rel_err(grads_c[k].numpy(), grads_p[k].numpy()))


def test_train_step_simt_exact(P):
    """fp32 CUDA-core GEMM backend + 3 planes: validates every hand-derived backward to ~1e-5."""
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    _check_step(P, cfg, 48, "bf16x6", 1, 2e-5, 2e-4)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16x6"])
def test_train_step_tcgen05(P, precision):
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    # parameter gradients: a ReLU pre-activation within ~1e-6 of zero can flip its 0/1 derivative between the
    # tensor-core forward and the fp32 reference, which moves single entries of the NeRF head gradients by O(1e-3)
    _check_step(P, cfg, 48, precision, 0, RTOL, 1e-2)


def test_train_step_tcgen05_c1_ragged_chunks(P):
    """C1 sample counts, rays not a multiple of the chunk -> ragged last chunk, perturbed strata, scene frame."""
    cfg = synth.PathConfig(n_samples=64, n_importance=16, up_sample_steps=2, n_outside=4, perturb=1.0, **synth.BRANDENBURG)
    noise = synth.make_perturb_noise(37, cfg.n_outside, seed=5)
    _check_step(P, cfg, 37, "bf16x3", 0, RTOL, 1e-2, chunk_rows=1024, noise=noise, pov=-1)


def test_train_step_recompute_path(P, monkeypatch):
    """NRW_RECOMPUTE=1: one slot, the backward pass recomputes each chunk's forward (minimum-memory mode)."""
    monkeypatch.setenv("NRW_RECOMPUTE", "1")
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    _check_step(P, cfg, 200, "bf16x3", 0, RTOL, 1e-2, chunk_rows=1024)


def test_train_step_bf16_fast_mode(P):
    """single-plane bf16 (north-star 'bf16 accumulate fp32'): looser, documented tolerance."""
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    batch = synth.make_rays(48, cfg, seed=11)
    res_p, loss_p, _ = port.train_step(P, cfg, batch, perturb_overwrite=0)
    s = build_system(P, cfg, precision="bf16", backend=0, chunk_rows=2048)
    res_c, loss_c, _ = cuda_train_step(s, cfg, batch, perturb_overwrite=0)
    assert rel_err(res_c["color"].numpy(), res_p["color"].detach().numpy()) < 5e-2
    assert abs(float(loss_c) - float(loss_p)) < 2e-2 * abs(float(loss_p))


@pytest.mark.parametrize("name", ["small_det", "c1_slice"])
def test_cuda_vs_reference_golden(P, name):
    """CUDA path vs tensors produced by the UNMODIFIED reference (tests/golden, oracle/make_golden.py)."""
    from oracle.make_golden import CASES, grad_probe

    cfg, n_rays, pov, rseed = CASES[name]
    G = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    batch = synth.make_rays(n_rays, cfg, seed=11)
    s = build_system(P, cfg, precision="bf16x3", backend=0, chunk_rows=2048)
    res_c, loss_c, grads_c = cuda_train_step(s, cfg, batch, perturb_overwrite=pov)
    for k, v in res_c.items():
        assert rel_err(v.numpy(), G["out." + k]) < RTOL, k
    assert abs(float(loss_c) - float(G["loss"])) < RTOL * abs(float(G["loss"]))
    z = s["renderer"].last_extras["z_vals"].cpu().numpy()
    assert rel_err(z, G["z_vals"]) < 2e-5
    gp = grad_probe(grads_c)
    big = max(float(np.abs(G[k]).max()) for k in G.files if k.startswith("gp."))
    for k, v in gp.items():
        if np.abs(G["gp." + k]).max() > 1e-3 * big:
            assert rel_err(v, G["gp." + k]) < 3e-3, k


# ------------------------------------------------------------------------------------------- full size
def test_full_size_properties():
    """BASELINE C2 shape (8192 rays x 128 samples): size-independent properties."""
    from nrw.synthetic import make_ray_batch
    from nrw.train import TrainSystem

    dev = torch.device("cuda", 0)
    sysm = TrainSystem(dev, precision="bf16x3", chunk_rows=32768)
    b = make_ray_batch(8192, seed=3, device=dev)
    sysm.renderer._noise_hook = None
    with torch.no_grad():
        torch.manual_seed(0)
        r1 = sysm.forward(b["rays"], b["ts"], b["label"])
        z1 = sysm.renderer.last_extras["z_vals"].clone()
        torch.manual_seed(0)
        r2 = sysm.forward(b["rays"], b["ts"], b["label"])
    assert z1.shape == (8192, 128) and torch.all(z1[:, 1:] >= z1[:, :-1])          # sorted sample list
    for k in ("color", "weights", "depth", "gradients"):
        assert torch.equal(r1[k], r2[k]), k                                          # forward is deterministic
    w = r1["weights"]
    assert torch.isfinite(w).all() and float(w.min()) >= 0.0
    assert float(w.sum(-1).max()) <= 1.0 + 1e-4                                     # partition of unity (<= 1)
    assert float(r1["weights_sum"].max()) <= 1.0 + 1e-4
    ins = r1["inside_sphere"]
    assert set(torch.unique(ins).tolist()) <= {0.0, 1.0}
    assert torch.isfinite(r1["color"]).all() and torch.isfinite(r1["gradient_error"]).all()
    # backward is linear in the upstream gradient: grads(2*L) == 2*grads(L)
    def grads(scale):
        for p in sysm.params:
            p.grad = None
        torch.manual_seed(0)
        res = sysm.forward(b["rays"], b["ts"], b["label"])
        loss = sum(sysm.loss(res, b["rgbs"]).values()) * scale
        loss.backward()
        return sysm.renderer.engine.last_flat_grad.clone()
    g1, g2 = grads(1.0), grads(2.0)
    assert torch.isfinite(g1).all()
    assert float((g2 - 2 * g1).abs().max()) <= 2e-3 * float(g1.abs().max())        # fp32 atomics reorder only
    # one optimiser step runs and changes the weights
    before = sysm.renderer.engine.flat.clone()
    loss = sysm.training_step(b)
    assert torch.isfinite(loss) and not torch.equal(before, sysm.renderer.engine.flat)


def test_train_step_mixed_precision(P):
    """'mixed': split-bf16 (3 products) forward -> outputs hold 1e-4; backward GEMMs in plain bf16."""
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    _check_step(P, cfg, 48, "mixed", 0, RTOL, 3e-2)
