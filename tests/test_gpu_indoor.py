"""GPU: the indoor configuration (config/train_indoor.yaml), whose background NeRF has no appearance head
(ENCODE_A_BG False: relu(views_linears.0([feature, viewPE])) -> rgb_linear).

  network backward   nrw_network_backward against fp64 autograd with injected upstream gradients, in every precision
                     mode at the floors of test_gpu_network_bwd.py (harness: util_network_bwd.py, with the
                     no-appearance NeRF's pre-activations, structural zeros and modules substituted)
  end to end         NeuconWRenderer.render + loss + backward at the indoor counts with a fine octree (injected trace
                     results, 10 boundary samples) against the CPU port
  drop-in            the reference's own NeuconWSystem built from train_indoor.yaml with the nrw patch; a reference
                     NeRF(encode_appearance=False) checkpoint through load_ckpt
  two engines        an appearance and a no-appearance engine alternating in one process"""
import argparse
import ctypes as C
import os
import warnings
from contextlib import contextmanager
from unittest import mock

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import util_network_bwd as un
from oracle import ref_import
from test_gpu_network_bwd import FLOORS, LINEARITY, MIN_COSINE, MODES, linearity_residue
from util_indoor import APP, build_indoor_system, indoor_cfg, indoor_params, noapp_port, port
from util_nrw import build_system, cuda_train_step, rel_err, synth

pytestmark = pytest.mark.gpu
NERF_KW = dict(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4], in_channels_a=48,
               in_channels_dir=27, use_viewdirs=True)

# ------------------------------------------------------------------------------------------ network backward vs fp64
# name: (R, S, n_outside, chunk_rows, recompute, variant, geometry seed), as util_network_bwd.CASES
CASES = {
    "ragged": (37, 28, 4, 1024, False, None, 12),
    "recompute": (37, 28, 4, 1024, True, None, 12),
    "dense_bg": (24, 28, 4, None, False, "dense_bg", 14),
    "outside8": (24, 34, 8, 1024, False, None, 15),     # the indoor counts: 8 + 16 samples + 10 boundary, 8 outside
}
# One exception to test_gpu_network_bwd.py's floors: with a three-product (bf16x3) forward, sv_bg_rgb of the no-appearance
# head is rgb_linear over one ReLU layer, whose sums cancel more than after the appearance head's four; on dense_bg one
# ray's background colour comes out at 6.0e-5 (H100, 700 W) where the fp32 reference is at 1.4e-5 and the floor is
# 5e-5.  bf16x6 meets the strict floors on the same ray, so the gap is the three-product forward's own rounding.
BG_RGB_FWD_FLOOR_X3 = 1e-4
DEAD_NOAPP = ("neuconw.xyz_encoding_final.", "neuconw.deviation_network.variance")
NERF_RGB_NOAPP = ("nerf.feature_linear.", "nerf.views_linears.", "nerf.rgb_linear.")


def nerf_preacts_noapp(Q, pts4, dirs, a, pre="nerf."):
    """pre-activations of the NeRF's eight point-layer ReLUs and the views_linears.0 ReLU (the `a` codes are unused)."""
    pe = port.posenc(pts4, 10)
    h, out = pe, []
    for i in range(8):
        out.append(F.linear(h, Q[f"{pre}pts_linears.{i}.weight"], Q[f"{pre}pts_linears.{i}.bias"]))
        h = F.relu(out[-1])
        if i == 4:
            h = torch.cat([pe, h], -1)
    feat = F.linear(h, Q[pre + "feature_linear.weight"], Q[pre + "feature_linear.bias"])
    out.append(F.linear(torch.cat([feat, port.posenc(dirs, 4)], -1), Q[pre + "views_linears.0.weight"],
                        Q[pre + "views_linears.0.bias"]))
    return out


def structural_zeros_noapp(case, st):
    """util_network_bwd.structural_zeros with views_linears.0 live and the background not reading the codes: the
    appearance-code gradient is exactly zero unless the colour net's rgb stream is in the set."""
    with mock.patch.multiple(un, DEAD=DEAD_NOAPP, NERF_RGB=NERF_RGB_NOAPP):
        zero = un.structural_zeros(case, st)
    if "rgb" not in st:
        zero["a_emb"] = None
    return zero


def make_engine_noapp(case, precision, backend, chunk_rows=None, recompute=False):
    """util_network_bwd.make_engine with nrw.NeRF(encode_appearance=False)."""
    import nrw
    from nrw.engine import Engine

    P = case["P"]
    neuconw = nrw.NeuconW(un.SDF_CONFIG, un.COLOR_CONFIG, dict(init_val=0.3), in_channels_a=un.N_A, encode_a=True)
    nerf = nrw.NeRF(**NERF_KW, encode_appearance=False)
    neuconw.load_state_dict({k[len("neuconw."):]: v for k, v in P.items() if k.startswith("neuconw.")})
    nerf.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")}, strict=True)
    dev = torch.device("cuda")
    neuconw, nerf = neuconw.to(dev), nerf.to(dev)
    eng = Engine(neuconw, nerf, n_vocab=un.N_VOCAB, n_a=un.N_A, precision=precision, backend=backend, chunk_rows=chunk_rows)
    eng._modules = (neuconw, nerf)
    with un._env("NRW_RECOMPUTE", "1" if recompute else "0"):
        eng.ensure(dev, case["R"], case["T"], 1, S=case["S"])
    eng.pack(dev)
    return eng


@contextmanager
def noapp_harness():
    with noapp_port(), mock.patch.multiple(un, _nerf_preacts=nerf_preacts_noapp, make_engine=make_engine_noapp):
        yield


@pytest.fixture(scope="module")
def refs():
    cache = {}

    def get(name):
        if name not in cache:
            R, S, n_o, _, _, variant, seed = CASES[name]
            with noapp_harness():
                case = un.make_case(R, S, n_o, variant, seed)      # kink masks from the no-appearance pre-activations
                case["P"] = {k: v for k, v in case["P"].items() if not k.startswith(APP)}
                cache[name] = (case, un.reference(case, torch.float64), un.reference(case, torch.float32))
        return cache[name]

    return get


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASES))
def test_noapp_network_backward_vs_fp64(name, mode, refs):
    case, (f64, g64), (f32, g32) = refs(name)
    prec, backend, kind = MODES[mode]
    _, _, _, chunk, recompute, _, _ = CASES[name]
    with noapp_harness():
        fwd, got, flats, eng = un.cuda_network(case, prec, backend, chunk, recompute)
    ffloor, gfloor = FLOORS.get(mode, (0.0, 0.0))
    fails, worst = [], (0.0, "")
    assert torch.equal(fwd["sv_z_feed"], un.z_feed(case))
    for k in f64:
        x = fwd[k].reshape(f64[k].shape)
        assert torch.isfinite(x).all(), k
        if kind == "reported":
            c = un.cosine(x, f64[k])
            if c < MIN_COSINE:
                fails.append(("fwd", k, c))
            continue
        floor = max(ffloor, BG_RGB_FWD_FLOOR_X3) if k == "sv_bg_rgb" and mode in ("bf16x3_tc", "mixed_tc") else ffloor
        e, a, bound, passed = un.judge(x, f64[k], f32[k], floor)
        print(f"[indoor-network] {name} {mode} fwd.{k}: kernel={e:.3e} fp32_ref={a:.3e} bound={bound:.3e}")
        if not passed:
            fails.append(("fwd", k, e, a, bound))
    full = g64[-1]
    unused = [n for n in eng.index if n.startswith(APP)]
    assert unused
    for st, x, r64, r32, flat in zip(un.stream_sets(case), got, g64, g32, flats):
        tag = "full" if len(st) > 1 else st[0]
        zeros = structural_zeros_noapp(case, st)
        for n in ["embedding_a.weight"] + unused:       # slots no kernel of this configuration writes
            _, off, numel = eng.index[n]
            assert not flat[off:off + numel].any(), (tag, n)
        if "bg_rgb" in st:
            assert float(x["nerf.views_linears.0.weight"].abs().max()) > 0, tag
        set_worst = (0.0, "")
        for k in r64:
            xk = x[k]
            assert torch.isfinite(xk).all(), (tag, k)
            if k in zeros:
                if un.zero_part(xk, zeros[k]).any():
                    fails.append((tag, k, "structural zero is not 0.0"))
                if zeros[k] is None:
                    continue
            if kind == "reported":
                c = un.cosine(xk, r64[k])
                if c < MIN_COSINE:
                    fails.append((tag, k, c))
                continue
            e = un.grad_err(k, xk, r64[k], full[k])
            a = un.grad_err(k, r32[k], r64[k], full[k])
            bound = max(un.ANCHOR_FACTOR * a, gfloor)
            set_worst = max(set_worst, (e, k))
            if not e <= bound:
                fails.append((tag, k, e, a, bound))
        if kind != "reported":
            print(f"[indoor-network] {name} {mode} {tag}: worst kernel error {set_worst[0]:.3e} ({set_worst[1]})")
            worst = max(worst, (set_worst[0], f"{tag}.{set_worst[1]}"))
    if prec == "bf16x6":
        bound = max(LINEARITY, un.ANCHOR_FACTOR * max(linearity_residue(g32, k) for k in full))
        for k in full:
            e = linearity_residue(got, k)
            if e > bound:
                fails.append(("linearity", k, e, bound))
    print(f"[indoor-network-worst] {name} {mode}: {worst[0]:.3e} ({worst[1]})")
    assert not fails, fails[:20]


def test_set_nerf_appearance_after_bind_is_refused(refs):
    case = refs("ragged")[0]
    with noapp_harness():
        eng = un.make_engine(case, "bf16x3", 0)
    assert eng.L.nrw_ctx_set_nerf_appearance(eng.ctx, 1) != 0
    assert b"before nrw_ctx_bind" in eng.L.nrw_last_error()


# ------------------------------------------------------------------------------------------ end to end
def install_injected_hits(renderer, hits):
    """the octree tracer replaced by injected trace results (as tests/test_gpu_parity2.py does)."""
    coarse, fine = {"tag": "coarse"}, {"tag": "fine", "voxel_size": hits["fine_voxel_sfm"]}

    def fake_trace(od, rays_o_sfm, rays_d):
        dev = rays_o_sfm.device
        if od is fine:
            return hits["surface"].to(dev), None
        return hits["sfm_near"].to(dev), hits["sfm_far"].to(dev)

    renderer._octree_near_far = fake_trace
    renderer.octree_data, renderer.fine_octree_data = coarse, fine
    renderer.nerf_far_override = True
    renderer.voxel_size = hits["voxel_size"]


@pytest.mark.parametrize("precision", ["bf16x3", "mixed"])
def test_indoor_train_step_with_fine_octree_vs_port(precision):
    """indoor counts (8 + 16 in 2 steps, 8 outside, 10 boundary samples from an injected fine octree), R = 64, against
    the port: 1e-4 on every output, the loss, and 1e-2 on every non-negligible parameter gradient (bf16x3; mixed: the
    gradients' cosine to the port's)."""
    cfg = indoor_cfg(boundary_samples=10, sample_range=8.0, **synth.BRANDENBURG)
    R = 64
    P = indoor_params()
    batch = synth.make_rays(R, cfg, seed=13)
    hits = synth.make_injected_hits(batch, cfg)
    with noapp_port():
        res_p, loss_p, grads_p = port.train_step(P, cfg, batch, perturb_overwrite=0, hits=hits)
    s = build_indoor_system(P, cfg, precision=precision, backend=0, chunk_rows=4096)
    install_injected_hits(s["renderer"], hits)
    res_c, loss_c, grads_c = cuda_train_step(s, cfg, batch, perturb_overwrite=0)
    assert res_c["weights"].shape == (R, 8 + 16 + 10 + 8)
    for k in res_p:
        a, b = res_c[k].numpy(), res_p[k].detach().numpy()
        assert a.shape == b.shape, k
        assert rel_err(a, b) < 1e-4, (k, rel_err(a, b))
    assert abs(float(loss_c) - float(loss_p)) < 1e-4 * abs(float(loss_p))
    assert set(grads_c) == set(grads_p) and not any(k.startswith(APP) for k in grads_c)
    gmax = max(float(g.abs().max()) for g in grads_p.values())
    for k in grads_p:
        if float(grads_p[k].abs().max()) < 1e-4 * gmax:
            continue
        if precision == "mixed":
            assert un.cosine(grads_c[k], grads_p[k]) > 0.99, k
        else:
            assert rel_err(grads_c[k].numpy(), grads_p[k].numpy()) < 1e-2, (k, rel_err(grads_c[k].numpy(), grads_p[k].numpy()))
    assert float(grads_c["nerf.views_linears.0.weight"].abs().max()) > 0


# ------------------------------------------------------------------------------------------ drop-in
@pytest.fixture(scope="module")
def system(tmp_path_factory):
    if not ref_import.available():
        pytest.skip("no reference copy (oracle/_ref) on this box")
    import yaml

    import nrw
    import nrw.generate_voxel as ngv
    from nrw.synthetic import sphere_shell_points

    m = ref_import.load_system()
    ns = m.ns
    ns.NeuconW, ns.NeRF, ns.NeuconWRenderer = nrw.NeuconW, nrw.NeRF, nrw.NeuconWRenderer                 # INTEGRATION.md patch
    ns.convert_to_dense, ns.gen_octree, ns.octree_to_spc = ngv.convert_to_dense, ngv.gen_octree, ngv.octree_to_spc
    root = tmp_path_factory.mktemp("scene")
    scene = dict(origin=[0.0, 0.0, 0.0], radius=1.0, sfm2gt=np.eye(4).tolist(), eval_bbx=[[-1.0] * 3, [1.0] * 3],
                 eval_bbx_detail=[[-0.6] * 3, [0.6] * 3], voxel_size=0.1, min_track_length=0)
    with open(root / "config.yaml", "w") as f:
        yaml.safe_dump(scene, f)
    config = m.get_cfg_defaults()
    config.merge_from_file(os.path.join(m.config_dir, "train_indoor.yaml"))
    config.DATASET.ROOT_DIR = str(root)
    config.NEUCONW.N_VOCAB = 64
    config.NEUCONW.UPDATE_FREQ = 1000
    config.TRAINER.LR = 1e-4
    config.TRAINER.SAVE_FREQ = 1000
    hparams = argparse.Namespace(num_gpus=1, test_batch_size=128, exp_name="indoor", num_epochs=1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sysm = m.NeuconWSystem(hparams, config, None)
    sysm.to("cuda")
    sysm.renderer.sfm_points = sphere_shell_points(0.5, 0.03, 4000, seed=1).numpy()
    sysm.renderer.scene_config = scene
    sysm.configure_optimizers()
    return m, sysm, config


def _batch(R, seed, n_vocab=64):
    b = synth.make_rays(R, synth.PathConfig(n_vocab=n_vocab), seed=seed)
    g = torch.Generator().manual_seed(seed)
    lab = torch.tensor([0.0, 2.0, 6.0, 12.0, 20.0])[torch.randint(0, 5, (R,), generator=g)]
    return {"rays": b["rays"].cuda(), "rgbs": b["rgbs"].cuda(), "ts": b["ts"].cuda(), "semantics": lab.cuda()}, lab


def test_reference_system_from_indoor_config_trains(system):
    import nrw

    m, sysm, config = system
    assert config.NEUCONW.ENCODE_A_BG is False and config.NEUCONW.RAY_MASK_LIST is None and config.NEUCONW.N_OUTSIDE == 8
    assert isinstance(sysm.nerf, nrw.NeRF) and not sysm.nerf.encode_appearance
    names = {k for k, _ in sysm.named_parameters()}
    assert "nerf.views_linears.0.weight" in names and not any(k.startswith(APP) for k in names)
    batch, lab = _batch(200, 3)
    before = {k: v.detach().clone() for k, v in sysm.named_parameters()}
    sysm.global_step = 1
    sysm.optimizer.zero_grad()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loss = sysm.training_step(batch, 0)
    assert torch.isfinite(loss) and loss.requires_grad
    loss.backward()
    assert sysm.renderer.last_extras["z_vals"].shape[0] == 200          # RAY_MASK_LIST None: no ray is dropped
    g = {k: p.grad for k, p in sysm.named_parameters()}
    for k in ("neuconw.sdf_net.lin0.weight_v", "nerf.views_linears.0.weight", "nerf.rgb_linear.weight",
              "nerf.alpha_linear.weight", "embedding_a.weight"):
        assert g[k] is not None and torch.isfinite(g[k]).all() and float(g[k].abs().max()) > 0, k
    sysm.optimizer.step()
    assert sum(int(not torch.equal(before[k], p.detach())) for k, p in sysm.named_parameters()) > 50


def test_reference_system_from_indoor_config_validates(system):
    m, sysm, config = system
    R = 300
    batch, _ = _batch(R, 5)
    vb = {"rays": batch["rays"][:, :8].unsqueeze(0), "rgbs": batch["rgbs"].unsqueeze(0), "ts": batch["ts"].unsqueeze(0),
          "semantics": batch["semantics"].unsqueeze(0), "img_wh": torch.tensor([[20, 15]])}
    sysm.global_step = 3
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        log = sysm.validation_step(vb, 1)
    assert set(log) == {"val_loss", "val_psnr"} and torch.isfinite(log["val_loss"]) and torch.isfinite(log["val_psnr"])
    torch.set_grad_enabled(True)


def test_reference_noapp_nerf_checkpoint_loads_and_reproduces_its_outputs(system, tmp_path):
    m, sysm, config = system
    ref = ref_import.load()
    torch.manual_seed(7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r_nerf = ref.NeRF(**NERF_KW, encode_appearance=False)
    path = str(tmp_path / "ref.ckpt")
    torch.save({"state_dict": {"nerf." + k: v for k, v in r_nerf.state_dict().items()}, "global_step": 1}, path)
    m.load_ckpt(sysm.nerf, path, model_name="nerf")
    assert {k: tuple(v.shape) for k, v in sysm.nerf.state_dict().items()} == \
        {k: tuple(v.shape) for k, v in r_nerf.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    n = 700
    p = torch.randn(n, 3, generator=g) * 3
    r = p.norm(dim=-1, keepdim=True).clamp_min(1.0)
    pts4 = torch.cat([p / r, 1.0 / r], -1)
    dirs = torch.randn(n, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    a = torch.randn(n, 48, generator=g)
    with torch.no_grad():
        dens_c, rgb_c = (t.cpu() for t in sysm.nerf(pts4.cuda(), dirs.cuda(), a.cuda()))
        dens_r, rgb_r = r_nerf(pts4, dirs, a)
        _, rgb_r2 = r_nerf(pts4, dirs, torch.zeros_like(a))
    assert torch.equal(rgb_r, rgb_r2)                    # the reference ignores the codes too
    assert float((dens_c.reshape(-1) - dens_r.reshape(-1)).abs().max()) < 1e-4 * float(dens_r.abs().max())
    assert float((rgb_c - rgb_r).abs().max()) < 1e-4 * float(rgb_r.abs().max())


# ------------------------------------------------------------------------------------------ two engines
def _steps(s, cfg, batches):
    return [cuda_train_step(s, cfg, b, perturb_overwrite=0) for b in batches]


def test_appearance_and_noapp_engines_alternate_in_one_process():
    """Each engine's per-ray and per-sample outputs equal, bit for bit, a run of the same engine on its own.  What float
    atomics sum in any order agrees to a tolerance instead: gradient_error (one scalar over all rays) and the loss that
    contains it to 1e-6, the gradients (weight-gradient GEMMs) to 1e-5."""
    cfg = indoor_cfg(**synth.BRANDENBURG)
    batches = [synth.make_rays(48, cfg, seed=s) for s in (21, 22)]
    mk = {"app": lambda: build_system(synth.make_params(seed=0), cfg, precision="mixed", backend=0, chunk_rows=2048),
          "noapp": lambda: build_indoor_system(indoor_params(), cfg, precision="mixed", backend=0, chunk_rows=2048)}
    both = {k: f() for k, f in mk.items()}
    mixed = {k: [] for k in mk}
    for b in batches:
        for k in mk:
            mixed[k].append(cuda_train_step(both[k], cfg, b, perturb_overwrite=0))
    del both
    for k, f in mk.items():
        alone = _steps(f(), cfg, batches)
        for (res_m, loss_m, g_m), (res_a, loss_a, g_a) in zip(mixed[k], alone):
            for key in res_a:
                if key == "gradient_error":
                    assert rel_err(res_m[key].numpy(), res_a[key].numpy()) <= 1e-6, (k, key)
                else:
                    assert torch.equal(res_m[key], res_a[key]), (k, key)
            assert abs(float(loss_m) - float(loss_a)) <= 1e-6 * abs(float(loss_a)), k
            for n in g_a:
                assert rel_err(g_m[n].numpy(), g_a[n].numpy()) <= 1e-5, (k, n)
    # the two configurations really differ in the background
    assert not torch.equal(mixed["app"][0][0]["color_bg"], mixed["noapp"][0][0]["color_bg"])
