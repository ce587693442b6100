"""GPU: appearance-code fitting on a cached appearance-free render prefix (csrc/appearance.cu, nrw/appearance.py) and the
eval split of PhototourismDataset.

  forward      AppearanceCache(...)(codes) against renderer.render(...)["color"] with the same codes in embedding_a, for
               bf16x6 on the CUDA cores, bf16x3 and mixed on the tensor cores; both NeRF variants, background_rgb given
               and None, n_outside 0 and > 0, a fine octree, several chunks with a ragged last 128-row tile
  gradient     grad_a_emb against fp64 autograd of the port (render_core_outside + render_core, the codes requiring
               grad) for a random upstream g_color, per ray; and against nrw_render_backward's grad_a_emb
  interleaving renders, SDF queries and render backwards between prepare, forward and backward change nothing
  fitting      codes fitted from zeros to a random a* reach a loss threshold; networks and other rows stay bit-identical;
               two runs are bit-identical; evaluate_held_out end to end
  eval split   rows equal RayGenerator's, halves by pixel column
  errors       every status of the four entries

Tolerances (FWD_TOL, GRAD_FLOOR) were measured on an H100 80GB HBM3 at a 700 W power limit; see their comments."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import util_cache
from util_indoor import build_indoor_system, indoor_cfg, indoor_params, noapp_port
from util_nrw import build_system, port, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

MODES = {"bf16x6_simt": ("bf16x6", 1), "bf16x3": ("bf16x3", 0), "mixed": ("mixed", 0)}
# max |cache colour - render colour| over every case of test_forward_equals_render.  The two differ only in how
# static_linear_0 forms W [x | a]: one GEMM over split-bf16 operands, or the fp32 pre-activation W [x | 0] + b plus an fp32
# product W_a a.  Measured maxima (H100 80GB HBM3, 700 W): 6.0e-8 in bf16x6 on the CUDA cores, 1.4e-7 in bf16x3 and
# mixed; the tolerances keep a margin of about 7x.
FWD_TOL = {"bf16x6_simt": 4e-7, "bf16x3": 1e-6, "mixed": 1e-6}
# grad_a_emb per ray: max|x - ref| / (max|ref| + GRAD_FLOOR_REL max over all rays |ref|), against fp64 autograd and against
# nrw_render_backward, below GRAD_TOL of the mode.  The batch-relative floor keeps rays whose code gradient nearly cancels
# from being judged on their rounding noise alone.  Measured maxima over both scenes against fp64 (H100 80GB HBM3, 700 W):
# 2.4e-5 in bf16x6 on the CUDA cores, 3.1e-3 in bf16x3, 6.9e-3 in mixed (its backward GEMMs run on one bf16 plane);
# against nrw_render_backward at most 1.6e-3.
GRAD_FLOOR_REL = 1e-2
GRAD_TOL = {"bf16x6_simt": 2e-4, "bf16x3": 2e-2, "mixed": 5e-2}


def _install_hits(renderer, hits):
    """the octree tracer replaced by injected trace results (tests/test_gpu_parity2.py)"""
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


def _case(kind, mode, R=101, chunk_rows=1024, seed=21):
    """(system, cfg, batch on the device, P): 16 + 8 samples in 2 rounds; `kind` picks the variant."""
    precision, backend = MODES[mode]
    if kind == "indoor":
        cfg = indoor_cfg(n_outside=4)
        P = indoor_params()
        s = build_indoor_system(P, cfg, precision=precision, backend=backend, chunk_rows=chunk_rows)
    else:
        kw = dict(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=0 if kind == "nobg" else 4)
        if kind == "fine":
            kw.update(boundary_samples=10, sample_range=8.0, **synth.BRANDENBURG)
        cfg = synth.PathConfig(**kw)
        P = synth.make_params(seed=0)
        s = build_system(P, cfg, precision=precision, backend=backend, chunk_rows=chunk_rows)
    batch = synth.make_rays(R, cfg, seed=seed)
    if kind == "fine":
        _install_hits(s["renderer"], synth.make_injected_hits(batch, cfg))
    return s, cfg, {k: v.to(DEV) for k, v in batch.items()}, P


FWD_CASES = [("app", torch.zeros(3)), ("app", None), ("nobg", torch.tensor([0.2, 0.5, 0.9])), ("indoor", torch.zeros(3)),
             ("fine", None)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("kind,bg", FWD_CASES, ids=[f"{k}-{'bg' if b is not None else 'nobgrgb'}" for k, b in FWD_CASES])
def test_forward_equals_render(mode, kind, bg):
    from nrw.appearance import AppearanceCache

    s, cfg, b, _ = _case(kind, mode)
    r = s["renderer"]
    bgd = None if bg is None else bg.to(DEV)
    with torch.no_grad():
        ref = r.render(b["rays"], b["ts"], None, perturb_overwrite=0, background_rgb=bgd)["color"]
        cache = AppearanceCache(r, b["rays"], b["ts"], background_rgb=bgd)
        got = cache(s["emb"].weight[b["ts"]])
    torch.cuda.synchronize()
    err = float((got - ref).abs().max())
    print(f"forward {mode} {kind} bg={bg is not None}: max err {err:.3e}")
    assert torch.isfinite(got).all()
    assert err < FWD_TOL[mode], (mode, kind, err)


def _fp64_color(P, cache, a, cfg, bg):
    """color of the port in fp64 on the cache's samples, differentiable in the per-ray codes a"""
    o, d, z, zo, sd, _ = (t.detach().double().cpu() for t in cache._inputs)
    Q = {k: v.double() for k, v in P.items()}
    sd = sd.reshape(-1, 1)
    bg_alpha = bg_rgb = None
    if cache.n_outside > 0:
        zf, _ = torch.sort(torch.cat([z, zo], -1), -1)
        bg_alpha, bg_rgb = port.render_core_outside(Q, o, d, zf, sd, a)
    return port.render_core(Q, cfg, o, d, z, sd, a, 0.0, bg_alpha, bg_rgb, bg)["color"]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("kind", ["app", "indoor"])
def test_gradient_vs_fp64_and_render_backward(mode, kind):
    from nrw.appearance import AppearanceCache

    s, cfg, b, P = _case(kind, mode, R=37)
    r = s["renderer"]
    bg = torch.zeros(3, dtype=torch.float64)
    codes = s["emb"].weight[b["ts"]].detach().clone()
    g = torch.Generator().manual_seed(5)
    g_color = torch.randn(37, 3, generator=g)
    cache = AppearanceCache(r, b["rays"], b["ts"], background_rgb=bg.float().to(DEV))
    a = codes.clone().requires_grad_(True)
    (cache(a) * g_color.to(DEV)).sum().backward()
    got = a.grad.cpu()
    a64 = codes.double().cpu().requires_grad_(True)
    ctx = noapp_port() if kind == "indoor" else _null()
    with ctx:
        col = _fp64_color(P, cache, a64, cfg, bg)
    (ref,) = torch.autograd.grad((col * g_color.double()).sum(), a64)
    err = _grad_err(got, ref)
    print(f"gradient {mode} {kind}: ray_err {err:.3e}, max|ref| {float(ref.abs().max()):.3e}")
    assert err < GRAD_TOL[mode], (mode, kind, err)
    # nrw_render_backward's code gradient for the same upstream
    leaf = codes.clone().requires_grad_(True)
    emb = r.embeddings
    r.embeddings = {"a": lambda ts: leaf}
    try:
        out = r.render(b["rays"], b["ts"], None, perturb_overwrite=0, background_rgb=bg.float().to(DEV))
        (g_r,) = torch.autograd.grad((out["color"] * g_color.to(DEV)).sum(), leaf)
    finally:
        r.embeddings = emb
    err_r = _grad_err(got, g_r.cpu().double())
    print(f"gradient {mode} {kind}: vs render backward {err_r:.3e}")
    assert err_r < GRAD_TOL[mode], (mode, kind, err_r)


def _grad_err(x, ref):
    x, ref = x.double(), ref.double()
    if not torch.isfinite(x).all():
        return float("inf")
    den = ref.abs().amax(1) + GRAD_FLOOR_REL * ref.abs().max()
    return float(((x - ref).abs().amax(1) / den).max())


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def test_interleaving_changes_nothing():
    from nrw.appearance import AppearanceCache

    s, cfg, b, _ = _case("app", "mixed", R=101)
    r, emb = s["renderer"], s["emb"]
    codes = emb.weight[b["ts"]].detach().clone()
    g_color = torch.randn(101, 3, device=DEV)

    def step(cache, between=lambda: None):
        a = codes.clone().requires_grad_(True)
        col = cache(a)
        between()
        (col * g_color).sum().backward()
        return col.detach().clone(), a.grad.clone()

    clean = AppearanceCache(r, b["rays"], b["ts"])
    c0, g0 = step(clean)
    b2 = {k: v.to(DEV) for k, v in synth.make_rays(77, cfg, seed=3).items()}

    def noise():
        out = r.render(b2["rays"], b2["ts"], None, perturb_overwrite=0)
        r.sdf(torch.rand(5000, 1, 3, device=DEV) - 0.5)
        (out["color"].sum() + out["depth"].sum()).backward()

    cache = AppearanceCache(r, b["rays"], b["ts"])
    noise()
    c1, g1 = step(cache, noise)
    assert torch.equal(c0, c1) and torch.equal(g0, g1)
    # render -> appearance step -> render backward == render -> render backward (parameters)
    params = [p for p in list(s["neuconw"].parameters()) + list(s["nerf"].parameters())]

    def grads(mid):
        for p in params:
            p.grad = None
        out = r.render(b2["rays"], b2["ts"], None, perturb_overwrite=0)
        mid()
        out["color"].sum().backward()
        return [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in params]

    ref = grads(lambda: None)
    got = grads(lambda: step(cache))
    for x, y in zip(got, ref):
        assert float((x - y).abs().max()) <= 1e-4 * float(y.abs().max()) + 1e-12


def _fit_setup(seed=3):
    s, cfg, b, _ = _case("app", "mixed", R=512, chunk_rows=8192)
    r, emb = s["renderer"], s["emb"]
    ts = torch.full((512,), 7, dtype=torch.long, device=DEV)
    ts[256:] = 9
    a_star = torch.randn(2, emb.embedding_dim, generator=torch.Generator().manual_seed(seed)).to(DEV)
    with torch.no_grad():
        emb.weight[7], emb.weight[9] = a_star[0], a_star[1]
        target = r.render(b["rays"], ts, None, perturb_overwrite=0)["color"]
        emb.weight[7] = 0
        emb.weight[9] = 0
    return s, b, ts, target


# colour loss after 60 Adam steps at lr 0.05 from zero codes: measured 0.0080 before, 0.0008 after (H100 80GB HBM3, 700 W)
FIT_LOSS_MAX = 0.002


def test_fit_reaches_target_and_touches_only_its_rows():
    from nrw.appearance import AppearanceCache, color_loss, fit_appearance

    s, b, ts, target = _fit_setup()
    r, emb = s["renderer"], s["emb"]
    before = {k: v.detach().clone() for k, v in list(s["neuconw"].state_dict().items()) + list(s["nerf"].state_dict().items())}
    w0 = emb.weight.detach().clone()
    loss0 = float(color_loss(AppearanceCache(r, b["rays"], ts)(emb.weight[ts].detach()), target))
    codes = fit_appearance(r, b["rays"], ts, target, steps=60, lr=0.05)
    loss = float(color_loss(AppearanceCache(r, b["rays"], ts)(emb.weight[ts].detach()), target))
    print(f"fit: loss {loss0:.4f} -> {loss:.4f}")
    assert loss < FIT_LOSS_MAX and loss < 0.5 * loss0
    after = dict(list(s["neuconw"].state_dict().items()) + list(s["nerf"].state_dict().items()))
    assert all(torch.equal(before[k], after[k]) for k in before)
    other = torch.ones(emb.num_embeddings, dtype=torch.bool, device=DEV)
    other[[7, 9]] = False
    assert torch.equal(emb.weight[other], w0[other])
    assert torch.equal(emb.weight[[7, 9]], codes)
    # the same run again: bit-identical codes
    with torch.no_grad():
        emb.weight[7] = 0
        emb.weight[9] = 0
    again = fit_appearance(r, b["rays"], ts, target, steps=60, lr=0.05)
    assert torch.equal(codes, again)


@pytest.fixture(scope="module")
def scene_dir(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("appearance") / "synth_scene")
    return util_cache.write_scene(root, n_train=4, n_test=2, n_points=3000, seed=0)


def test_eval_split_rows_and_halves(scene_dir):
    from nrw.phototourism import PhototourismDataset, RayGenerator

    ds = PhototourismDataset(scene_dir["root"], split="eval", img_downscale=2, semantic_map_path="semantic_maps", device=0)
    s = ds.scene
    assert len(ds) == len(ds.img_ids_test) == 2
    assert all(s.splits[i] == "test" for i in ds.img_ids_test)
    gen = RayGenerator(s, DEV, True, "semantic_maps", use_voxel=False, bounds=ds.gen.bounds)
    for idx, id_ in enumerate(ds.img_ids_test):
        smp = ds[idx]
        img, sem = gen.decode(id_)
        rows, rgbs, _ = gen.run(id_, img, sem)
        h, w = img.shape[0], img.shape[1]
        assert smp["img_wh"].tolist() == [w, h]
        assert torch.equal(smp["rays"], rows[:, :8].cpu()) and torch.equal(smp["rgbs"], rgbs.cpu())
        assert (smp["ts"] == id_).all() and (smp["ts_train"] == id_).all() and (smp["ts_eval"] == id_).all()
        x = torch.arange(h * w) % w
        left = x < w // 2
        assert torch.equal(smp["rays_train"], smp["rays"][left]) and torch.equal(smp["rays_eval"], smp["rays"][~left])
        assert torch.equal(smp["rgbs_train_gt"], smp["rgbs"][left]) and torch.equal(smp["rgbs_eval_gt"], smp["rgbs"][~left])
        assert smp["rays_train"].shape[0] == h * (w // 2) and smp["rays_eval"].shape[0] == h * (w - w // 2)
        assert smp["image_name"] == s.image_paths[id_]
        assert torch.equal(smp["extrinsic"], torch.FloatTensor(s.poses[s.img_ids.index(id_)]))


def test_evaluate_held_out_end_to_end(scene_dir):
    import yaml

    from nrw.appearance import evaluate_held_out
    from nrw.phototourism import PhototourismDataset

    ds = PhototourismDataset(scene_dir["root"], split="eval", img_downscale=4, semantic_map_path="semantic_maps", device=0)
    with open(os.path.join(scene_dir["root"], "config.yaml")) as f:
        conf = yaml.load(f, Loader=yaml.FullLoader)
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4, n_vocab=64,
                           origin=tuple(conf.get("origin", (0.0, 0.0, 0.0))), radius=float(conf.get("radius", 1.0)))
    s = build_system(synth.make_params(seed=0, n_vocab=64), cfg, precision="mixed", backend=0, chunk_rows=65536)
    res = evaluate_held_out(s["renderer"], ds, steps=3, lr=0.01, n_fit_rays=256, seed=0)
    print("evaluate_held_out:", res)
    assert len(res["psnr"]) == 2 and all(np.isfinite(res["psnr"])) and np.isfinite(res["mean_psnr"])


def test_error_statuses():
    from nrw import _lib
    from nrw.engine import PRECISIONS, make_render_cfg

    L = _lib.lib()
    s, cfg, b, _ = _case("app", "mixed", R=8)
    eng = s["renderer"].engine
    R, S, n_o = 8, 24, 4
    rcfg = make_render_cfg(R, S, n_o, 0.0, None, True)
    f = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=DEV)
    o, d, z, zo, sd, inv_s = f(R, 3), f(R, 3), f(R, S), f(R, n_o), f(R), f(1)
    need = int(L.nrw_appearance_cache_bytes(eng.ctx, R, S, n_o))
    buf = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    cp = C.c_void_p((buf.data_ptr() + 255) // 256 * 256)
    p = _lib.ptr
    st = _lib.stream_ptr()
    prep = lambda ctx, cache, nbytes, cfg_=rcfg, zz=z: L.nrw_appearance_prepare(ctx, C.byref(cfg_), p(o), p(d), p(zz), p(zo), p(sd),
                                                                          p(inv_s), cache, nbytes, st)
    # a context that was never bound
    raw = C.c_void_p()
    assert L.nrw_ctx_create(C.byref(raw), PRECISIONS["mixed"], 0, cfg.n_vocab, 48) == 0
    assert prep(raw, cp, need) == -4
    L.nrw_ctx_destroy(raw)
    # bound for a forward only: prepare and forward work, backward is refused
    eng.ensure(DEV, R, S + n_o, 0)
    eng.pack(DEV)
    assert prep(eng.ctx, cp, need - 1) == -3
    assert prep(eng.ctx, None, need) == -1
    assert prep(eng.ctx, cp, need, zz=None) == -1
    bad = make_render_cfg(0, S, n_o, 0.0, None, True)
    assert prep(eng.ctx, cp, need, cfg_=bad) == -1
    assert int(L.nrw_appearance_cache_bytes(eng.ctx, 0, S, n_o)) == -1
    assert prep(eng.ctx, cp, need) == 0
    a, col, g, ga = f(R, 48), f(R, 3), f(R, 3), f(R, 48)
    assert L.nrw_appearance_forward(eng.ctx, cp, p(a), p(col), st) == 0
    assert L.nrw_appearance_forward(eng.ctx, cp, None, p(col), st) == -1
    assert L.nrw_appearance_backward(eng.ctx, cp, p(a), p(g), p(ga), st) == -4
    assert L.nrw_appearance_backward(eng.ctx, cp, p(a), None, p(ga), st) == -1
    # a cache address this context never prepared
    other = C.c_void_p(cp.value + 256)
    assert L.nrw_appearance_forward(eng.ctx, other, p(a), p(col), st) == -4
    torch.cuda.synchronize()
