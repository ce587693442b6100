"""The NeuS compositing kernels (csrc/composite.cu) against render_core in fp64, through nrw_composite_forward /
nrw_composite_backward with injected per-sample inputs, at every per-lane width (CPL = 5 / 8 / 16 / 40), with and
without a background, and under each upstream gradient alone.  Tolerance rule and cases: tests/util_composite.py.

Also: determinism, the argument edges (T > 1280, R = 0), and full training steps / renders in the configurations
no other test runs (render_bg=False, trim_sphere=False, T = 196 in a training step, the reference defaults)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import util_composite as uc
from test_gpu_parity import RTOL, _check_step
from util_nrw import build_system, port, rel_err, synth

pytestmark = pytest.mark.gpu
NAMES = sorted(uc.CASES)


@pytest.fixture(scope="module")
def P():
    return synth.make_params(seed=0)


@functools.lru_cache(maxsize=4)
def _refs(name):
    case = uc.make_named_case(name)
    ups = uc.make_ups(case, seed=uc.case_seed(name))
    sets = uc.upstream_sets()
    return case, ups, uc.reference(case, torch.float64, ups, sets), uc.reference(case, torch.float32, ups, sets)


def _report(name, tag, e, a, bound):
    print(f"[composite] {name} CPL={uc.cpl(uc.CASES[name][1] + uc.CASES[name][2])} {tag}: kernel={e:.3e} "
          f"fp32_ref={a:.3e} bound={bound:.3e}")


# --------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("name", NAMES)
def test_forward_vs_fp64(name):
    case, ups, (f64, _), (f32, _) = _refs(name)
    got, _ = uc.cuda_composite(case)
    ok = case["ok"]
    fails = []
    for k in uc.FWD_KEYS:
        x = got[k].reshape(f64[k].shape)
        e, a, bound, passed = uc.judge(x, f64[k], f32[k], uc.FWD_FLOOR, ok)
        _report(name, "fwd." + k, e, a, bound)
        if not passed:
            fails.append((k, e, a, bound))
    assert not fails, fails
    # masks: exact; the gradients output is a copy of the injected normals
    assert torch.equal(got["inside_sphere"], f64["inside_sphere"].float())
    assert float(got["sv_relax_sum"]) == uc.relax_count(case)
    assert torch.equal(got["gradients"], case["normals"])


# --------------------------------------------------------------------------------------------------- backward
@pytest.mark.parametrize("name", NAMES)
def test_backward_vs_fp64_one_upstream_at_a_time(name):
    case, ups, (_, g64), (_, g32) = _refs(name)
    sets = uc.upstream_sets()
    _, got = uc.cuda_composite(case, ups, sets)
    ok = case["ok"]
    fails = []
    for st, x, r64, r32 in zip(sets, got, g64, g32):
        tag = "all" if len(st) > 1 else st[0]
        for k in uc.BWD_KEYS:
            assert torch.isfinite(x[k]).all(), (tag, k)
            e, a, bound, passed = uc.judge(x[k].reshape(r64[k].shape), r64[k], r32[k], uc.bwd_floor(case, st, k), ok,
                                           g64[-1][k])
            _report(name, f"bwd.{tag}.{k}", e, a, bound)
            if not passed:
                fails.append((tag, k, e, a, bound))
        if not case["n_outside"]:
            assert not x["d_bg_alpha"].any() and not x["d_bg_rgb"].any(), tag
    assert not fails, fails


# --------------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("name", ["c5_T160_bg_notrim_sat", "c8_T256_nobg_sat", "c16_T512_bg32", "c40_T1280_bg32_notrim"])
def test_deterministic(name):
    """bit-identical results over two runs, except the float atomicAdd reductions over rays (gradient_error,
    grad_inv_s)."""
    case, ups, _, _ = _refs(name)
    sets = [uc.UPSTREAM]
    f1, b1 = uc.cuda_composite(case, ups, sets)
    f2, b2 = uc.cuda_composite(case, ups, sets)
    for k in f1:
        if k != "gradient_error":
            assert torch.equal(f1[k], f2[k]), k
    for k in uc.BWD_KEYS:
        if k != "grad_inv_s":
            assert torch.equal(b1[0][k], b2[0][k]), k


# --------------------------------------------------------------------------------------------------- argument edges
def _raw_call(R, S, n_o):
    """forward + backward status codes for R rays of S + n_o samples (buffers sized for the shape)."""
    from nrw import _lib
    from nrw._lib import RenderGrads
    from nrw.engine import _io_struct, make_render_cfg

    L = _lib.lib()
    T = S + n_o
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device="cuda")
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device="cuda")
    t = dict(o=f(R, 3), d=f(R, 3), z_vals=f(R, S), z_out=f(R, n_o), sample_dist=f(R), a_emb=f(R, 48), inv_s=f(1) + 20,
             color=f(R, 3), color_sphere=f(R, 3), color_bg=f(R, 3), cdf=f(R, S), gradients=f(R, S, 3), weights=f(R, T),
             weights_sum=f(R), inside_sphere=f(R, S), depth=f(R), normals=f(R, 3), gradient_error=nan(1),
             sv_sdf=f(R, S), sv_rgb=f(R, S, 3), sv_bg_alpha=f(R, T), sv_bg_rgb=f(R, T, 3), sv_z_feed=f(R, T),
             sv_relax_sum=nan(1))
    nrm = f(R, S, 3)
    rcfg = make_render_cfg(R, S, n_o, 0.3, None, True)
    io = _io_struct(t)
    scratch = nan(2)
    st_f = L.nrw_composite_forward(C.byref(rcfg), C.byref(io), _lib.ptr(t["sv_sdf"]), _lib.ptr(nrm),
                                   _lib.ptr(t["sv_rgb"]), _lib.ptr(t["sv_bg_alpha"]), _lib.ptr(t["sv_bg_rgb"]),
                                   _lib.ptr(scratch), _lib.stream_ptr())
    torch.cuda.synchronize()
    gr = RenderGrads()
    ups = {k: f(1) for k in ("g_color", "g_gradient_error")}
    gr.g_color, gr.g_gradient_error = _lib.ptr(ups["g_color"]), _lib.ptr(ups["g_gradient_error"])
    g_invs = nan(1)
    gr.grad_inv_s = _lib.ptr(g_invs)
    d = [f(R, S), f(R, S, 3), f(R, S, 3), f(R, T), f(R, T, 3)]
    st_b = L.nrw_composite_backward(C.byref(rcfg), C.byref(io), C.byref(gr), _lib.ptr(nrm),
                                    *[_lib.ptr(x) for x in d], _lib.stream_ptr())
    torch.cuda.synchronize()
    return st_f, st_b, t, g_invs


def test_more_than_1280_samples_per_ray_is_rejected():
    from nrw import _lib

    st_f, st_b, _, _ = _raw_call(1, 1249, 32)                   # T = 1281
    assert st_f == -1 and st_b == -1                             # NRW_ERR_ARG, checked before any launch
    assert b"1280" in _lib.lib().nrw_last_error()


def test_zero_rays():
    """R = 0: no per-ray launch; gradient_error and sv_relax_sum are finalised to 0 and grad_inv_s is zeroed."""
    st_f, st_b, t, g_invs = _raw_call(0, 24, 4)
    assert st_f == 0 and st_b == 0
    assert float(t["gradient_error"]) == 0.0 and float(t["sv_relax_sum"]) == 0.0
    assert float(g_invs) == 0.0


# --------------------------------------------------------------------------------------------------- end to end
def test_train_step_without_background(P):
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4, render_bg=False)
    _check_step(P, cfg, 48, "bf16x3", 0, RTOL, 1e-2)


def test_train_step_untrimmed_background(P):
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4, trim_sphere=False)
    _check_step(P, cfg, 48, "bf16x3", 0, RTOL, 1e-2)


def test_train_step_cpl8_kernel(P):
    """64 + 128 samples in 4 rounds + 4 outside: T = 196, the 8-per-lane compositing kernel in a training step."""
    cfg = synth.PathConfig(n_samples=64, n_importance=128, up_sample_steps=4, n_outside=4)
    assert uc.cpl(cfg.n_samples + cfg.n_importance + cfg.n_outside) == 8
    _check_step(P, cfg, 32, "bf16x3", 0, RTOL, 1e-2)


@pytest.mark.parametrize("precision,backend", [("bf16x3", 0), ("bf16x6", 1)])
def test_render_at_reference_defaults(P, precision, backend):
    """512 + 512 samples in 4 rounds + 32 outside (the reference's defaults): T = 1056, the 40-per-lane kernel.
    Forward only, against the fp32 oracle, with the tensor-core network (bf16x3) and the fp32 CUDA-core one."""
    cfg = synth.PathConfig(n_samples=512, n_importance=512, up_sample_steps=4, n_outside=32)
    assert uc.cpl(cfg.n_samples + cfg.n_importance + cfg.n_outside) == 40
    R = 8
    batch = synth.make_rays(R, cfg, seed=11)
    extras = {}
    with torch.no_grad():
        res_p = port.render(P, cfg, batch["rays"], batch["ts"], batch["label"], perturb_overwrite=0,
                            background_rgb=torch.zeros(1, 3), cos_anneal_ratio=cfg.cos_anneal_ratio, extras=extras)
    s = build_system(P, cfg, precision=precision, backend=backend, chunk_rows=16384)
    dev = torch.device("cuda")
    b = {k: v.to(dev) for k, v in batch.items()}
    with torch.no_grad():
        res_c = s["renderer"].render(b["rays"], b["ts"], b["label"], perturb_overwrite=0,
                                     background_rgb=torch.zeros([1, 3], device=dev),
                                     cos_anneal_ratio=cfg.cos_anneal_ratio)
    assert res_c["weights"].shape == (R, 1056)
    assert set(res_c) == set(res_p)
    errs = {}
    for k in res_p:
        a, ref = res_c[k].detach().cpu().numpy(), res_p[k].detach().numpy()
        assert a.shape == ref.shape, k
        errs[k] = rel_err(a, ref)
    # bf16x3 only: weights_sum, depth, color_sphere are sums over the ~1e3 samples inside the unit sphere, where the
    # synthetic scene puts little weight (weights_sum and color_sphere ~1e-2), and the tensor-core network's rounding
    # of sdf / rgb accumulates to 1.6e-4 - 2.2e-4 of these small values (measured on an H100).  The fp32 CUDA-core
    # network (bf16x6, backend 1) runs the same sampler and compositing and is held to RTOL on every output.
    tol = dict(weights_sum=5e-4, depth=5e-4, color_sphere=5e-4) if backend == 0 else {}
    print(f"[composite] defaults render {precision} rel_err: " + " ".join(f"{k}={v:.2e}" for k, v in sorted(errs.items())))
    bad = {k: v for k, v in errs.items() if not v < tol.get(k, RTOL)}
    assert not bad, bad
    z = s["renderer"].last_extras["z_vals"].cpu().numpy()
    assert rel_err(z, extras["z_vals"].numpy()) < 2e-5
    assert np.array_equal(res_c["inside_sphere"].cpu().numpy(), res_p["inside_sphere"].numpy())
