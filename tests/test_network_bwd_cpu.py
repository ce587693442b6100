"""Checks of the network-backward harness (tests/util_network_bwd.py) that need no GPU: the case table and its
margins, the fp64 reference's second-order autograd against central differences, the structural-zero table, the
linearity of the reference and the size of the fp32 reference's error, which anchors the tolerance of
tests/test_gpu_network_bwd.py."""
import functools

import pytest
import torch

import util_network_bwd as un

GEOMETRIES = ["one_ray", "ragged", "c2_counts", "dense_bg"]      # "recompute" shares ragged's inputs
# fp32 reference error bounds, max over every stream set: every NeRF tensor sits behind the 2^9-frequency encoding of the
# point, whose fp32 rounding dominates (measured <= 3.2e-5); the SDF net, colour net and a_emb measure <= 1.1e-5.
FP32_ANCHOR_BOUND_NERF = 1e-4
FP32_ANCHOR_BOUND = 2e-5


@functools.lru_cache(maxsize=None)
def _case(name):
    return un.make_named_case(name)


@functools.lru_cache(maxsize=None)
def _refs(name):
    case = _case(name)
    return un.reference(case, torch.float64), un.reference(case, torch.float32)


def test_case_table_covers_every_case():
    assert set(un.CASES) == {"one_ray", "ragged", "c2_counts", "recompute", "dense_bg"}
    R, S, n_o, chunk, recompute, variant, _ = un.CASES["one_ray"]
    assert (R, S, n_o) == (1, 28, 0) and R * S < 128
    R, S, n_o, chunk, recompute, _, seed = un.CASES["ragged"]
    assert (R, S, n_o, chunk, recompute) == (37, 28, 4, 1024, False)
    # SDF chunks of chunk // S rays, NeRF chunks of chunk // T rays (engine.cu render_forward)
    rows = lambda T: [min(chunk // T, R - r0) * T for r0 in range(0, R, chunk // T)]
    assert rows(S) == [1008, 28] and rows(S + n_o) == [1024, 160]
    assert un.CASES["recompute"][:4] == un.CASES["ragged"][:4] and un.CASES["recompute"][4]
    assert un.geometry("recompute") == un.geometry("ragged")
    R, S, n_o = un.CASES["c2_counts"][:3]
    assert S == 128 and S + n_o == 132 and 16 <= R <= 32
    assert un.CASES["dense_bg"][5] == "dense_bg" and un.CASES["dense_bg"][2] > 0


@pytest.mark.parametrize("name", GEOMETRIES)
def test_case_margins(name):
    """inputs are finite and ordered, z_out lies behind z_vals, the kink mask keeps most rows, and the unmasked rows
    really are KINK_DELTA x rms away from every ReLU kink."""
    case = _case(name)
    R, S, T = case["R"], case["S"], case["T"]
    for k in ("o", "d", "z_vals", "z_out", "sample_dist", "a_emb"):
        assert case[k].dtype == torch.float32 and torch.isfinite(case[k]).all(), k
    assert torch.all(case["z_vals"][:, 1:] >= case["z_vals"][:, :-1])
    if case["n_outside"]:
        assert torch.all(case["z_out"][:, 1:] >= case["z_out"][:, :-1])
        assert torch.all(case["z_out"][:, 0] > case["z_vals"][:, -1])
    mc, mn = case["mask_rgb"], case["mask_bg"]
    print(f"[network-case] {name}: R={R} S={S} T={T} masked colour rows {float(mc.float().mean()):.3f} "
          f"NeRF rows {float(mn.float().mean()):.3f}")
    # measured: 9-11 % of colour rows, 80 % of NeRF rows (the point layers' 1e-3 margin)
    assert float(mc.float().mean()) <= 0.15 and float(mn.float().mean()) <= 0.85
    assert not case["ups"]["rgb"][mc].any()
    if case["n_outside"]:
        assert not case["ups"]["bg_alpha"][mn].any() and not case["ups"]["bg_rgb"][mn].any()
    pc, pn = un.preacts(case)
    for pres, keep, nerf in ((pc, ~mc.reshape(-1), False), (pn, ~mn.reshape(-1), True)):
        assert not pres or keep.sum() >= 16
        for z, delta in zip(pres, un.kink_deltas(pres, nerf)):
            rms = float(z.pow(2).mean().sqrt())
            assert float(z[keep].abs().min()) >= delta * rms


@pytest.mark.parametrize("name", GEOMETRIES)
def test_kink_margin_exceeds_fp32_preactivation_error(name):
    """every layer's kink margin is >= 10x the largest error of an fp32 evaluation of its ReLU pre-activations,
    relative to the layer's rms: a strictly checked kernel (fp32-class products) cannot cross a kink on an unmasked
    row."""
    case = _case(name)
    p64 = un.preacts(case, torch.float64)
    p32 = un.preacts(case, torch.float32)
    deltas = un.kink_deltas(p64[0], False) + un.kink_deltas(p64[1], True)
    ratio = 0.0
    for a64, a32, delta in zip(p64[0] + p64[1], p32[0] + p32[1], deltas):
        err = float((a32.double() - a64).abs().max() / a64.pow(2).mean().sqrt())
        assert err > 0
        ratio = max(ratio, err / delta)
    print(f"[network-case] {name}: largest fp32 pre-activation error / margin {ratio:.3f}")
    assert ratio <= 0.1


def test_dense_bg_straddles_the_softplus_threshold():
    """at least 10 % of the NeRF rows on each side of density 20 (the two branches of head_kernel and head_bwd)."""
    dens = un.density(_case("dense_bg"))
    above = float((dens > un.SOFTPLUS_THRESHOLD).double().mean())
    print(f"[network-case] dense_bg: share of densities > 20: {above:.3f}")
    assert 0.1 <= above <= 0.9
    assert float((un.density(_case("ragged")) > un.SOFTPLUS_THRESHOLD).double().mean()) == 0.0


def _direction(case, seed):
    g = torch.Generator().manual_seed(seed)
    Q, a = un.leaves(case, torch.float64)
    v = {k: torch.randn(t.shape, generator=g, dtype=torch.float64) for k, t in Q.items()}
    v["a_emb"] = torch.randn(a.shape, generator=g, dtype=torch.float64)
    n = sum(float(x.pow(2).sum()) for x in v.values()) ** 0.5
    return {k: x / n for k, x in v.items()}


@pytest.mark.parametrize("stream", un.STREAMS)
def test_reference_directional_derivative(stream):
    """<grad L, v> of the fp64 reference against (L(p + h v) - L(p - h v)) / 2h over every parameter and a_emb: pins
    the second-order autograd (normals, and the colour net fed by them) that every other check trusts.  The direction
    has unit norm; h = 1e-4 balances truncation and rounding (h = 1e-6 leaves ~1e-6 of rounding noise)."""
    case = un.make_case(2, 6, 2, None, 5)
    _, (grads,) = un.reference(case, torch.float64, [(stream,)])
    h = 1e-4
    for seed in (1, 2):
        v = _direction(case, seed)
        dot = sum(float((grads[k] * v[k]).sum()) for k in v)
        Q, a = un.leaves(case, torch.float64)
        with torch.no_grad():
            Qp = {k: t + h * v[k] for k, t in Q.items()}
            Qm = {k: t - h * v[k] for k, t in Q.items()}
        fd = (un.loss_value(case, (stream,), Qp, a.detach() + h * v["a_emb"])
              - un.loss_value(case, (stream,), Qm, a.detach() - h * v["a_emb"])) / (2 * h)
        print(f"[network-fd] {stream} seed {seed}: autograd {dot:.12e} difference {fd:.12e}")
        assert abs(dot) > 0
        assert abs(fd - dot) <= 1e-7 * abs(dot)


@pytest.mark.parametrize("name", GEOMETRIES)
def test_structural_zero_table_matches_fp64_autograd(name):
    """every entry of structural_zeros is exactly 0 in fp64, and every gradient it does not cover is not."""
    case = _case(name)
    (_, g64), _ = _refs(name)
    for st, r in zip(un.stream_sets(case), g64):
        zeros = un.structural_zeros(case, st)
        assert set(zeros) <= set(r)
        for k, x in r.items():
            if k in zeros:
                assert float(un.zero_part(x, zeros[k]).abs().max()) == 0.0, (st, k)
                rest = un.nonzero_part(x, zeros[k])
                assert rest.numel() == 0 or float(rest.abs().max()) > 0.0, (st, k)
            else:
                assert float(x.abs().max()) > 0.0, (st, k)


@pytest.mark.parametrize("name", GEOMETRIES)
def test_reference_backward_is_linear(name):
    (_, g64), _ = _refs(name)
    single, full = g64[:-1], g64[-1]
    for k in full:
        s = sum(g[k] for g in single)
        assert float((s - full[k]).abs().max()) <= 1e-12 * max(float(full[k].abs().max()), 1.0), k


@pytest.mark.parametrize("name", GEOMETRIES)
def test_fp32_reference_error(name):
    """the fp32 evaluation of the reference against fp64 under the tolerance rule: finite, non-zero on the full
    gradients, and below FP32_ANCHOR_BOUND (NeRF tensors: FP32_ANCHOR_BOUND_NERF; forward outputs: 1e-5), so the 4x
    anchor of the GPU test cannot open up far enough to let a wrong kernel through."""
    case = _case(name)
    (f64, g64), (f32, g32) = _refs(name)
    worst = {}
    for k in f64:
        worst["fwd." + k] = un.ray_err(f32[k], f64[k])
        assert 0 < worst["fwd." + k] <= 1e-5, (k, worst["fwd." + k])
    full = g64[-1]
    for st, r64, r32 in zip(un.stream_sets(case), g64, g32):
        zeros = un.structural_zeros(case, st)
        tag = "full" if len(st) > 1 else st[0]
        for k in r64:
            if zeros.get(k, 0) is None:
                continue
            worst[f"{tag}.{k}"] = un.grad_err(k, r32[k], r64[k], full[k])
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    print(f"[network-anchor] {name}: " + " ".join(f"{k}={v:.2e}" for k, v in top))
    for k, v in worst.items():
        bound = FP32_ANCHOR_BOUND_NERF if ".nerf." in k else FP32_ANCHOR_BOUND
        assert v == v and v <= bound, (k, v)
    assert max(v for k, v in worst.items() if k.startswith("full.")) > 0
