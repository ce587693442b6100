"""Checks of the compositing harness (tests/util_composite.py) that need no GPU: the case table's coverage, the
generator's margins and ray kinds, the fp64 reference's gradients (gradcheck, linearity) and the size of the fp32
reference's error, which anchors the tolerance of tests/test_gpu_composite.py."""
import functools

import pytest
import torch

import util_composite as uc


@functools.lru_cache(maxsize=None)
def _refs(name):
    case = uc.make_named_case(name)
    ups = uc.make_ups(case, seed=uc.case_seed(name))
    sets = uc.upstream_sets()
    return case, uc.reference(case, torch.float64, ups, sets), uc.reference(case, torch.float32, ups, sets)


def test_case_table_covers_every_setting():
    rows = list(uc.CASES.values())
    T = {S + n for _, S, n, *_ in rows}
    assert {28, 160, 161, 256, 257, 512, 513, 1056, 1280} <= T
    assert {0, 4, 32} <= {r[2] for r in rows}
    assert {0, 1} <= {r[5] for r in rows}
    assert {None, "zeros", "color"} <= {r[6] for r in rows}
    assert {0.0, 0.3, 1.0} <= {r[4] for r in rows}
    assert {1.0, 20.0, 1e3, 1e4} <= {r[3] for r in rows}
    assert {1, 37, 300} <= {r[0] for r in rows}
    for c in (5, 8, 16, 40):                                      # every kernel width with and without a background
        assert {r[2] > 0 for r in rows if uc.cpl(r[1] + r[2]) == c} == {True, False}, c
    # trim_sphere only matters with a background: both values must run with one
    assert {r[5] for r in rows if r[2] > 0} == {0, 1}
    assert len(rows) >= 20


@pytest.mark.parametrize("name", sorted(uc.CASES))
def test_case_generation_and_margins(name):
    case = uc.make_named_case(name)
    R, S, T = case["R"], case["S"], case["T"]
    excluded = int((~case["ok"]).sum())
    print(f"[composite-case] {name}: R={R} S={S} T={T} CPL={uc.cpl(T)} excluded rays={excluded}")
    assert excluded <= 0.01 * R
    m = uc.margins(case)
    assert all(m.values()), m
    assert case["z_vals"].shape == (R, S) and case["normals"].shape == (R, S, 3) and case["rgb"].shape == (R, S, 3)
    if case["n_outside"]:
        assert case["bg_alpha"].shape == (R, T) and case["bg_rgb"].shape == (R, T, 3)
        # the background leaves the surface visible: merged transmittance at the first inside sample
        tr = uc.bg_transmittance(case)
        print(f"[composite-case] {name}: min background transmittance at the sphere {float(tr.nan_to_num(1.0).min()):.3f}")
        assert float(tr.nan_to_num(1.0).min()) >= 0.1
    else:
        assert case["bg_alpha"] is None and case["bg_rgb"] is None
    for t in (case["o"], case["d"], case["z_vals"], case["sdf"], case["normals"], case["rgb"]):
        assert t.dtype == torch.float32 and torch.isfinite(t).all()
    assert torch.all(case["z_vals"][:, 1:] >= case["z_vals"][:, :-1])
    dist, mid, pn = uc._mid_pn(case["o"], case["d"], case["z_vals"], case["sample_dist"])
    kind = case["kind"]
    inside, relax = pn < 1.0, pn < 1.2
    if R >= uc.N_KINDS:
        assert set(kind.tolist()) == set(range(uc.N_KINDS))
    for r in range(R):
        k = int(kind[r])
        if k in (0, 3):
            assert inside[r].any() and (case["sdf"][r] > 0).any() and (case["sdf"][r] < 0).any()
        if k == 1:
            assert not relax[r].any()
        if k == 2:
            assert case["sdf"][r, 0] < 0 and (case["sdf"][r, int(case["pinned"][r]):] > 0).any()
        if k == 3:
            assert (dist[r] == 0).any()
        if k == 4:
            assert (relax[r] & ~inside[r]).any()


def _tiny(bg):
    return uc.make_case(2, 6, 2 if bg else 0, 20.0, 0.3, 1, "color", seed=5)


@pytest.mark.parametrize("bg", [True, False])
def test_reference_gradcheck(bg):
    """the seam differentiates through everything the kernel differentiates: all six inputs (four without a
    background), every differentiable output."""
    case = _tiny(bg)
    assert all(uc.margins(case).values())
    lv = uc.make_leaves(case, torch.float64)
    names = [n for n in uc.LEAVES if lv[n] is not None]
    assert len(names) == (6 if bg else 4)

    def f(*xs):
        out = uc.render_leaves(case, dict(lv, **dict(zip(names, xs))), torch.float64)
        return tuple(out[k] for k in uc.UPSTREAM if out[k].requires_grad)

    assert torch.autograd.gradcheck(f, tuple(lv[n] for n in names), eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("name", ["c5_T28_bg", "c5_T28_nobg", "c8_T256_bg32", "c16_T257_bg_notrim_sat",
                                  "c40_T513_nobg_R1_sat"])
def test_reference_backward_is_linear(name):
    _, (_, g64), _ = _refs(name)
    single, together = g64[:-1], g64[-1]
    for k in uc.BWD_KEYS:
        s = sum(g[k] for g in single)
        scale = float(together[k].abs().max()) if together[k].numel() else 0.0
        assert float((s - together[k]).abs().max() if s.numel() else 0.0) <= 1e-12 * max(scale, 1.0), k


@pytest.mark.parametrize("name", sorted(uc.CASES))
def test_fp32_reference_error(name):
    """the fp32 evaluation of the reference against fp64: finite, non-zero, and small enough that the 4x anchor of
    the GPU tests is neither reduced to its floor nor toothless.

    Bounds: 1e-3 for every forward output and for the gradients under all ten upstream gradients together, 2.5e-3
    under a single upstream gradient (so no GPU bound, 4x this, exceeds 1e-2).  One named exception, 2e-2: d_sdf under
    weights, weights_sum or normals alone at inv_s >= 1e3.  There the ray is opaque behind its surface and that
    gradient at the surface sample is the residue of suffix terms ~1e4 times larger (dA = g*T - (later g*w) /
    (1 - alpha + 1e-7)), of which fp32 keeps ~1e-7; measured 1.5e-2 (c5_T160_bg_notrim_sat, weights_sum),
    1.1e-2 (c16_T512_bg32, weights), 3.3e-3 (c16_T512_bg32, normals)."""
    case, (f64, g64), (f32, g32) = _refs(name)
    ok = case["ok"]
    worst, bound = {}, {}
    for k in uc.FWD_KEYS:
        worst["fwd." + k] = uc.ray_err(f32[k], f64[k], ok)
        bound["fwd." + k] = 1e-3
    for st, r64, r32 in zip(uc.upstream_sets(), g64, g32):
        tag = "all" if len(st) > 1 else st[0]
        for k in uc.BWD_KEYS:
            worst[f"bwd.{tag}.{k}"] = uc.ray_err(r32[k], r64[k], ok, g64[-1][k])
            residue = (k == "d_sdf" and tag in ("weights", "weights_sum", "normals") and float(case["inv_s"]) >= 1e3)
            bound[f"bwd.{tag}.{k}"] = 1e-3 if len(st) > 1 else (2e-2 if residue else 2.5e-3)
    print(f"[composite-anchor] {name}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v == v and v < float("inf"), k
        assert v <= bound[k], (k, v)
    # non-zero: fp32 rounding acts on every forward output that is not identically zero, and on the full gradients
    for k in uc.FWD_KEYS:
        assert worst["fwd." + k] > 0 or not f64[k].abs().max() > 0, k
    for k in ("d_sdf", "d_nrm", "d_rgb", "grad_inv_s") + (("d_bg_alpha",) if case["n_outside"] else ()):
        assert worst["bwd.all." + k] > 0, k
