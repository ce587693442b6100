"""CPU checks of the indoor configuration (background NeRF without appearance head): module layout against the
reference, the C-ABI switch and its byte counts, and the CPU port against the reference's own results
(tests/golden/indoor_checks.npz, written by tools/make_indoor_golden.py)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from conftest import ROOT  # noqa: F401  (puts the package on sys.path)
from oracle import synth
from util_indoor import APP, GOLDEN, N_RAYS, RAY_SEED, grad_sample_index, indoor_cfg, indoor_params, port_train_step

NERF_KW = dict(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4], in_channels_a=48,
               in_channels_dir=27, use_viewdirs=True)


@pytest.fixture(scope="module")
def G():
    return np.load(GOLDEN)


def test_noapp_nerf_has_the_reference_layout_and_loads_its_state_dict(G):
    import nrw

    ref_shapes = {k: tuple(v) for k, v in json.loads(str(G["nerf_state_dict_shapes"])).items()}
    n = nrw.NeRF(**NERF_KW, encode_appearance=False)
    assert not hasattr(n, "apperence_encoding")
    assert {k: tuple(v.shape) for k, v in n.state_dict().items()} == ref_shapes
    assert list(n.state_dict()) == sorted(ref_shapes, key=list(n.state_dict()).index)
    P = indoor_params()
    n.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")}, strict=True)
    assert torch.equal(n.views_linears[0].weight, P["nerf.views_linears.0.weight"])
    # the appearance variant keeps its layout
    a = nrw.NeRF(**NERF_KW, encode_appearance=True)
    assert any(k.startswith("apperence_encoding.") for k in a.state_dict())


def test_other_unsupported_configurations_still_raise():
    import nrw
    from util_nrw import COLOR_CONFIG, SDF_CONFIG

    with pytest.raises(nrw.NrwError):
        nrw.NeuconW(SDF_CONFIG, COLOR_CONFIG, dict(init_val=0.3), in_channels_a=48, encode_a=False)
    with pytest.raises(nrw.NrwError):
        nrw.NeRF(D=4)
    with pytest.raises(nrw.NrwError):
        nrw.NeRF(**dict(NERF_KW, use_viewdirs=False), encode_appearance=False)


def _ctx(L, n_planes=2, app=None):
    ctx = C.c_void_p()
    assert L.nrw_ctx_create(C.byref(ctx), n_planes, 0, 64, 48) == 0
    if app is not None:
        assert L.nrw_ctx_set_nerf_appearance(ctx, app) == 0
    return ctx


def test_set_nerf_appearance_rejects_bad_values():
    from nrw import _lib

    L = _lib.lib()
    ctx = _ctx(L)
    try:
        assert L.nrw_ctx_set_nerf_appearance(ctx, 2) != 0
        assert b"set_nerf_appearance" in L.nrw_last_error()
    finally:
        L.nrw_ctx_destroy(ctx)


@pytest.mark.parametrize("n_planes", [1, 2, 3])
def test_noapp_workspace_is_smaller_and_packed_no_larger(n_planes):
    from nrw import _lib

    L = _lib.lib()
    base, on, off = _ctx(L, n_planes), _ctx(L, n_planes, 1), _ctx(L, n_planes, 0)
    try:
        shapes = [(262144, 1, 8192, 40, 4, 4), (262144, 0, 8192, 40, 1, 1), (4096, 1, 64, 40, 1, 2)]
        for sh in shapes:
            w0, w1, w2 = (L.nrw_workspace_bytes(c, *sh) for c in (base, on, off))
            assert w1 == w0 and w2 < w0, sh
        assert L.nrw_packed_bytes(on) == L.nrw_packed_bytes(base)
        assert L.nrw_packed_bytes(off) <= L.nrw_packed_bytes(base)
        # switching back restores the default exactly
        assert L.nrw_ctx_set_nerf_appearance(off, 1) == 0
        assert L.nrw_workspace_bytes(off, *shapes[0]) == L.nrw_workspace_bytes(base, *shapes[0])
    finally:
        for c in (base, on, off):
            L.nrw_ctx_destroy(c)


def test_port_noapp_path_matches_reference(G):
    cfg = indoor_cfg(**synth.BRANDENBURG)
    batch = synth.make_rays(N_RAYS, cfg, seed=RAY_SEED)
    P = indoor_params()
    res_p, loss_p, grads_p = port_train_step(P, cfg, batch, perturb_overwrite=0)
    loss_r = float(G["loss"])
    assert abs(loss_r - float(loss_p)) < 1e-5 * abs(loss_r)
    keys = [k[len("out."):] for k in G.files if k.startswith("out.")]
    assert set(keys) == set(res_p)
    for k in keys:
        a, b = res_p[k].detach().numpy(), G["out." + k]
        assert a.shape == b.shape, k
        if a.size:
            assert np.abs(a - b).max() <= 1e-4 * (np.abs(b).max() + 1e-12), k
    stored = {k.split(".", 1)[1] for k in G.files if k.startswith(("g.", "gs."))}
    assert stored == set(grads_p) and not any(k.startswith(APP) for k in stored)
    for k, g in grads_p.items():
        if "g." + k in G.files:
            a, b, scale = g.numpy(), G["g." + k], np.abs(G["g." + k]).max()
        else:
            a, b, scale = g.reshape(-1)[grad_sample_index(k, g.numel())].numpy(), G["gs." + k], float(G["gmax." + k])
        assert np.abs(a - b).max() <= 1e-4 * (scale + 1e-12), k
    assert float(np.abs(G["gs.nerf.views_linears.0.weight"]).max()) > 0
