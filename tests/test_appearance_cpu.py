"""CPU side of appearance-code fitting (include/nrw.h nrw_appearance_*, nrw/appearance.py): the exported symbols, the
cache's byte count, the argument and state checks that run before any device work, and the loss / PSNR formulas."""
import ctypes as C

import pytest
import torch

from conftest import ROOT  # noqa: F401  (puts the package on sys.path)

ENTRIES = ("nrw_appearance_cache_bytes", "nrw_appearance_prepare", "nrw_appearance_forward", "nrw_appearance_backward")


@pytest.fixture(scope="module")
def lib():
    from nrw import _lib

    return _lib.lib()


def _ctx(L, nerf_app=1, precision=4):
    ctx = C.c_void_p()
    assert L.nrw_ctx_create(C.byref(ctx), precision, 0, 64, 48) == 0
    if not nerf_app:
        assert L.nrw_ctx_set_nerf_appearance(ctx, 0) == 0
    return ctx


def test_symbols_are_exported(lib):
    from nrw import _lib

    for name in ENTRIES:
        assert name in _lib.EXPORTS and hasattr(lib, name)


def _expected_bytes(R, S, n_out, nerf_app):
    """the cache layout of csrc/appearance.cu: fp32 arrays, each rounded up to 256 bytes"""
    r = lambda floats: (floats * 4 + 255) // 256 * 256
    RS, RT = R * S, R * (S + n_out)
    n = r(RS * 128) + r(RS * 3) * 2 + r(RS) * 2 + r(R * 3)
    if n_out > 0:
        n += r(RT) * 2
        n += r(RT * 128) + r(RT) if nerf_app else r(RT * 3)
    return n


@pytest.mark.parametrize("nerf_app", [1, 0])
@pytest.mark.parametrize("R,S,n_out", [(1, 1, 0), (3, 5, 2), (8192, 128, 4), (37, 34, 8), (100000, 142, 0)])
def test_cache_bytes(lib, nerf_app, R, S, n_out):
    ctx = _ctx(lib, nerf_app)
    try:
        got = lib.nrw_appearance_cache_bytes(ctx, R, S, n_out)
        assert got == _expected_bytes(R, S, n_out, nerf_app)
        # the per-sample part dominates: 128 fp32 pre-activations per sample of each network that reads the code
        assert got >= 512 * R * S + (512 * R * (S + n_out) if (n_out and nerf_app) else 0)
    finally:
        lib.nrw_ctx_destroy(ctx)


def test_cache_bytes_rejects_bad_sizes(lib):
    ctx = _ctx(lib)
    try:
        for R, S, n_out in ((0, 5, 2), (-1, 5, 2), (3, 0, 2), (3, 5, -1)):
            assert lib.nrw_appearance_cache_bytes(ctx, R, S, n_out) == -1
        assert lib.nrw_appearance_cache_bytes(None, 3, 5, 2) == -1
    finally:
        lib.nrw_ctx_destroy(ctx)


def test_argument_and_state_checks_before_device_work(lib):
    """NULL pointers and R <= 0 are NRW_ERR_ARG, an unbound context or an unprepared cache NRW_ERR_STATE; none of these
    paths touches device memory (the fake addresses below are never dereferenced)."""
    from nrw._lib import RenderCfg

    ctx = _ctx(lib)
    fake = C.c_void_p(1 << 20)
    cfg = RenderCfg()
    cfg.R, cfg.S, cfg.n_outside = 4, 8, 2
    try:
        prep = lambda c, cache=fake, z_out=fake: lib.nrw_appearance_prepare(ctx, C.byref(c), fake, fake, fake, z_out, fake,
                                                                             fake, cache, 1 << 30, None)
        assert prep(cfg, cache=None) == -1
        assert prep(cfg, z_out=None) == -1                 # n_outside > 0 needs z_out
        bad = RenderCfg()
        bad.R, bad.S, bad.n_outside = 0, 8, 2
        assert prep(bad) == -1
        assert prep(cfg) == -4                             # not bound
        assert lib.nrw_appearance_forward(ctx, fake, fake, None, None) == -1
        assert lib.nrw_appearance_forward(ctx, fake, fake, fake, None) == -4        # never prepared
        assert lib.nrw_appearance_backward(ctx, fake, fake, fake, None, None) == -1
        assert lib.nrw_appearance_backward(ctx, fake, fake, fake, fake, None) == -4
        assert b"not prepared" in lib.nrw_last_error()
    finally:
        lib.nrw_ctx_destroy(ctx)


def test_loss_and_psnr_follow_the_reference():
    from nrw.appearance import color_loss, psnr

    g = torch.Generator().manual_seed(0)
    x, y = torch.rand(50, 3, generator=g, dtype=torch.float64), torch.rand(50, 3, generator=g, dtype=torch.float64)
    # losses.py:22-27 with masks = ones: l1_loss(sum) / (masks.sum() + 1e-5)
    ref = torch.nn.functional.l1_loss(x - y, torch.zeros_like(x), reduction="sum") / (torch.ones(50, 1, dtype=torch.float64).sum() + 1e-5)
    assert torch.allclose(color_loss(x, y), ref.double(), rtol=1e-12, atol=0)
    assert torch.allclose(psnr(x, y), -10 * torch.log10(((x - y) ** 2).mean()), rtol=1e-12, atol=0)
