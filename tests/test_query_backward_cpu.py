"""CPU checks of the point-query backward (nrw_neuconw_backward / nrw_nerf_backward):

  * the encoding derivatives its pointwise input-gradient kernels use (csrc/pointwise.cu pe_bwd_kernel,
    sdf_point_bwd_kernel), restated below and checked against fp64 autograd of the port's positional encoding;
  * the argument errors of the two entries, which return before touching the device."""
import ctypes as C

import pytest
import torch

from util_nrw import port


def pe_bwd(x, n_freq, dE):
    """J_PE(x)^T dE as pe_bwd_kernel forms it: coordinate c feeds column c, sin column D + 2Dk + c, cos column
    2D + 2Dk + c (f = 2^k): dE[c] + sum_k f (cos(f x) dE[sin] - sin(f x) dE[cos])."""
    D = x.shape[1]
    out = dE[:, :D].clone()
    for k in range(n_freq):
        f = 2.0 ** k
        out += f * (torch.cos(f * x) * dE[:, D + 2 * D * k:2 * D + 2 * D * k]
                    - torch.sin(f * x) * dE[:, 2 * D + 2 * D * k:3 * D + 2 * D * k])
    return out


def pe_second(x, n_freq, v, dn):
    """dn_c sum_j v_j E_j''(x_c), the term of sdf_point_bwd_kernel that differentiates J_PE itself (E'' is diagonal):
    sin'' = -f^2 sin, cos'' = -f^2 cos, the identity columns have none."""
    D = x.shape[1]
    out = torch.zeros_like(x)
    for k in range(n_freq):
        f = 2.0 ** k
        out -= f * f * (torch.sin(f * x) * v[:, D + 2 * D * k:2 * D + 2 * D * k]
                        + torch.cos(f * x) * v[:, 2 * D + 2 * D * k:3 * D + 2 * D * k])
    return out * dn


@pytest.mark.parametrize("D, n_freq", [(3, 6), (3, 4), (4, 10)])     # SDF points, view directions, NeRF points
def test_encoding_jacobian_transpose_matches_autograd(D, n_freq):
    g = torch.Generator().manual_seed(D * 100 + n_freq)
    x = (torch.rand(64, D, generator=g, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    E = port.posenc(x, n_freq)
    dE = torch.randn(E.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(E, x, dE)
    assert torch.allclose(pe_bwd(x.detach(), n_freq, dE), ref, rtol=1e-12, atol=1e-12)


def test_encoding_second_derivative_matches_autograd():
    """d/dx <dn, J_PE(x)^T v> with v held fixed: the point gradient of a normal n = J_PE^T v beyond the one through v."""
    g = torch.Generator().manual_seed(7)
    x = (torch.rand(64, 3, generator=g, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    v = torch.randn(64, 39, generator=g, dtype=torch.float64)
    dn = torch.randn(64, 3, generator=g, dtype=torch.float64)
    (n,) = torch.autograd.grad(port.posenc(x, 6), x, v, create_graph=True)
    assert torch.allclose(n, pe_bwd(x.detach(), 6, v), rtol=1e-12, atol=1e-12)
    (ref,) = torch.autograd.grad((n * dn).sum(), x)
    assert torch.allclose(pe_second(x.detach(), 6, v, dn), ref, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------------- argument errors
NRW_ERR_ARG, NRW_ERR_STATE = -1, -4


@pytest.fixture()
def ctx():
    """an unbound context of each NeRF kind (nrw_ctx_create and set_nerf_appearance stay on the host)."""
    from nrw import _lib

    L = _lib.lib()
    made = {}
    for app in (1, 0):
        c = C.c_void_p()
        _lib.check(L.nrw_ctx_create(C.byref(c), 2, 0, 0, 48), "nrw_ctx_create")
        _lib.check(L.nrw_ctx_set_nerf_appearance(c, app), "nrw_ctx_set_nerf_appearance")
        made[app] = c
    yield L, made
    for c in made.values():
        L.nrw_ctx_destroy(c)


def _p():
    return C.c_void_p(4096)     # never dereferenced: every call below returns before any device work


def test_neuconw_backward_argument_errors(ctx):
    L, c = ctx
    p = _p()
    call = lambda n, dirs, a, g_rgb: L.nrw_neuconw_backward(c[1], p, dirs, a, n, p, p, g_rgb, p, p, p, p, None)
    assert call(-1, p, p, None) == NRW_ERR_ARG
    assert b"n=-1" in L.nrw_last_error()
    assert call(8, None, p, p) == NRW_ERR_ARG          # g_rgb without dirs
    assert call(8, p, None, p) == NRW_ERR_ARG          # ... or without a
    assert b"g_rgb" in L.nrw_last_error()
    assert L.nrw_neuconw_backward(None, p, p, p, 8, p, p, p, p, p, p, p, None) == NRW_ERR_ARG
    assert call(0, None, None, None) == 0              # n == 0: nothing to do
    assert call(8, None, None, None) == NRW_ERR_STATE  # not bound for backward
    assert b"bind" in L.nrw_last_error()


def test_nerf_backward_argument_errors(ctx):
    L, c = ctx
    p = _p()
    call = lambda k, n, a, g_rgb, grad_a: L.nrw_nerf_backward(c[k], p, p, a, n, p, g_rgb, p, p, p, grad_a, None)
    assert call(1, -3, p, p, p) == NRW_ERR_ARG
    assert call(1, 8, None, p, None) == NRW_ERR_ARG    # g_rgb without a, appearance head on
    assert call(0, 8, None, p, p) == NRW_ERR_ARG       # grad_a without the appearance head
    assert b"appearance head" in L.nrw_last_error()
    assert L.nrw_nerf_backward(c[1], p, None, p, 8, p, p, p, p, p, p, None) == NRW_ERR_ARG    # no dirs
    assert call(1, 0, p, p, p) == 0
    assert call(0, 8, None, p, None) == NRW_ERR_STATE  # without the head the code is not needed; not bound
    assert call(1, 8, p, p, p) == NRW_ERR_STATE
