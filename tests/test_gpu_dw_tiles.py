"""GPU: the cooperative weight-gradient schedule of gemm_tc.cu (Sched::COOP).  One-plane MN-major split-K GEMMs with M >= 256
run 256 x 128 items that both consumer warpgroups share and reduce into the fp32 output straight from the accumulator
fragment; everything else keeps the 128 x 128 ping-pong items.  dW = dY^T X is compared against an fp64 product of the
bf16-rounded operands, and the per-warpgroup item counters of the debug profile buffer show which schedule ran."""
import ctypes as C

import numpy as np
import pytest
import torch

from util_nrw import gemm_test, rel_err

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def _nonempty_items(Ks, M, N, ks, tile_m):
    kb_total = _cdiv(Ks, 64)
    kb_per = _cdiv(kb_total, ks)
    return _cdiv(M, tile_m) * _cdiv(N, 128) * _cdiv(kb_total, kb_per)


def _run(Ks, M, N, ks, planes, seed):
    """(dW, reference, items counted by warpgroup 0, items counted by warpgroup 1)"""
    from nrw import _lib

    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    dY = torch.randn(Ks, M, device="cuda", generator=g)
    X = torch.randn(Ks, N, device="cuda", generator=g) / np.sqrt(Ks)
    if planes == 1:
        ref = dY.bfloat16().double().T @ X.bfloat16().double()
    else:
        ref = dY.double().T @ X.double()
    prof = torch.zeros(_sms() * 16, dtype=torch.int64, device="cuda")
    L.nrw_debug_gemm_profile(C.c_void_p(prof.data_ptr()))
    try:
        D = gemm_test(0, planes, 1, ks, dY, X)
    finally:
        L.nrw_debug_gemm_profile(None)
    s = prof.view(-1, 16).sum(0).cpu()
    return D.cpu(), ref.cpu(), int(s[6]), int(s[14])


# (sample rows, Np = dW rows, Kp = dW columns, k_slices); item counts on a 132-SM H100
COOP_SHAPES = [
    (1000, 256, 128, 2),      # 2 items: every CTA runs one; 1000 samples = 15 k-blocks + 40 rows
    (4100, 256, 384, 7),      # 65 k-blocks in slices of 10 (the last one 5), 21 items
    (640, 512, 256, 8),       # 10 k-blocks over 8 slices of 2: slices 5-7 are empty
    (33333, 512, 640, 10),    # 100 items, ragged last k-block
    (40000, 512, 512, 40),    # 320 items: CTAs 0-55 run three
    (5000, 320, 192, 4),      # ragged rows (second row tile holds 64) and columns (128 + 64)
]


@pytest.mark.parametrize("shape", COOP_SHAPES)
def test_cooperative_dw_matches_fp64(shape):
    Ks, M, N, ks = shape
    D, ref, wg0, wg1 = _run(Ks, M, N, ks, 1, seed=sum(shape))
    assert rel_err(D, ref) < 1e-4, shape
    items = _nonempty_items(Ks, M, N, ks, 256)
    assert wg0 == items and wg1 == items, (shape, wg0, wg1, items)   # both warpgroups on every non-empty item


@pytest.mark.parametrize("shape", [(9000, 512, 512, 6), (640, 256, 384, 8)])
def test_multi_plane_dw_keeps_the_ping_pong_tiles(shape):
    Ks, M, N, ks = shape
    D, ref, wg0, wg1 = _run(Ks, M, N, ks, 2, seed=sum(shape))
    assert rel_err(D, ref) < 5e-5, shape
    assert wg0 + wg1 == _nonempty_items(Ks, M, N, ks, 128), (shape, wg0, wg1)   # one warpgroup per item


def test_item_counts_cover_the_schedule():
    """The shapes above keep covering one item per CTA, three items per CTA and empty K-slices on this device."""
    n_sm = _sms()
    items = [_cdiv(M, 256) * _cdiv(N, 128) * ks for _, M, N, ks in COOP_SHAPES]
    assert min(items) <= n_sm
    assert max(items) > 2 * n_sm
    assert any(_nonempty_items(Ks, M, N, ks, 256) < _cdiv(M, 256) * _cdiv(N, 128) * ks for Ks, M, N, ks in COOP_SHAPES)
