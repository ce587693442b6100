"""CPU-side byte counts of the chunk workspace (nrw_workspace_bytes is host-only).  In 'mixed' a forward slot keeps only
the hi plane of its two-plane activations (slots share one lo plane) and the backward scratch has the backward's one
plane, so a C2 or C3 training batch keeps every chunk's forward resident within 70 % of an 80 GB H100."""
import ctypes as C

import pytest

from conftest import ROOT  # noqa: F401  (puts the package on sys.path)

BUDGET_80GB = 0.7 * 80e9
C2 = (262144, 1, 8192, 132)     # chunk_rows, with_backward, rays, T = 128 samples + 4 outside
C3 = (232832, 1, 8192, 142)     # the balanced chunk of 8192 x 142


def _ctx(L, precision, backend=0):
    ctx = C.c_void_p()
    assert L.nrw_ctx_create(C.byref(ctx), precision, backend, 64, 48) == 0
    return ctx


@pytest.fixture(scope="module")
def ws():
    from nrw import _lib
    from nrw.engine import PRECISIONS

    L = _lib.lib()
    ctxs = {m: _ctx(L, PRECISIONS[m]) for m in PRECISIONS}
    ctxs.update({f"{m}_simt": _ctx(L, PRECISIONS[m], _lib.NRW_GEMM_SIMT) for m in ("bf16x6", "mixed")})
    yield lambda mode, shape, k_sdf, k_nerf: L.nrw_workspace_bytes(ctxs[mode], *shape, k_sdf, k_nerf)
    for c in ctxs.values():
        L.nrw_ctx_destroy(c)


def _slot_bytes_per_row(ws, mode):
    base = ws(mode, C2, 1, 1)
    return (ws(mode, C2, 2, 1) - base) / C2[0], (ws(mode, C2, 1, 2) - base) / C2[0]


def test_mixed_shares_one_lo_plane_and_keeps_every_c2_and_c3_chunk_within_the_80gb_budget(ws):
    assert ws("mixed", C2, 4, 5) == 53_001_172_992          # 79,475,619,840 with two planes per slot tensor
    assert ws("mixed", C3, 5, 5) == 54_084_727_808          # 82,605,716,480
    assert ws("mixed", C2, 4, 5) < BUDGET_80GB and ws("mixed", C3, 5, 5) < BUDGET_80GB
    # a slot beyond the first costs the hi plane only: 30,024 B per row for SDF + colour, 6,424 for NeRF
    assert _slot_bytes_per_row(ws, "mixed") == (30024, 6424)
    # the backward scratch has the backward's one plane: 10,880 B per row less than with two
    assert ws("mixed", C2, 1, 1) == 25_505_413_120 - 10880 * C2[0]


@pytest.mark.parametrize("mode, sdf_row, nerf_row, c2_full, c2_one, c3_full", [
    ("bf16x3", 57672, 12824, 88_065_554_432, 29_263_509_504, 91_665_675_264),
    ("bf16", 36168, 6424, 54_276_241_408, 19_096_516_608, 56_647_742_464),
    ("bf16x6", 79176, 19224, 121_854_867_456, 39_430_502_400, 126_683_608_064),
    ("bf16x6_simt", 79176, 19224, 121_854_867_456, 39_430_502_400, 126_683_608_064),   # the CUDA cores: same layout
])
def test_modes_whose_backward_reads_every_plane_keep_their_layout(ws, mode, sdf_row, nerf_row, c2_full, c2_one, c3_full):
    assert _slot_bytes_per_row(ws, mode) == (sdf_row, nerf_row)
    assert (ws(mode, C2, 4, 5), ws(mode, C2, 1, 1), ws(mode, C3, 5, 5)) == (c2_full, c2_one, c3_full)


def test_mixed_on_the_cuda_cores_keeps_fp32_side_streams_and_shares_the_lo_plane(ws):
    """gemm_simt takes no bf16 side streams, so 'mixed' there stores Q_l and the second-order terms in fp32; its slots
    beyond the first still keep the hi plane only."""
    assert _slot_bytes_per_row(ws, "mixed_simt") == (36168, 6424)
    assert (ws("mixed_simt", C2, 4, 5), ws("mixed_simt", C2, 1, 1), ws("mixed_simt", C3, 5, 5)) == \
        (61_591_107_584, 26_411_382_784, 63_144_686_592)


@pytest.mark.parametrize("precision", [0, 5])
def test_ctx_create_rejects_an_unknown_precision_and_names_the_valid_ones(precision):
    from nrw import _lib

    L = _lib.lib()
    ctx = C.c_void_p()
    assert L.nrw_ctx_create(C.byref(ctx), precision, 0, 64, 48) == -1   # NRW_ERR_ARG
    msg = L.nrw_last_error().decode()
    assert all(v in msg for v in ("1 (bf16)", "2 (bf16x3)", "3 (bf16x6)", "4 (mixed)")), msg
