"""GPU: work distributions of the ping-pong GEMM schedule (gemm_tc.cu::gemm_tc_kernel).  A CTA's items alternate between
its two consumer warpgroups, so these cases cover what only that schedule has: CTAs whose second warpgroup gets no item,
odd item counts, many items per warpgroup with a ragged last row tile, empty K-slices, per-warpgroup column-sum
accumulators (bias gradients) and the per-warpgroup SDF-head partials of the per-layer chain.  Every case is compared
against an fp64 reference (or the CPU oracle) at the tolerances of test_gpu_parity.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_gpu_parity import _check_step
from util_nrw import gemm_test, rel_err, synth

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (M, N, K): 128 x 128 items (64-wide when N <= 64)
FORWARD_SHAPES = [
    (300, 640, 128),       # 15 items: fewer than SMs, odd; no CTA's second warpgroup has an item
    (6734, 640, 256),      # 265 items: CTA 0 takes three (warpgroup 0, 1, 0), ragged last row tile
    (20000, 512, 512),     # 628 items: ~5 per CTA, ragged last row tile (20000 = 156 x 128 + 32)
    (33333, 64, 192),      # 64-wide tiles, 261 items, ragged
]


@pytest.mark.parametrize("shape", FORWARD_SHAPES)
def test_forward_form_item_distributions(shape):
    M, N, K = shape
    torch.manual_seed(3)
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(N, K, device="cuda") / np.sqrt(K)
    bias = torch.randn(N, device="cuda")
    ref = (A.double() @ B.double().T + bias.double()).float().cpu()
    for planes, tol in ((1, 6e-3), (2, 2e-5), (3, 2e-5)):
        D = gemm_test(0, planes, 0, 1, A, B, bias, 0).cpu()
        assert rel_err(D, ref) < tol, (shape, planes)


# (K rows, M, N, k_slices) of the split-K weight-gradient form
SPLITK_SHAPES = [
    (9000, 768, 512, 5),     # 120 items: fewer than SMs
    (40000, 512, 512, 18),   # 288 items: some CTAs take three
    (640, 768, 768, 8),      # 10 k-blocks over 8 slices of 2: slices 5-7 are empty, 288 items
]


@pytest.mark.parametrize("shape", SPLITK_SHAPES)
def test_weight_gradient_form_item_distributions(shape):
    Ks, M, N, ks = shape
    torch.manual_seed(4)
    A = torch.randn(Ks, M, device="cuda")
    B = torch.randn(Ks, N, device="cuda") / np.sqrt(Ks)
    ref = (A.double().T @ B.double()).float().cpu()
    for planes, tol in ((1, 8e-3), (2, 5e-5), (3, 5e-5)):
        D = gemm_test(0, planes, 1, ks, A, B, None, 0).cpu()
        assert rel_err(D, ref) < tol, (shape, planes)


def test_item_counts_cover_the_schedule():
    """The shapes above keep covering an idle second warpgroup and three items per CTA on this device."""
    n_sm = _sms()
    items = [-(-M // 128) * -(-N // (64 if N <= 64 else 128)) for M, N, _ in FORWARD_SHAPES]
    assert min(items) < n_sm and min(items) % 2 == 1
    assert max(items) > 2 * n_sm


def test_train_step_column_sums_over_many_items():
    """Bias gradients come from the column-sum epilogues, now one accumulator per warpgroup.  One chunk of 600 rays x 24
    samples puts 113 row tiles (the last one ragged) into every layer's backward GEMM, so both warpgroups of most CTAs
    contribute to each column and flush at every n-tile change."""
    P = synth.make_params(seed=0)
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    _check_step(P, cfg, 600, "bf16x3", 0, 1e-4, 1e-2, chunk_rows=32768)


def test_per_layer_sdf_head_partials():
    """NRW_SDF_FUSED=0: the SDF query runs the per-layer chain whose last layer writes per-row head partials from each 64-row
    half of a warpgroup's tile (read once per process, hence the subprocess)."""
    code = (
        "import sys, torch; sys.path.insert(0, 'tests'); sys.path.insert(0, '.'); sys.path.insert(0, 'neuralrecon-w_b200')\n"
        "from util_nrw import build_system, port, rel_err, synth\n"
        "P = synth.make_params(seed=0)\n"
        "s = build_system(P, synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4), precision='mixed', backend=0)\n"
        "for n in (300, 40000):\n"
        "    g = torch.Generator().manual_seed(n); x = torch.rand(n, 1, 3, generator=g) * 2.4 - 1.2\n"
        "    with torch.no_grad():\n"
        "        out = s['renderer'].sdf(x.cuda()).reshape(-1).cpu()\n"
        "        ref = port.sdf_forward(P, x.reshape(-1, 3))[:, 0].detach()\n"
        "    e = rel_err(out, ref); assert e < 1e-4, (n, e)\n"
        "print('head ok')\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, NRW_SDF_FUSED="0"), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "head ok" in r.stdout, r.stdout + r.stderr
