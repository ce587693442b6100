"""GPU: the wgmma GEMM epilogue works through a tile in rounds of 64 columns, each warp taking a pair of 16-column chunks
(columns nc and nc + 32) whose side streams are loaded together.  A pair where either chunk is ragged - a partial last row
tile, a tile narrower than the pair, or the skip layer's stored-column boundary at 473 - takes the per-chunk path for both
chunks.  A training render and backward at row counts whose last row tile ends inside a warp's 32 rows runs through all of
these on the 512-, 256-, 128- and 64-wide layers; every output and gradient is compared against the CPU oracle at the
tolerances of test_gpu_parity.py, and the per-ray forward outputs must be bit-identical between two runs (gradient_error is
a float atomicAdd reduction over blocks, and so is the loss term built on it: neither is compared bit for bit)."""
import pytest
import torch

from test_gpu_parity import RTOL, _check_step
from util_nrw import build_system, cuda_train_step, synth

pytestmark = pytest.mark.gpu

CFG = dict(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)

# (rays, chunk_rows): 24 SDF rows and 4 NeRF rows per ray
#   601 rays, one chunk: 14424 SDF rows (last row tile: 88 rows), 2404 NeRF rows (100 rows)
#   437 rays, chunks of 2048 rows: the last SDF chunk has 248 rows (last row tile: 120 rows)
CASES = [(601, 32768), (437, 2048)]


@pytest.mark.parametrize("rays,chunk_rows", CASES)
def test_ragged_pairs_against_oracle(rays, chunk_rows):
    P = synth.make_params(seed=0)
    _check_step(P, synth.PathConfig(**CFG), rays, "bf16x3", 0, RTOL, 1e-2, chunk_rows=chunk_rows)


@pytest.mark.parametrize("precision", ["bf16x3", "mixed"])
def test_forward_bit_identical_between_runs(precision):
    P = synth.make_params(seed=0)
    cfg = synth.PathConfig(**CFG)
    batch = synth.make_rays(601, cfg, seed=11)
    s = build_system(P, cfg, precision=precision, backend=0, chunk_rows=32768)
    res_a, _, _ = cuda_train_step(s, cfg, batch)
    res_b, _, _ = cuda_train_step(s, cfg, batch)
    assert set(res_a) == set(res_b)
    for k in res_a:
        if k != "gradient_error":
            assert torch.equal(res_a[k], res_b[k]), k
