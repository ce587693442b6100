"""GPU: the fused forward-only SDF chain (gemm_tc.cu::sdf_fused_kernel, models/neuconw.py:263-282 in one kernel) against
(a) the torch-CPU oracle, (b) the per-layer tensor-core chain it replaces (NRW_SDF_FUSED=0, separate process: the switch is read
once), on ragged sizes around the 64-row CTA tile and the 128-row pair tile, and (c) itself (run-to-run bit-identical)."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT
from oracle import neuconw_port as port
from oracle import synth
from util_nrw import build_system

pytestmark = pytest.mark.gpu

SIZES = (1, 63, 64, 65, 127, 128, 129, 1000, 70001)


def _points(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 1, 3, generator=g) * 2.4 - 1.2)


def _query(sizes):
    P = synth.make_params(seed=0)
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    s = build_system(P, cfg, precision="mixed", backend=0)
    out = {}
    with torch.no_grad():
        for n in sizes:
            out[n] = s["renderer"].sdf(_points(n, 100 + n).cuda()).reshape(-1).cpu()
    return P, out


def test_fused_chain_vs_oracle_and_per_layer_chain(tmp_path):
    assert os.environ.get("NRW_SDF_FUSED", "1") != "0", "this test needs the default (fused) configuration"
    P, fused = _query(SIZES)
    _, again = _query(SIZES)
    for n in SIZES:
        assert torch.equal(fused[n], again[n]), f"fused chain is not run-to-run deterministic at n={n}"
    # (a) oracle: SDFNetwork.sdf of the restated reference, fp32 on the CPU
    for n in (1, 129, 1000):
        with torch.no_grad():
            ref = port.sdf_forward(P, _points(n, 100 + n).reshape(-1, 3))[:, 0].detach()
        err = float((fused[n] - ref).abs().max()) / float(ref.abs().max())
        assert err < 1e-4, (n, err)
    # (b) the per-layer chain in its own process
    code = (
        "import sys, torch; sys.path.insert(0, 'tests'); sys.path.insert(0, '.'); sys.path.insert(0, 'neuralrecon-w_b200')\n"
        "import test_gpu_sdf_fused as t\n"
        f"_, out = t._query({SIZES!r})\n"
        f"torch.save(out, r'{tmp_path / 'unfused.pt'}')\nprint('unfused ok')\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, NRW_SDF_FUSED="0"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "unfused ok" in r.stdout, r.stdout + r.stderr
    unfused = torch.load(tmp_path / "unfused.pt")
    worst = 0.0
    for n in SIZES:
        assert fused[n].shape == unfused[n].shape == (n,)
        worst = max(worst, float((fused[n] - unfused[n]).abs().max()) / max(float(unfused[n].abs().max()), 1e-3))
    print(f"[parity] fused SDF chain vs per-layer chain: max rel diff {worst:.3g} over sizes {SIZES}")
    assert worst < 3e-5, worst        # different fp32 accumulation order over k-blocks; both are 1e-5 from the fp32 reference
