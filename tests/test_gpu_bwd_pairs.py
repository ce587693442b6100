"""GPU: paired backward launches (gemm_tc.cu, Sched::PAIR).  A backward layer's data GEMM and its weight gradient run as one
launch: 128 x 128 data tiles with their specialised epilogue and 128 x 128 x K-slice dW items with the fragment red.add.
Through nrw_gemm_pair_test, every data output of the paired launch is bit-identical to the same GEMM launched alone (the
tile MMAs and the epilogue are unchanged), column sums agree to fp32 reordering, and dW agrees with an fp64 product of the
bf16 operands.  The per-warpgroup item counters show that every non-empty item ran once, on the warpgroup the round
schedule gives it.  At step level, a C2-shaped `mixed` step with pairing matches one without (NRW_BWD_PAIR=0)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from util_nrw import rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {"generic": 0, "tangent": 1, "reverse": 2, "relu_bwd": 3}


def _cdiv(a, b):
    return -(-a // b)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _expected_counts(M, N, Mw, Nw, Kw, ks):
    """[warpgroup][0 data, 1 dW] non-empty items under the round schedule of a paired launch"""
    n_data = _cdiv(M, 128) * _cdiv(N, 128)
    tiles = _cdiv(Mw, 128) * _cdiv(Nw, 128)
    n_dw = tiles * ks
    kb_total = _cdiv(Kw, 64)
    kb_per = _cdiv(kb_total, ks)
    G = min(_sms(), n_data + n_dw)
    rd, rw = _cdiv(n_data, G), _cdiv(n_dw, G)
    ri = min(rd, rw)
    counts = [[0, 0], [0, 0]]
    for b in range(G):
        for j in range(rd + rw):
            if j < 2 * ri:
                dw, r = j & 1, j >> 1
            else:
                dw, r = int(rd <= ri), j - ri
            i = r * G + b
            ok = i < n_data if not dw else (i < n_dw and (i // tiles) * kb_per < kb_total)
            counts[j & 1][dw] += int(ok)
    assert counts[0][0] + counts[1][0] == n_data
    assert counts[0][1] + counts[1][1] == tiles * _cdiv(kb_total, kb_per)
    return counts


def _run(paired, kind, M, N, K, Mw, Nw, Kw, ks, scale=1.0, n_store=1 << 30, rowvec=False, out_f32=False,
         bcast_q=False, seed=0):
    from nrw import _lib

    L = _lib.lib()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    bf = torch.bfloat16
    A = torch.randn(M, K, device=dev, generator=g).to(bf)
    B = (torch.randn(N, K, device=dev, generator=g) / np.sqrt(K)).to(bf)
    dY = torch.randn(Kw, Mw, device=dev, generator=g).to(bf)
    X = (torch.randn(Kw, Nw, device=dev, generator=g) / np.sqrt(Kw)).to(bf)
    if kind in ("tangent", "reverse"):
        side_h = (torch.rand(M, N, device=dev, generator=g) * 0.05).to(bf)   # u = softplus100(a): gates across the kink
    else:
        side_h = torch.randn(M, N, device=dev, generator=g).to(bf)            # ReLU mask
    side_f = None if bcast_q else torch.randn(M, N, device=dev, generator=g)
    rv = torch.randn(M, device=dev, generator=g) if rowvec else None
    cv = torch.randn(N, device=dev, generator=g)
    out_pl = torch.zeros(M, N, dtype=bf, device=dev)
    of32 = torch.zeros(M, N, device=dev) if out_f32 else None
    out2 = torch.zeros(M, N, device=dev)
    colsum = torch.zeros(N, device=dev)
    dW = torch.zeros(Mw, Nw, device=dev)
    prof = torch.zeros(_sms() * 16, dtype=torch.int64, device=dev)
    L.nrw_debug_gemm_profile(C.c_void_p(prof.data_ptr()))
    try:
        _lib.check(L.nrw_gemm_pair_test(paired, KINDS[kind], M, N, K, Mw, Nw, Kw, ks, _lib.ptr(A), _lib.ptr(B), _lib.ptr(dY),
                                        _lib.ptr(X), _lib.ptr(side_h), _lib.ptr(side_f), _lib.ptr(rv), _lib.ptr(cv), scale,
                                        n_store, _lib.ptr(out_pl), _lib.ptr(of32), _lib.ptr(out2), _lib.ptr(colsum),
                                        _lib.ptr(dW), _lib.stream_ptr()), "nrw_gemm_pair_test")
        torch.cuda.synchronize()
    finally:
        L.nrw_debug_gemm_profile(None)
    s = prof.view(-1, 16).sum(0).cpu()
    ref = dY.double().T @ X.double()
    outs = dict(out_pl=out_pl, out2=out2, colsum=colsum)
    if of32 is not None:
        outs["out_f32"] = of32
    return {k: v.cpu() for k, v in outs.items()}, dW.cpu(), ref.cpu(), [[int(s[6]), int(s[7])], [int(s[14]), int(s[15])]]


S2 = 0.70710678118654752440
# (name, kind, data M, N, K, dW Mw, Nw, Kw, k_slices, extra)
CASES = [
    ("tangent_ragged", "tangent", 1000, 512, 512, 512, 512, 1000, 3, {}),           # 1000 samples: last slice 4 k-blocks, ragged
    ("tangent_skip", "tangent", 4173, 512, 512, 512, 512, 4173, 2, dict(scale=S2, n_store=473)),
    ("tangent_last", "tangent", 300, 512, 512, 512, 512, 300, 1, dict(out_f32=True, bcast_q=True)),
    ("reverse_feature", "reverse", 2000, 512, 512, 512, 512, 2000, 2, dict(rowvec=True)),
    ("reverse_skip", "reverse", 3000, 512, 512, 512, 512, 3000, 4, dict(scale=S2, n_store=473)),
    ("relu_more_data", "relu_bwd", 20000, 256, 256, 256, 256, 20000, 4, {}),       # 314 data tiles vs 16 dW items
    ("relu_rowvec", "relu_bwd", 1500, 256, 256, 256, 256, 1500, 2, dict(rowvec=True)),
    ("relu_single_tile", "relu_bwd", 128, 128, 128, 128, 128, 40000, 60, {}),       # one data tile, 60 dW items
    ("generic_wide_dw", "generic", 5000, 512, 128, 128, 640, 5000, 5, {}),
    ("generic_ragged_dw", "generic", 777, 128, 256, 256, 192, 777, 3, {}),          # dW columns 128 + 64; 13 k-blocks / 3
    ("generic_empty_slices", "generic", 640, 256, 256, 256, 256, 640, 8, {}),       # 10 k-blocks over 8 slices of 2
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_paired_launch_matches_separate_launches(case):
    _, kind, M, N, K, Mw, Nw, Kw, ks, extra = case
    alone, dW0, ref, _ = _run(0, kind, M, N, K, Mw, Nw, Kw, ks, seed=M + Kw, **extra)
    paired, dW1, ref1, counts = _run(1, kind, M, N, K, Mw, Nw, Kw, ks, seed=M + Kw, **extra)
    assert torch.equal(ref, ref1)
    for k in alone:
        if k == "colsum":
            assert rel_err(paired[k], alone[k]) < 1e-5, (k, rel_err(paired[k], alone[k]))
        else:
            assert torch.equal(paired[k], alone[k]), (k, rel_err(paired[k].float(), alone[k].float()))
    assert rel_err(dW1, ref) < 1e-4, rel_err(dW1, ref)
    assert rel_err(dW0, ref) < 1e-4, rel_err(dW0, ref)
    assert counts == _expected_counts(M, N, Mw, Nw, Kw, ks), counts


def test_cases_cover_the_schedule():
    """More dW items than data items and the other way round, and both orders of leftover rounds on this device."""
    n_sm = _sms()
    more_dw = more_data = 0
    for _, _, M, N, _, Mw, Nw, _, ks, _ in CASES:
        n_data, n_dw = _cdiv(M, 128) * _cdiv(N, 128), _cdiv(Mw, 128) * _cdiv(Nw, 128) * ks
        more_dw += n_dw > n_data
        more_data += _cdiv(n_data, n_sm) > _cdiv(n_dw, n_sm)
    assert more_dw and more_data


def test_ineligible_pair_is_refused():
    """A 64-column weight gradient cannot share the launch: the export reports it instead of running something else."""
    from nrw import _lib

    with pytest.raises(_lib.NrwError):
        _run(1, "generic", 256, 512, 128, 512, 64, 256, 1)


_STEP = """
import sys, torch
sys.path.insert(0, {root!r}); sys.path.insert(0, {pkg!r})
from nrw.synthetic import make_ray_batch
from nrw.train import TrainSystem
dev = torch.device("cuda", 0)
sysm = TrainSystem(dev, n_samples=64, n_importance=64, up_sample_steps=4, n_outside=4, precision="mixed", chunk_rows=65536,
                   batch_size=1024, seed=66)
b = make_ray_batch(1024, seed=3, device=dev)
torch.manual_seed(0)
res = sysm.forward(b["rays"], b["ts"], b["label"])
loss = sum(sysm.loss(res, b["rgbs"]).values())
loss.backward()
torch.save(dict(loss=loss.detach().cpu(), grad=sysm.renderer.engine.last_flat_grad.cpu()), {out!r})
print("step ok")
"""


def _step(path, pair):
    code = _STEP.format(root=ROOT, pkg=os.path.join(ROOT, "neuralrecon-w_b200"), out=str(path))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, NRW_BWD_PAIR=pair), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0 and "step ok" in r.stdout, r.stdout + r.stderr
    return torch.load(path)


def test_training_step_matches_unpaired(tmp_path):
    """C2 sample counts, 1024 rays in chunks of 65,536 rows: the forward is untouched, so the loss is bit-identical; the
    gradient differs by the order of fp32 atomics."""
    a = _step(tmp_path / "paired.pt", "1")
    b = _step(tmp_path / "unpaired.pt", "0")
    assert torch.equal(a["loss"], b["loss"])
    ga, gb = a["grad"].double(), b["grad"].double()
    assert torch.isfinite(ga).all()
    rel = float((ga - gb).norm() / gb.norm())
    print(f"[pairs] flat gradient, paired vs NRW_BWD_PAIR=0: relative L2 {rel:.3g}")
    assert rel <= 5e-5, rel
