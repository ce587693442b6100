"""CPU checks of test_gpu_query_forward's inputs and references: the level-set rows lie on the fp64 SDF's zero level set,
the NeRF points reach the ends of their range, and the fp32 evaluation of every query's reference (the anchor of the
tolerance rule) agrees with the fp64 one to fp32 level on those inputs."""
import pytest
import torch

import test_gpu_query_forward as qf
from util_nrw import port

N = 300
# fp32 anchor error per output on edge_inputs(N): ~10x the worst over the queries measured on the CPU (sdf 8.7e-7,
# normals 3.8e-6, rgb 3.0e-6, density 4.5e-7)
FP32_LEVEL = dict(sdf=1e-5, normals=4e-5, rgb=3e-5, density=5e-6)


def test_edge_inputs_reach_the_edges():
    inp = qf.edge_inputs(qf.CHUNK + 10)
    on = torch.arange(0, qf.CHUNK, 4)
    Q = {k: v.double() for k, v in qf.qb.params(variant=qf.VARIANT).items() if k.startswith("neuconw.sdf_net.")}
    with torch.no_grad():
        sdf = port.sdf_forward(Q, inp["pts"].double())[:, 0]
    assert float(sdf[on].abs().max()) < 1e-6 and float(sdf.abs().max()) > 0.5
    assert float(inp["pts"].abs().max()) > 1.19
    inv_r = inp["pts4"][:, 3]
    assert float(inv_r.max()) == 1.0 and float(inv_r.min()) <= 1.0001e-4
    assert torch.allclose(inp["pts4"][:, :3].norm(dim=-1), torch.ones(len(inv_r)), atol=1e-6)
    assert torch.allclose(inp["dirs"].norm(dim=-1), torch.ones(len(inv_r)), atol=1e-6)
    assert float(inp["a"].abs().max()) == 5.0


@pytest.mark.parametrize("query", list(qf.OUTPUTS))
def test_fp32_reference_agrees_with_fp64(query):
    r64, r32 = qf.reference(query, N, torch.float64), qf.reference(query, N, torch.float32)
    assert set(r64) == set(qf.OUTPUTS[query])
    for k in r64:
        e = qf.output_err(k, r32[k], r64[k])
        print(f"[query-fwd-cpu] {query} {k}: fp32 error {e:.3e}")
        assert 0.0 < e < FP32_LEVEL[k], (k, e)
