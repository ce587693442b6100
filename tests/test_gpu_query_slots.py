"""GPU: a point query between a grad-enabled render and its backward.  NeuconW.forward, NeRF.forward and the SDF query
on its per-layer path run in slot 0 of their pass, which holds chunk 0 of the render's forward when every chunk has a
slot.  The backward must then recompute that forward instead of reading the query's activations, and give the gradient
of a backward without the query."""
import pytest
import torch

from util_nrw import build_system, rel_err, synth

pytestmark = pytest.mark.gpu

R = 300            # rays: at least 3 SDF and 3 NeRF chunks of 2048 rows (asserted below)
N = 2048           # query points: one whole chunk, so the query fills slot 0 without rebinding the workspace
CFG = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)


def _query(s, kind):
    g = torch.Generator(device="cuda").manual_seed(5)
    pts = torch.rand(N, 3, device="cuda", generator=g) * 1.6 - 0.8
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, device="cuda", generator=g), dim=-1)
    a = torch.randn(N, CFG.n_a, device="cuda", generator=g)
    if kind == "neuconw_forward":
        s["neuconw"](torch.cat([pts, dirs, a], -1).view(1, N, -1))
    elif kind == "nerf_forward":
        s["nerf"](torch.cat([pts, torch.rand(N, 1, device="cuda", generator=g)], -1), dirs, a)
    else:
        s["neuconw"].sdf(pts)


@pytest.mark.parametrize("precision, kind", [
    ("mixed", "neuconw_forward"), ("mixed", "nerf_forward"),
    ("bf16x3", "neuconw_forward"), ("bf16x3", "nerf_forward"),
    ("bf16", "sdf"),               # one plane: the SDF query runs per layer through the chunk workspace, not fused
])
def test_point_query_before_backward_recomputes_the_forward(precision, kind):
    P = synth.make_params(seed=0)
    b = {k: v.cuda() for k, v in synth.make_rays(R, CFG, seed=1).items()}
    bg = torch.zeros(1, 3, device="cuda")
    s = build_system(P, CFG, precision=precision, backend=0, chunk_rows=2048)
    r = s["renderer"]

    def grads(query):
        for m in (s["neuconw"], s["nerf"], s["emb"]):
            m.zero_grad(set_to_none=True)
        res = r.render(b["rays"], b["ts"], b["label"], perturb_overwrite=0, background_rgb=bg, cos_anneal_ratio=0.5)
        if query:
            _query(s, kind)
        (res["color"].sum() + res["gradient_error"].sum()).backward()
        return r.engine.last_flat_grad.clone(), s["emb"].weight.grad.clone()

    g_ref, e_ref = grads(False)
    eng = r.engine
    bound = eng.bound
    max_rays, max_T, _, chunk = bound
    n_sdf, n_nerf = -(-max_rays // (chunk // eng.bound_S)), -(-max_rays // (chunk // max_T))
    assert n_sdf >= 3 and n_nerf >= 3 and eng.slots == (n_sdf, n_nerf), (eng.slots, n_sdf, n_nerf)
    g_q, e_q = grads(True)
    assert eng.bound == bound                        # the query ran in the bound workspace
    assert rel_err(g_q.cpu().numpy(), g_ref.cpu().numpy()) < 2e-4      # fp32 atomics reorder only
    assert rel_err(e_q.cpu().numpy(), e_ref.cpu().numpy()) < 2e-4
