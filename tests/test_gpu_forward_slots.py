"""GPU: forward slots of a training render.  Every chunk that has a slot of its own, and the last chunk, is consumed by the
backward without recomputing its forward; the rest are recomputed into the last slot.  In 'mixed' the slots share one lo
plane, which only a chunk's own forward reads.  Each case is compared with NRW_RECOMPUTE=1 (one slot per pass)."""
import pytest
import torch

from util_nrw import build_system, rel_err, synth

pytestmark = pytest.mark.gpu

R = 300            # rays: at least 3 SDF and 3 NeRF chunks of 2048 rows (asserted below)


def _system(precision):
    from nrw.train import TrainSystem

    return TrainSystem(torch.device("cuda", 0), n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4, n_vocab=64,
                       precision=precision, chunk_rows=2048, batch_size=R)


def _batch():
    from nrw.synthetic import make_ray_batch

    b = make_ray_batch(R, seed=4, n_vocab=64, device="cuda")
    b["label"] = torch.zeros(R, device="cuda")
    return b


def _step(precision):
    sysm = _system(precision)
    torch.manual_seed(7)          # the renderer's perturbation draws
    loss, flat, emb = sysm.compute_grads(_batch())
    return sysm.renderer.engine, loss, flat.clone(), emb.clone()


def _chunks(eng):
    """(SDF chunks, NeRF chunks) of the bound training batch."""
    max_rays, max_T, _, chunk = eng.bound
    return -(-max_rays // (chunk // eng.bound_S)), -(-max_rays // (chunk // max_T))


def _budget_gb(eng, k_sdf, k_nerf):
    max_rays, max_T, wb, chunk = eng.bound
    return eng.L.nrw_workspace_bytes(eng.ctx, chunk, wb, max_rays, max_T, k_sdf, k_nerf) * (1 + 1e-9) / 2 ** 30


def _same_step(eng_loss_grads, ref):
    _, loss, flat, emb = eng_loss_grads
    _, loss_r, flat_r, emb_r = ref
    assert torch.equal(loss, loss_r)                  # the forward arithmetic does not depend on the slot
    assert rel_err(flat.cpu().numpy(), flat_r.cpu().numpy()) < 2e-4      # fp32 atomics reorder only
    assert rel_err(emb.cpu().numpy(), emb_r.cpu().numpy()) < 2e-4


@pytest.fixture(scope="module")
def references():
    mp = pytest.MonkeyPatch()
    mp.setenv("NRW_RECOMPUTE", "1")
    try:
        refs = {p: _step(p) for p in ("mixed", "bf16x3")}
    finally:
        mp.undo()
    for eng, *_ in refs.values():
        assert eng.slots == (1, 1)
    return refs


@pytest.mark.parametrize("precision", ["mixed", "bf16x3"])
def test_every_chunk_resident(precision, references):
    got = _step(precision)
    n_sdf, n_nerf = _chunks(got[0])
    assert n_sdf >= 3 and n_nerf >= 3
    assert got[0].slots == (n_sdf, n_nerf)
    _same_step(got, references[precision])


@pytest.mark.parametrize("precision", ["mixed", "bf16x3"])
def test_partial_residency(precision, references, monkeypatch):
    monkeypatch.setenv("NRW_SLOT_BUDGET_GB", str(_budget_gb(references[precision][0], 2, 2)))
    got = _step(precision)
    n_sdf, n_nerf = _chunks(got[0])
    k_sdf, k_nerf = got[0].slots
    assert 1 < k_sdf < n_sdf and 1 <= k_nerf <= n_nerf, (got[0].slots, n_sdf, n_nerf)
    _same_step(got, references[precision])


def test_partial_residency_nerf(references, monkeypatch):
    eng_r = references["mixed"][0]
    n_sdf, n_nerf = _chunks(eng_r)
    monkeypatch.setenv("NRW_SLOT_BUDGET_GB", str(_budget_gb(eng_r, n_sdf, 2)))
    got = _step("mixed")
    assert got[0].bound == eng_r.bound and got[0].slots == (n_sdf, 2)
    _same_step(got, references["mixed"])


@pytest.mark.parametrize("precision", ["mixed", "bf16x3"])
def test_backward_of_an_older_render_with_fewer_slots_than_chunks(precision, monkeypatch):
    """A second grad-enabled render of the same shape overwrites the slots; the backward of the first one must recompute
    every chunk, including those that would otherwise still be resident."""
    P = synth.make_params(seed=0)
    cfg = synth.PathConfig(n_samples=16, n_importance=8, up_sample_steps=2, n_outside=4)
    bA = {k: v.cuda() for k, v in synth.make_rays(R, cfg, seed=1).items()}
    bB = {k: v.cuda() for k, v in synth.make_rays(R, cfg, seed=2).items()}
    bg = torch.zeros(1, 3, device="cuda")

    def grads_of(s, also_second):
        r = s["renderer"]
        for m in (s["neuconw"], s["nerf"], s["emb"]):
            m.zero_grad(set_to_none=True)
        resA = r.render(bA["rays"], bA["ts"], bA["label"], perturb_overwrite=0, background_rgb=bg, cos_anneal_ratio=0.5)
        if also_second:
            r.render(bB["rays"], bB["ts"], bB["label"], perturb_overwrite=0, background_rgb=bg, cos_anneal_ratio=0.5)
        (resA["color"].sum() + resA["gradient_error"].sum()).backward()
        return r.engine.last_flat_grad.clone()

    full = build_system(P, cfg, precision=precision, backend=0, chunk_rows=2048)
    g_ref = grads_of(full, False)
    eng = full["renderer"].engine
    n_sdf, n_nerf = _chunks(eng)
    assert eng.slots == (n_sdf, n_nerf) and n_sdf >= 3 and n_nerf >= 3
    monkeypatch.setenv("NRW_SLOT_BUDGET_GB", str(_budget_gb(eng, 2, 2)))
    part = build_system(P, cfg, precision=precision, backend=0, chunk_rows=2048)
    g_one = grads_of(part, False)
    k_sdf, k_nerf = part["renderer"].engine.slots
    assert 1 < k_sdf < n_sdf, part["renderer"].engine.slots
    g_two = grads_of(part, True)
    assert rel_err(g_one.cpu().numpy(), g_ref.cpu().numpy()) < 2e-4
    assert rel_err(g_two.cpu().numpy(), g_ref.cpu().numpy()) < 2e-4
