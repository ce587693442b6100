"""Comparison of the oracle port with results of the unmodified reference, stored by oracle/make_golden.py
(reference_checks) as tests/golden/reference_checks.npz."""
import json

import numpy as np
import pytest
import torch

from oracle import neuconw_port as port
from oracle import synth
from oracle.make_golden import LIVE_CFG, LIVE_RAYS, LIVE_SEED, REF_CHECKS, grad_sample_index


@pytest.fixture(scope="module")
def G():
    return np.load(REF_CHECKS)


def test_port_vs_reference_live(params, G):
    cfg = synth.PathConfig(**LIVE_CFG, **synth.BRANDENBURG)
    batch = synth.make_rays(LIVE_RAYS, cfg, seed=LIVE_SEED)
    res_p, loss_p, grads_p = port.train_step(params, cfg, batch, perturb_overwrite=0)
    loss_r = float(G["live.loss"])
    assert abs(loss_r - float(loss_p)) < 1e-5 * abs(loss_r)
    keys = [k[len("live.out."):] for k in G.files if k.startswith("live.out.")]
    assert set(keys) == set(res_p)
    for k in keys:
        a, b = res_p[k].detach().numpy(), G["live.out." + k]
        assert a.shape == b.shape, k
        if a.size:
            assert np.abs(a - b).max() <= 1e-4 * (np.abs(b).max() + 1e-12), k
    stored = {k.split(".", 2)[2] for k in G.files if k.startswith(("live.g.", "live.gs."))}
    assert stored == set(grads_p)
    for k, g in grads_p.items():
        if "live.g." + k in G.files:                       # small tensors: every element
            a, b, scale = g.numpy(), G["live.g." + k], np.abs(G["live.g." + k]).max()
        else:                                              # large ones: a seeded sample, tolerance from the full tensor's max
            a, b, scale = g.reshape(-1)[grad_sample_index(k, g.numel())].numpy(), G["live.gs." + k], float(G["live.gmax." + k])
        assert np.abs(a - b).max() <= 1e-4 * (scale + 1e-12), k


def test_state_dict_names_match_reference(params, G):
    """oracle.synth parameter names/shapes == reference checkpoint layout (SURVEY.md §9.4)."""
    names = {k: tuple(v) for k, v in json.loads(str(G["state_dict_shapes"])).items()}
    assert names == {k: tuple(v.shape) for k, v in params.items()}
