"""The indoor configuration (config/train_indoor.yaml: ENCODE_A_BG False, N_OUTSIDE 8, 8 + 16 samples in 2 steps):
CPU port of the background NeRF without appearance head, parameters without `nerf.apperence_encoding.*`, and the
nrw system built from them.  Shared by the CPU and GPU indoor tests."""
import contextlib
import os
import sys
from unittest import mock

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "neuralrecon-w_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import neuconw_port as port  # noqa: E402
from oracle import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "indoor_checks.npz")
INDOOR = dict(n_samples=8, n_importance=16, up_sample_steps=2, n_outside=8)
N_RAYS, RAY_SEED = 24, 5
FULL_GRAD_NUMEL = 2048     # gradients up to this size are stored whole, larger ones as a seeded sample of 1024 elements
APP = "nerf.apperence_encoding."


def indoor_cfg(**kw):
    return synth.PathConfig(**{**INDOOR, **kw})


def indoor_params(seed=0):
    """oracle.synth.make_params without the background's appearance head (the reference's NeRF(encode_appearance=False)
    state dict, plus embedding_a and neuconw)."""
    return {k: v for k, v in synth.make_params(seed=seed).items() if not k.startswith(APP)}


def grad_sample_index(name, numel, n=1024):
    gen = torch.Generator().manual_seed(7 + sum(map(ord, name)) % 100003)
    return torch.randperm(numel, generator=gen)[:n]


def nerf_forward_noapp(P, pts4, dirs, a, pre="nerf."):
    """NeRF.forward, use_viewdirs without encode_appearance (models/nerf.py:156-182): the code `a` is ignored."""
    pe = port.posenc(pts4, 10)
    vd = port.posenc(dirs, 4)
    h = pe
    for i in range(8):
        h = F.relu(F.linear(h, P[f"{pre}pts_linears.{i}.weight"], P[f"{pre}pts_linears.{i}.bias"]))
        if i == 4:
            h = torch.cat([pe, h], -1)
    alpha = F.linear(h, P[pre + "alpha_linear.weight"], P[pre + "alpha_linear.bias"])
    feat = F.linear(h, P[pre + "feature_linear.weight"], P[pre + "feature_linear.bias"])
    h = F.relu(F.linear(torch.cat([feat, vd], -1), P[pre + "views_linears.0.weight"], P[pre + "views_linears.0.bias"]))
    rgb = F.linear(h, P[pre + "rgb_linear.weight"], P[pre + "rgb_linear.bias"])
    return alpha, rgb


def _nerf_forward_any(P, pts4, dirs, a, pre="nerf."):
    if f"{pre}apperence_encoding.static_linear_0.weight" in P:
        return _port_nerf_forward(P, pts4, dirs, a, pre)
    return nerf_forward_noapp(P, pts4, dirs, a, pre)


_port_nerf_forward = port.nerf_forward


@contextlib.contextmanager
def noapp_port():
    """oracle.neuconw_port with the background branch chosen by whether P holds the appearance head."""
    with mock.patch.object(port, "nerf_forward", _nerf_forward_any):
        yield port


def port_train_step(P, cfg, batch, **kw):
    with noapp_port():
        return port.train_step(P, cfg, batch, **kw)


def build_indoor_system(P, cfg, device="cuda", precision=None, backend=None, chunk_rows=None):
    """tests/util_nrw.build_system with nrw.NeRF(encode_appearance=False) (P: indoor_params)."""
    import nrw
    from util_nrw import COLOR_CONFIG, SDF_CONFIG

    neuconw = nrw.NeuconW({**SDF_CONFIG, "inside_outside": True}, COLOR_CONFIG, dict(init_val=0.3), in_channels_a=cfg.n_a,
                          encode_a=True)
    nerf = nrw.NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4],
                    encode_appearance=False, in_channels_a=cfg.n_a, in_channels_dir=27, use_viewdirs=True)
    emb = torch.nn.Embedding(cfg.n_vocab, cfg.n_a)
    neuconw.load_state_dict({k[len("neuconw."):]: v for k, v in P.items() if k.startswith("neuconw.")})
    nerf.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")})
    emb.load_state_dict({"weight": P["embedding_a.weight"]})
    neuconw, nerf, emb = neuconw.to(device), nerf.to(device), emb.to(device)
    renderer = nrw.NeuconWRenderer(
        nerf=nerf, neuconw=neuconw, embeddings={"a": emb}, n_samples=cfg.n_samples, s_val_base=cfg.s_val_base,
        n_importance=cfg.n_importance, n_outside=cfg.n_outside, up_sample_steps=cfg.up_sample_steps,
        perturb=cfg.perturb, origin=list(cfg.origin), radius=cfg.radius, render_bg=cfg.render_bg,
        mesh_mask_list=cfg.mesh_mask_list, floor_normal=False, floor_labels=["road"], depth_loss=cfg.depth_loss,
        spc_options=dict(voxel_size=0.1, recontruct_path=None, min_track_length=0), sample_range=cfg.sample_range,
        boundary_samples=cfg.boundary_samples, nerf_far_override=False, trim_sphere=cfg.trim_sphere,
        precision=precision, gemm_backend=backend, chunk_rows=chunk_rows)
    return dict(neuconw=neuconw, nerf=nerf, emb=emb, renderer=renderer)
