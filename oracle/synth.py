"""Deterministic synthetic parameters and ray batches (TEST INFRASTRUCTURE).

Everything here is generated from ``torch.Generator`` streams with fixed seeds so
that the build container (where golden vectors are produced from the real
reference) and the GPU box (where only this file travels) construct bit-identical
inputs.  Shapes/names follow the reference checkpoint layout (SURVEY.md §9.4;
models/neuconw.py:183-259, models/nerf.py:86-154).
"""
import math
from dataclasses import dataclass, field, asdict
from typing import List, Optional

import torch


@dataclass
class PathConfig:
    """Sampler / renderer knobs (config/defaults.py:7-40, rendering/renderer.py:52-135)."""
    n_samples: int = 64
    n_importance: int = 64
    up_sample_steps: int = 4
    n_outside: int = 4
    s_val_base: int = 3
    perturb: float = 0.0
    origin: tuple = (0.0, 0.0, 0.0)
    radius: float = 1.0
    n_vocab: int = 5000
    n_a: int = 48
    mesh_mask_list: Optional[List[str]] = field(default_factory=lambda: ["sky"])
    depth_loss: bool = True
    render_bg: bool = True
    trim_sphere: bool = True
    boundary_samples: int = 0
    sample_range: float = 16.0
    cos_anneal_ratio: float = 0.5
    # loss weights (config/train_brandenburg_gate.yaml:62-68)
    igr_weight: float = 0.0001
    mask_weight: float = 0.1
    depth_weight: float = 0.1

    def to_dict(self):
        return asdict(self)


C1 = PathConfig(n_samples=64, n_importance=16, up_sample_steps=2, n_outside=4)
C2 = PathConfig(n_samples=64, n_importance=64, up_sample_steps=4, n_outside=4)
BRANDENBURG = dict(origin=(0.568699, -0.0935532, 6.28958), radius=4.6)

SDF_DIMS = [(512, 39), (512, 512), (512, 512), (473, 512), (512, 512), (512, 512), (512, 512),
            (512, 512), (513, 512)]
COLOR_DIMS = [(256, 134), (256, 256), (256, 256), (256, 256), (3, 256)]
NERF_PTS = [(256, 84), (256, 256), (256, 256), (256, 256), (256, 256), (256, 340), (256, 256),
            (256, 256)]


def _linear_default(gen, o, i):
    """torch.nn.Linear default init statistics: U(-1/sqrt(i), 1/sqrt(i)) for weight and bias."""
    b = 1.0 / math.sqrt(i)
    w = (torch.rand(o, i, generator=gen) * 2 - 1) * b
    bias = (torch.rand(o, generator=gen) * 2 - 1) * b
    return w, bias


def make_params(seed: int = 0, n_vocab: int = 5000, n_a: int = 48, jitter: float = 1.0):
    """State dict with the reference's parameter names (prefixes embedding_a./neuconw./nerf.).

    SDF net follows the statistics of the reference's geometric init
    (models/neuconw.py:222-254) so that sdf(x) ~ |x| - 0.5, with small ``jitter``
    perturbations so weight-norm gains, biases and PE columns are all exercised.
    """
    g = torch.Generator().manual_seed(1000 + seed)
    P = {}
    P["embedding_a.weight"] = torch.randn(n_vocab, n_a, generator=g)
    for l, (o, i) in enumerate(SDF_DIMS):
        if l == 8:
            w = math.sqrt(math.pi) / math.sqrt(i) + 1e-4 * torch.randn(o, i, generator=g)
            b = torch.full((o,), -0.5)
        else:
            w = torch.randn(o, i, generator=g) * (math.sqrt(2) / math.sqrt(o))
            b = torch.zeros(o)
            if l == 0:
                w[:, 3:] *= 0.05 * jitter
            if l == 4:
                w[:, -36:] *= 0.05 * jitter
        b = b + 0.01 * jitter * torch.randn(o, generator=g)
        gain = w.norm(dim=1, keepdim=True) * (1.0 + 0.05 * jitter * torch.randn(o, 1, generator=g))
        pre = f"neuconw.sdf_net.lin{l}."
        P[pre + "bias"] = b
        P[pre + "weight_g"] = gain
        P[pre + "weight_v"] = w
    w, b = _linear_default(g, 512, 512)
    P["neuconw.xyz_encoding_final.weight"], P["neuconw.xyz_encoding_final.bias"] = w, b
    P["neuconw.deviation_network.variance"] = torch.tensor(0.3)
    for l, (o, i) in enumerate(COLOR_DIMS):
        w, b = _linear_default(g, o, i)
        gain = w.norm(dim=1, keepdim=True) * (1.0 + 0.05 * jitter * torch.randn(o, 1, generator=g))
        pre = f"neuconw.color_net.lin{l}."
        P[pre + "bias"], P[pre + "weight_g"], P[pre + "weight_v"] = b, gain, w
    for name, (o, i) in (("static_linear_0", (128, 539 + n_a)), ("static_linear_1", (128, 128))):
        w, b = _linear_default(g, o, i)
        P[f"neuconw.color_net.static_encoding.{name}.weight"] = w
        P[f"neuconw.color_net.static_encoding.{name}.bias"] = b
    w, b = _linear_default(g, 512, 512)
    P["neuconw.color_net.xyz_encoding_final.weight"], P["neuconw.color_net.xyz_encoding_final.bias"] = w, b
    for l, (o, i) in enumerate(NERF_PTS):
        w, b = _linear_default(g, o, i)
        P[f"nerf.pts_linears.{l}.weight"], P[f"nerf.pts_linears.{l}.bias"] = w, b
    for l, (o, i) in enumerate([(128, 283 + n_a), (128, 128), (128, 128), (128, 128)]):
        w, b = _linear_default(g, o, i)
        P[f"nerf.apperence_encoding.static_linear_{l}.weight"] = w
        P[f"nerf.apperence_encoding.static_linear_{l}.bias"] = b
    for name, (o, i) in (("views_linears.0", (128, 283)), ("feature_linear", (256, 256)),
                         ("alpha_linear", (1, 256)), ("rgb_linear", (3, 128))):
        w, b = _linear_default(g, o, i)
        P[f"nerf.{name}.weight"], P[f"nerf.{name}.bias"] = w, b
    return P


def make_rays(n_rays: int, cfg: PathConfig, seed: int = 1, with_depth: bool = True):
    """Synthetic pinhole-camera ray batch (SURVEY.md §8d; datasets/ray_utils.py:5-52).

    400x400 camera, fx=fy=400, cx=cy=200, placed at (0,0,-3)*radius+origin looking +z;
    no +0.5 pixel offset; camera-space dirs [(i-cx)/fx, -(j-cy)/fy, -1] rotated by c2w
    then L2-normalised.  Returns dict(rays[R,10|8], ts[R] i64, label[R] f32, rgbs[R,3]).
    """
    g = torch.Generator().manual_seed(seed)
    H = W = 400
    f = 400.0
    cx = cy = 200.0
    pix = torch.randint(0, H * W, (n_rays,), generator=g)
    i = (pix % W).float()
    j = (pix // W).float()
    d_cam = torch.stack([(i - cx) / f, -(j - cy) / f, -torch.ones_like(i)], -1)
    rot = torch.diag(torch.tensor([-1.0, 1.0, -1.0]))  # 180 deg about y: camera -z -> world +z
    d = d_cam @ rot.T
    d = d / d.norm(dim=-1, keepdim=True)
    origin = torch.tensor(cfg.origin, dtype=torch.float32)
    o = (torch.tensor([0.0, 0.0, -3.0]) * cfg.radius + origin).expand(n_rays, 3)
    near = torch.full((n_rays, 1), 2.0 * cfg.radius)
    far = torch.full((n_rays, 1), 4.0 * cfg.radius)
    cols = [o, d, near, far]
    if with_depth:
        has = torch.rand(n_rays, generator=g) < 0.2
        dgt = (near + (far - near) * torch.rand(n_rays, 1, generator=g)).squeeze(1)
        dw = 2.0 * (1.0 - torch.rand(n_rays, generator=g))  # (0, 2]
        cols += [(dgt * has).unsqueeze(1), (dw * has).unsqueeze(1)]
    rays = torch.cat(cols, 1).float().contiguous()
    ts = torch.randint(0, cfg.n_vocab, (n_rays,), generator=g)
    label = torch.tensor([0.0, 1.0, 2.0, 6.0])[torch.randint(0, 4, (n_rays,), generator=g)]
    rgbs = torch.rand(n_rays, 3, generator=g)
    return dict(rays=rays, ts=ts, label=label, rgbs=rgbs)


def make_perturb_noise(n_rays: int, n_outside: int, seed: int = 7):
    """The two uniform draws the sampler consumes when perturb>0 (renderer.py:499,506-508)."""
    g = torch.Generator().manual_seed(seed)
    u_ray = torch.rand(n_rays, 1, generator=g)
    u_out = torch.rand(n_rays, max(n_outside, 1), generator=g)[:, :n_outside]
    return u_ray, u_out


def make_injected_hits(batch, cfg: PathConfig, voxel_size: float = 0.1, fine_voxel: float = 0.02, seed: int = 3):
    """Synthetic results of the two octree traces of config C3 (tools/prepare_data/generate_voxel.py:311-439 is
    Kaolin and cannot run here), INJECTED identically into the reference, the port and the CUDA path:

      sfm_near, sfm_far [R]  first-hit / last-entry depth of the SfM octree in SfM units (0 = miss), the values
                             get_near_far returns to NeuconWRenderer.get_near_far_octree (renderer.py:392-402)
      surface [R]            first-hit depth of the SDF-derived octree (0 = miss), returned to get_near_far_sdf
                             (renderer.py:431-441)

    Geometry: the ray / sphere(|x| = 0.5, unit frame) intersection, jittered; ~1/8 of the hit rays are turned
    into misses of either octree so both branches of both masks are exercised."""
    g = torch.Generator().manual_seed(seed)
    rays = batch["rays"]
    origin = torch.tensor(cfg.origin, dtype=torch.float64).float()
    o = (rays[:, 0:3] - origin) / cfg.radius
    d = rays[:, 3:6]
    b = (o * d).sum(-1)
    c = (o * o).sum(-1) - 0.25
    disc = b * b - c
    hit = disc > 0
    t_in = (-b - torch.sqrt(disc.clamp_min(0))) * cfg.radius
    t_out = (-b + torch.sqrt(disc.clamp_min(0))) * cfg.radius
    R = rays.shape[0]
    drop_a = torch.rand(R, generator=g) < 0.125
    drop_b = torch.rand(R, generator=g) < 0.125
    jit = (torch.rand(R, generator=g) - 0.5) * voxel_size
    sfm_near = torch.where(hit & ~drop_a, t_in - 0.2 * cfg.radius + jit, torch.zeros(R))
    sfm_far = torch.where(hit & ~drop_a, t_out + 0.1 * cfg.radius + jit, torch.zeros(R))
    surface = torch.where(hit & ~drop_b, t_in - 0.5 * fine_voxel * cfg.radius, torch.zeros(R))
    return dict(sfm_near=sfm_near.float(), sfm_far=sfm_far.float(), surface=surface.float(), voxel_size=voxel_size,
                fine_voxel_sfm=float(fine_voxel * cfg.radius))


def injected_near_far(hits, cfg: PathConfig, near, far):
    """renderer.py:380-456 on injected trace results, float32 torch ops in the reference's order:
    returns (near, far, sample_near, sample_far), all [R,1] in the unit-sphere frame."""
    vn, vf = hits["sfm_near"].to(near.device), hits["sfm_far"].to(near.device)
    hit = (vn > 0).reshape(-1, 1)
    near = torch.where(hit, vn.float().reshape(-1, 1) / cfg.radius, near)
    far = torch.where(hit, (vf.float().reshape(-1, 1) + hits["voxel_size"]) / cfg.radius, far)
    surf = hits["surface"].to(near.device).reshape(-1, 1)
    miss = surf <= 0
    tvs = hits["fine_voxel_sfm"]
    s_near = torch.where(miss, near, (surf - cfg.sample_range * tvs).float() / cfg.radius)
    s_far = torch.where(miss, far, (surf + cfg.sample_range * tvs).float() / cfg.radius)
    return near, far, s_near, s_far
