"""nn.Module mirrors of the reference networks with the reference's constructor signatures,
parameter names and shapes (checkpoint-compatible, SURVEY.md 9.4), whose forward passes run in
libnrw.so.  Only the architecture the CUDA kernels are written for is accepted: anything else
raises instead of silently falling back.

  reference                                   here
  models/neuconw.py:183-296  SDFNetwork        SDFNetwork   (lin{l}.weight_g / weight_v / bias)
  models/neuconw.py:59-170   RenderingNetwork  RenderingNetwork
  models/neuconw.py:173-179  SingleVarianceNetwork
  models/neuconw.py:299-376  NeuconW           NeuconW
  models/nerf.py:86-184      NeRF              NeRF
"""
import math
from collections import OrderedDict

import numpy as np
import torch
from torch import nn

from ._lib import NrwError


class WNLinear(nn.Module):
    """Parameters of torch.nn.utils.weight_norm(nn.Linear) under their legacy names."""

    def __init__(self, in_features, out_features, weight=None, bias=None, weight_norm=True):
        super().__init__()
        lin = nn.Linear(in_features, out_features)
        if weight is not None:
            lin.weight.data.copy_(weight)
        if bias is not None:
            lin.bias.data.copy_(bias)
        self.in_features, self.out_features = in_features, out_features
        self.bias = nn.Parameter(lin.bias.data.clone())
        if weight_norm:
            self.weight_g = nn.Parameter(lin.weight.data.norm(dim=1, keepdim=True))
            self.weight_v = nn.Parameter(lin.weight.data.clone())
        else:
            self.weight = nn.Parameter(lin.weight.data.clone())


def _engine_of(module, n_a=48):
    ref = getattr(module, "_nrw_engine", None)
    eng = ref() if ref is not None else None
    if eng is None:
        from .engine import Engine

        if isinstance(module, NeRF):
            eng = Engine(neuconw=None, nerf=module, n_a=module.in_channels_a)
        else:
            eng = Engine(neuconw=module, nerf=None, n_a=n_a)
        module._nrw_engine_strong = eng
    return eng


class SDFNetwork(nn.Module):
    def __init__(self, d_in, d_out, d_hidden, n_layers, skip_in=(4,), multires=6, bias=0.5, scale=1,
                 geometric_init=True, weight_norm=True, inside_outside=False):
        super().__init__()
        if (d_in, d_out, d_hidden, n_layers, tuple(skip_in), multires, scale, bool(weight_norm)) != \
                (3, 513, 512, 8, (4,), 6, 1, True):
            raise NrwError("SDFNetwork: the CUDA path implements d_in=3, d_out=513, d_hidden=512, n_layers=8, "
                           "skip_in=(4,), multires=6, scale=1, weight_norm=True only")
        dims = [39] + [d_hidden] * n_layers + [d_out]
        self.num_layers = len(dims)
        self.skip_in, self.scale, self.multires = tuple(skip_in), scale, multires
        for l in range(self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if (l + 1) in self.skip_in else dims[l + 1]
            w = torch.empty(out_dim, dims[l])
            b = torch.empty(out_dim)
            nn.init.kaiming_uniform_(w, a=math.sqrt(5))
            nn.init.uniform_(b, -1 / math.sqrt(dims[l]), 1 / math.sqrt(dims[l]))
            if geometric_init:  # models/neuconw.py:222-254
                if l == self.num_layers - 2:
                    sign = -1.0 if inside_outside else 1.0
                    nn.init.normal_(w, mean=sign * np.sqrt(np.pi) / np.sqrt(dims[l]), std=0.0001)
                    nn.init.constant_(b, -sign * bias)
                elif l == 0:
                    nn.init.constant_(b, 0.0)
                    nn.init.constant_(w[:, 3:], 0.0)
                    nn.init.normal_(w[:, :3], 0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif l in self.skip_in:
                    nn.init.constant_(b, 0.0)
                    nn.init.normal_(w, 0.0, np.sqrt(2) / np.sqrt(out_dim))
                    nn.init.constant_(w[:, -(dims[0] - 3):], 0.0)
                else:
                    nn.init.constant_(b, 0.0)
                    nn.init.normal_(w, 0.0, np.sqrt(2) / np.sqrt(out_dim))
            setattr(self, "lin" + str(l), WNLinear(dims[l], out_dim, w, b, weight_norm=True))


class RenderingNetwork(nn.Module):
    def __init__(self, d_feature, mode, d_in, d_out, d_hidden, n_layers, head_channels=128, in_channels_dir_a=48,
                 static_head_layers=2, weight_norm=True, multires_view=4, squeeze_out=True, encode_apperence=True):
        super().__init__()
        if (d_feature, mode, d_in, d_out, d_hidden, n_layers, head_channels, static_head_layers, bool(weight_norm),
                multires_view, bool(squeeze_out), bool(encode_apperence)) != \
                (512, "idr", 9, 3, 256, 4, 128, 2, True, 4, True, True):
            raise NrwError("RenderingNetwork: unsupported configuration for the CUDA path (see config/train.yaml COLOR_CONFIG)")
        dims = [d_in + head_channels - 3] + [d_hidden] * n_layers + [d_out]
        self.num_layers = len(dims)
        for l in range(self.num_layers - 1):
            setattr(self, "lin" + str(l), WNLinear(dims[l], dims[l + 1], weight_norm=True))
        enc = OrderedDict([("static_linear_0", nn.Linear(d_feature + in_channels_dir_a + 27, head_channels))])
        for s in range(1, static_head_layers):
            enc[f"static_linear_{s}"] = nn.Linear(head_channels, head_channels)
        self.static_encoding = nn.Sequential(enc)
        self.xyz_encoding_final = nn.Linear(d_feature, d_feature)


class SingleVarianceNetwork(nn.Module):
    def __init__(self, init_val):
        super().__init__()
        self.register_parameter("variance", nn.Parameter(torch.tensor(float(init_val))))

    def forward(self, x):
        return torch.ones([len(x), 1], device=x.device) * torch.exp(self.variance * 10.0)


class NeuconW(nn.Module):
    """models/neuconw.py:299-376.  forward(x[R,S,3+3+N_A]) -> (rgb[R,S,3], inv_s[1,1], sdf[R,S], gradients[R,S,3]).

    sdf, gradient and forward are differentiable when grad mode is on and an input tensor requires grad (gradient marks
    its x, as the reference does): every parameter, the points, the view directions and the appearance codes then
    receive gradients, computed by a CUDA backward that recomputes the query's forward.  Otherwise they are inference
    calls whose outputs carry no grad_fn (the reference's always require grad).  The outputs are the same either way.
    They are once-differentiable: a gradient of the gradient (create_graph=True, third order) raises.  The training path
    goes through NeuconWRenderer.render."""

    def __init__(self, sdfNet_config, colorNet_config, SNet_config, in_channels_a, encode_a):
        super().__init__()
        if not encode_a:
            raise NrwError("NeuconW: encode_a=False is not implemented in the CUDA path")
        self.sdfNet_config, self.colorNet_config, self.SNet_config = sdfNet_config, colorNet_config, SNet_config
        self.in_channels_a, self.encode_a = in_channels_a, encode_a
        self.sdf_net = SDFNetwork(**dict(sdfNet_config))
        self.xyz_encoding_final = nn.Linear(512, 512)  # dead parameter of the reference (neuconw.py:319); kept
        self.deviation_network = SingleVarianceNetwork(**dict(SNet_config))
        self.color_net = RenderingNetwork(**dict(colorNet_config), in_channels_dir_a=in_channels_a,
                                          encode_apperence=encode_a)

    def inv_s(self):
        return torch.exp(self.deviation_network.variance * 10.0).clamp(1e-6, 1e6).reshape(1, 1)

    def sdf(self, input_xyz):
        return _engine_of(self, self.in_channels_a).sdf(input_xyz).reshape(-1, 1)

    def gradient(self, x):
        x.requires_grad_(True)      # models/neuconw.py:285
        _, _, nrm = _engine_of(self, self.in_channels_a).neuconw_forward(x, None, None, want_rgb=False)
        return nrm

    def forward(self, x):
        n_rays, n_samples, _ = x.shape
        xyz, dirs, a = torch.split(x, [3, 3, self.in_channels_a], dim=-1)
        rgb, sdf, nrm = _engine_of(self, self.in_channels_a).neuconw_forward(
            xyz.reshape(-1, 3), dirs.reshape(-1, 3), a.reshape(n_rays * n_samples, -1))
        return (rgb.view(n_rays, n_samples, 3), self.inv_s(), sdf.view(n_rays, n_samples),
                nrm.view(n_rays, n_samples, 3))


class NeRF(nn.Module):
    """Background field, models/nerf.py:86-184 (D=8, W=256, 4-D inverted-sphere input).  With encode_appearance the
    colour branch is the 4-layer appearance head over [feature, viewPE, a]; without it (config/train_indoor.yaml,
    ENCODE_A_BG: False) it is relu(views_linears.0([feature, viewPE])), there is no apperence_encoding and the
    appearance code passed to forward is ignored."""

    def __init__(self, D=8, W=256, d_in=3, d_in_view=3, multires=0, multires_view=0, output_ch=4, skips=[4],
                 in_channels_a=48, in_channels_dir=27, encode_appearance=False, use_viewdirs=False):
        super().__init__()
        if (D, W, d_in, d_in_view, multires, multires_view, list(skips), in_channels_dir,
                bool(use_viewdirs)) != (8, 256, 4, 3, 10, 4, [4], 27, True):
            raise NrwError("NeRF: the CUDA path implements D=8, W=256, d_in=4, multires=10, multires_view=4, "
                           "skips=[4], use_viewdirs=True only")
        self.D, self.W, self.in_channels_a, self.in_channels_dir = D, W, in_channels_a, in_channels_dir
        self.input_ch, self.input_ch_view = 84, 27
        self.skips, self.use_viewdirs, self.encode_appearance = skips, use_viewdirs, bool(encode_appearance)
        self.pts_linears = nn.ModuleList(
            [nn.Linear(self.input_ch, W)] +
            [nn.Linear(W, W) if i not in skips else nn.Linear(W + self.input_ch, W) for i in range(D - 1)])
        if self.encode_appearance:
            enc = OrderedDict([("static_linear_0", nn.Linear(W + in_channels_dir + in_channels_a, W // 2))])
            for s in range(1, D // 2):
                enc[f"static_linear_{s}"] = nn.Linear(W // 2, W // 2)
            self.apperence_encoding = nn.Sequential(enc)
        # live only without the appearance head; kept either way, as the reference does (nerf.py:143)
        self.views_linears = nn.ModuleList([nn.Linear(self.input_ch_view + W, W // 2)])
        self.feature_linear = nn.Linear(W, W)
        self.alpha_linear = nn.Linear(W, 1)
        self.rgb_linear = nn.Linear(W // 2, 3)

    def forward(self, input_pts, input_views, embedding_a):
        return _engine_of(self).nerf_forward(input_pts, input_views, embedding_a)
