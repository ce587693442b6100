"""Drop-in mirror of the reference's NeuconWRenderer (rendering/renderer.py:51-961): same constructor
keywords, same attributes mutated by NeuconWSystem (nerf_far_override, octree_data, fine_octree_data,
origin, radius, recontruct_path), same methods (render, sdf, rgb, get_octree) and the same 16-key
result dict, with the arithmetic executed by libnrw.so."""
import ctypes as C
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from ._lib import NrwError, check, ptr, stream_ptr
from .engine import Engine, make_render_cfg, make_sampler_cfg

# ADE20K ids of the labels the path uses (datasets/mask_utils.py:11-160)
LABEL_IDS = {"sky": 2, "tree": 4, "road": 6, "person": 12, "car": 20, "minibike": 116, "bicycle": 127}


class NeuconWRenderer:
    def __init__(self, nerf, neuconw, embeddings, n_samples, n_importance, n_outside, up_sample_steps, perturb,
                 origin, radius, s_val_base=0, spc_options=None, sample_range=None, boundary_samples=None,
                 nerf_far_override=False, render_bg=True, trim_sphere=True, save_sample=False,
                 save_step_sample=False, mesh_mask_list=None, floor_normal=False, depth_loss=False,
                 floor_labels=None, precision=None, gemm_backend=None, chunk_rows=None):
        if save_sample or save_step_sample:
            raise NrwError("save_sample / save_step_sample are debugging dumps of the reference and are not implemented")
        if floor_normal:
            raise NrwError("floor_normal=True (FLOOR_NORMAL) is not implemented in the CUDA path")
        self.nerf, self.neuconw, self.embeddings = nerf, neuconw, embeddings
        self.n_samples, self.n_importance, self.n_outside = n_samples, n_importance, n_outside
        self.up_sample_steps, self.perturb, self.s_val_base = up_sample_steps, perturb, s_val_base
        self.boundary_samples = boundary_samples
        self.nerf_far_override = nerf_far_override
        self.octree_data = None
        self.sample_range = sample_range
        self.fine_octree_data = None
        spc_options = spc_options or {}
        self.recontruct_path = spc_options.get("recontruct_path")
        self.min_track_length = spc_options.get("min_track_length")
        self.voxel_size = spc_options.get("voxel_size")
        self.sfm_to_gt = torch.eye(4, dtype=torch.float64)
        if self.recontruct_path is not None:  # renderer.py:103-110
            scene_config_path = os.path.join(self.recontruct_path, "config.yaml")
            if os.path.isfile(scene_config_path):
                import yaml

                with open(scene_config_path, "r") as f:
                    sc = yaml.load(f, Loader=yaml.FullLoader)
                origin, radius = sc["origin"], sc["radius"]
                self.sfm_to_gt = torch.from_numpy(np.array(sc["sfm2gt"]))
        self.origin = torch.from_numpy(np.array(origin, dtype=np.float64))
        self.radius = radius
        self.render_bg, self.trim_sphere = render_bg, trim_sphere
        self.floor_normal, self.floor_labels = floor_normal, floor_labels
        self.depth_loss, self.mesh_mask_list = depth_loss, mesh_mask_list
        self.save_sample = self.save_step_sample = False
        n_vocab = embeddings["a"].num_embeddings if embeddings and "a" in embeddings else 0
        n_a = embeddings["a"].embedding_dim if embeddings and "a" in embeddings else neuconw.in_channels_a
        self.engine = Engine(neuconw=neuconw, nerf=nerf, n_vocab=n_vocab, n_a=n_a, precision=precision,
                             backend=gemm_backend, chunk_rows=chunk_rows)
        self._noise_hook = None  # tests inject the two uniform draws here
        self.last_extras = {}

    # ------------------------------------------------------------------------------------------------
    def get_octree(self, device):
        """renderer.py:137-155.  Reading COLMAP's points3D.bin / the scene's config.yaml is data loading and stays
        with the caller: set `renderer.sfm_points` ([P,3], track-length filtered, generate_voxel.py:56-61) and
        `renderer.scene_config` (dict with sfm2gt, eval_bbx); the octree itself is built on the GPU (K0)."""
        pts = getattr(self, "sfm_points", None)
        cfg = getattr(self, "scene_config", None)
        if pts is None or cfg is None:
            raise NrwError("get_octree: set renderer.sfm_points ([P,3] SfM points) and renderer.scene_config "
                           "(sfm2gt, eval_bbx), or assign renderer.octree_data directly "
                           "(keys octree, scene_origin, scale, level, spc_data)")
        from .octree import make_octree_data
        return make_octree_data(cfg, pts, self.voxel_size, device=device)

    def _octree_near_far(self, od, rays_o_sfm, rays_d):
        """get_near_far (tools/prepare_data/generate_voxel.py:311-439) on the CUDA octree tracer."""
        L = _lib.lib()
        dev = rays_o_sfm.device
        R = rays_o_sfm.shape[0]
        spc = od["spc_data"]
        octree = od["octree"].to(dev).contiguous()
        prefix = spc["prefix"].to(dev).to(torch.int32).contiguous()
        pyramid = spc["pyramid"].detach().cpu().to(torch.int32).contiguous()
        so = od["scene_origin"].detach().float().cpu().reshape(3).tolist()
        near = torch.empty(R, dtype=torch.float32, device=dev)
        far = torch.empty(R, dtype=torch.float32, device=dev)
        pid = torch.empty(R, dtype=torch.int32, device=dev)
        cnt = torch.empty(R, dtype=torch.int32, device=dev)
        ro = rays_o_sfm.detach().float().contiguous()
        rd = rays_d.detach().float().contiguous()
        check(L.nrw_octree_near_far(ptr(octree), ptr(prefix), C.c_void_p(pyramid.data_ptr()), int(od["level"]),
                                    ptr(ro), ptr(rd), R, (C.c_float * 3)(*so), float(od["scale"]), ptr(near),
                                    ptr(far), ptr(pid), ptr(cnt), stream_ptr()), "nrw_octree_near_far")
        return near, far

    def get_near_far_octree(self, octree_data, rays_o, rays_d, near, far):
        """renderer.py:380-413"""
        rays_o_sfm = (rays_o * self.radius).view(-1, 3) + self.origin
        vn, vf = self._octree_near_far(octree_data, rays_o_sfm, rays_d)
        hit = (vn > 0).reshape(-1, 1)
        voxel_near = vn.reshape(-1, 1) / self.radius
        voxel_far = (vf.reshape(-1, 1) + self.voxel_size) / self.radius
        near = torch.where(hit, voxel_near, near)
        far = torch.where(hit, voxel_far, far)
        return near, far, hit

    def get_near_far_sdf(self, octree_data, rays_o, rays_d, near, far):
        """renderer.py:415-456"""
        rays_o_sfm = (rays_o * self.radius).view(-1, 3) + self.origin
        surf, _ = self._octree_near_far(octree_data, rays_o_sfm, rays_d)
        surf = surf.reshape(-1, 1)
        miss = surf <= 0
        tvs = octree_data["voxel_size"]
        vn = (surf - self.sample_range * tvs) / self.radius
        vf = (surf + self.sample_range * tvs) / self.radius
        vn = torch.where(miss, near, vn)
        vf = torch.where(miss, far, vf)
        return vn, vf, ~miss

    # ------------------------------------------------------------------------------------------------
    def sparse_sampler(self, rays_o, rays_d, near, far, perturb):
        """renderer.py:458-568 -> (n_samples, z_vals, z_vals_outside, sample_dist[R,1])"""
        dev = rays_o.device
        R = rays_o.shape[0]
        if self.nerf_far_override:
            if self.octree_data is None:
                self.octree_data = self.get_octree(dev)
            near, far, _ = self.get_near_far_octree(self.octree_data, rays_o, rays_d, near, far)
        s_near = s_far = None
        if self.fine_octree_data is not None:
            s_near, s_far, _ = self.get_near_far_sdf(self.fine_octree_data, rays_o, rays_d, near, far)
        n_out = self.n_outside if self.render_bg else 0
        scfg = make_sampler_cfg(self.n_samples, self.n_importance, self.up_sample_steps, n_out, self.s_val_base,
                                self.boundary_samples if self.fine_octree_data is not None else 0, perturb > 0)
        u_ray = u_out = None
        if perturb > 0:
            if self._noise_hook is not None:
                u_ray, u_out = self._noise_hook(R, n_out, dev)
            else:  # same two draws, same order as renderer.py:499,506-508
                u_ray = torch.rand([R, 1], device=dev)
                if n_out > 0:
                    u_out = torch.rand([R, n_out], device=dev)
        z, zo, sd, _, _ = self.engine.sample(scfg, rays_o, rays_d, near, far, s_near, s_far, u_ray, u_out)
        return z.shape[1], z, (zo if n_out > 0 else None), sd.reshape(-1, 1), near, far

    def render(self, rays, ts, label, perturb_overwrite=-1, background_rgb=None, cos_anneal_ratio=0.0):
        """renderer.py:785-916"""
        dev = rays.device
        if not rays.is_cuda:
            raise NrwError("NeuconWRenderer.render: the nrw path is CUDA-only (rays are on %s)" % dev)
        if self.origin.device != dev:
            self.origin = self.origin.to(dev).float()
            self.sfm_to_gt = self.sfm_to_gt.to(dev).float()
        rays_o, rays_d = rays[:, 0:3], rays[:, 3:6]
        near, far = rays[:, 6:7], rays[:, 7:8]
        if rays.size()[1] >= 10:
            depth_gt, depth_weight = rays[:, 8], rays[:, 9]
        else:
            depth_gt = depth_weight = torch.zeros_like(near).squeeze()
        rays_o = ((rays_o - self.origin).float() / self.radius).float().contiguous()
        rays_d = rays_d.float().contiguous()
        near = (near / self.radius).float()
        far = (far / self.radius).float()
        depth_gt = (depth_gt / self.radius).float()
        a_embedded = self.embeddings["a"](ts)
        perturb = self.perturb if perturb_overwrite < 0 else perturb_overwrite
        with torch.no_grad():
            S, z_vals, z_out, sample_dist, near, far = self.sparse_sampler(rays_o, rays_d, near, far, perturb)
        R = rays.shape[0]
        n_out = self.n_outside if (self.render_bg and self.n_outside > 0) else 0
        if z_out is None:
            z_out = torch.empty(R, 0, dtype=torch.float32, device=dev)
        rcfg = make_render_cfg(R, S, n_out, cos_anneal_ratio, background_rgb, self.trim_sphere)
        inv_s = self.neuconw.inv_s()
        out = self.engine.render(rcfg, rays_o, rays_d, z_vals, z_out, sample_dist.reshape(-1), a_embedded, inv_s)
        self.last_extras = dict(z_vals=z_vals, z_vals_outside=z_out, sample_dist=sample_dist)
        weights_sum = out["weights_sum"].reshape(-1, 1)
        if self.mesh_mask_list is not None:
            mask = torch.ones_like(near)
            for name in self.mesh_mask_list:
                mask[LABEL_IDS[name] == label] = 0
            mask_error = F.binary_cross_entropy(weights_sum.clip(1e-3, 1.0 - 1e-3), mask, reduction="none")
        else:
            mask_error = torch.zeros_like(weights_sum)
        depth = out["depth"]
        if self.depth_loss and torch.sum(depth_weight > 0) > 0:
            sfm_depth_loss = (((depth - depth_gt) ** 2) * depth_weight)[depth_weight > 0]
        else:
            sfm_depth_loss = torch.zeros_like(depth)
        zeros3 = torch.zeros_like(out["normals"])
        return {
            "color": out["color"], "color_sphere": out["color_sphere"], "color_bg": out["color_bg"],
            "s_val": 1.0 / inv_s, "cdf_fine": out["cdf"], "gradients": out["gradients"],
            "mask_error": mask_error, "weights": out["weights"], "weights_sum": weights_sum,
            "weights_max": torch.max(out["weights"], dim=-1, keepdim=True)[0],
            "gradient_error": torch.ones(1, device=dev) * out["gradient_error"],
            "inside_sphere": out["inside_sphere"], "depth": depth,
            "floor_normal_error": zeros3, "floor_y_error": zeros3.clone(), "sfm_depth_loss": sfm_depth_loss,
        }

    # ------------------------------------------------------------------------------------------------
    def sdf(self, pts):
        """renderer.py:947-949: pts [n,1,3] -> [n,1]"""
        return self.engine.sdf(pts.reshape(-1, 3)).reshape(-1, 1)

    def rgb(self, pts, rays_d, a_embedded):
        """renderer.py:951-961: [n,1,3] x3 -> [n,3]"""
        n = pts.shape[0]
        rgb, _, _ = self.engine.neuconw_forward(pts.reshape(-1, 3), rays_d.reshape(-1, 3), a_embedded.reshape(n, -1))
        return rgb.reshape(n, 3)
