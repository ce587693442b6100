"""Minimal training harness around the drop-in classes: the pieces of NeuconWSystem / train.py the hot
path needs (lightning_modules/neuconw_system.py:61-176,337-360; losses.py:21-43; utils/__init__.py:23-41;
train.py:21-25,61), without PyTorch-Lightning.  One process per GPU; data-parallel ranks reduce the
flat gradient buffer with one NCCL all-reduce."""
import math
import os

import torch
import torch.distributed as dist

from .models import NeRF, NeuconW
from .renderer import LABEL_IDS, NeuconWRenderer

_SKIP_REDUCE = os.environ.get("NRW_DIAG_SKIP_REDUCE") == "1"     # diagnosis only (scaling analysis): ranks run unsynchronised

SDF_CONFIG = dict(d_in=3, d_out=513, d_hidden=512, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1,
                  geometric_init=True, weight_norm=True, inside_outside=False)
COLOR_CONFIG = dict(d_in=9, d_feature=512, mode="idr", d_out=3, d_hidden=256, n_layers=4, head_channels=128,
                    static_head_layers=2, weight_norm=True, multires_view=4)


class NeuconWLoss(torch.nn.Module):
    """losses.py:21-43 (masks=None branch; floor term off)."""

    def __init__(self, coef=1.0, igr_weight=0.1, mask_weight=0.1, depth_weight=0.1, use_mask=True, use_depth=True):
        super().__init__()
        self.coef, self.igr_weight, self.mask_weight, self.depth_weight = coef, igr_weight, mask_weight, depth_weight
        self.use_mask, self.use_depth = use_mask, use_depth

    def forward(self, inputs, targets):
        mask_sum = float(targets.shape[0]) + 1e-5
        ret = {"color_loss": (inputs["color"] - targets).abs().sum() / mask_sum,
               "normal_loss": self.igr_weight * inputs["gradient_error"].mean()}
        if self.use_mask:
            ret["mask_error"] = self.mask_weight * inputs["mask_error"].mean()
        if self.use_depth:
            ret["sfm_depth_loss"] = self.depth_weight * inputs["sfm_depth_loss"].mean()
        return {k: self.coef * v for k, v in ret.items()}


class FusedClipAdam:
    """clip_grad_norm_(max_norm) + Adam.step (train.py:61 gradient_clip_val; utils/__init__.py:30) on flat fp32
    buffers through nrw_grad_sumsq / nrw_adam_clip_step: ONE pass over parameter, gradient and moments per buffer, the clip
    coefficient stays on the device.  Groups are (param_flat, grad_getter) pairs; all groups share one gradient norm,
    as clip_grad_norm_ over the whole parameter list does."""

    def __init__(self, lr, betas=(0.9, 0.999), eps=1e-7, max_norm=0.99):
        from . import _lib
        self._lib, self.L = _lib, _lib.lib()
        self.lr, self.betas, self.eps, self.max_norm = lr, betas, eps, max_norm
        self.step_count = 0
        self.state = {}          # id -> (m, v)
        self.acc = None
        self.param_groups = [{"lr": lr}]     # schedulers mutate this, like torch.optim

    def zero_grad(self, set_to_none=True):
        pass                      # gradients are overwritten by the backward pass

    def step(self, groups):
        """groups: list of (param tensor, grad tensor), contiguous fp32 on one device."""
        lib, L = self._lib, self.L
        groups = [(p, g) for p, g in groups if g is not None]
        if not groups:
            return
        dev = groups[0][0].device
        if self.acc is None or self.acc.device != dev:
            self.acc = torch.zeros(1, dtype=torch.float64, device=dev)
        self.acc.zero_()
        self.step_count += 1
        s = lib.stream_ptr()
        for p, g in groups:
            if not (p.is_contiguous() and g.is_contiguous() and p.dtype == torch.float32 and g.dtype == torch.float32):
                raise lib.NrwError("FusedClipAdam: parameters and gradients must be contiguous fp32")
            lib.check(L.nrw_grad_sumsq(lib.ptr(g), g.numel(), lib.ptr(self.acc), s), "nrw_grad_sumsq")
        lr = self.param_groups[0]["lr"]
        for p, g in groups:
            st = self.state.get(p.data_ptr())
            if st is None:
                st = self.state[p.data_ptr()] = (torch.zeros_like(p), torch.zeros_like(p))
            lib.check(L.nrw_adam_clip_step(lib.ptr(p), lib.ptr(g), lib.ptr(st[0]), lib.ptr(st[1]), p.numel(), lib.ptr(self.acc),
                                           float(self.max_norm), float(lr), float(self.betas[0]), float(self.betas[1]),
                                           float(self.eps), self.step_count, s), "nrw_adam_clip_step")
            torch._C._increment_version([p])       # written through the raw pointer: tell torch (and Engine.pack) it changed


class TrainSystem:
    """embedding_a + neuconw + nerf + renderer + loss + Adam, i.e. what NeuconWSystem owns."""

    def __init__(self, device, n_samples=64, n_importance=64, up_sample_steps=4, n_outside=4, s_val_base=3,
                 n_vocab=5000, n_a=48, origin=(0.0, 0.0, 0.0), radius=1.0, precision=None, chunk_rows=None,
                 batch_size=8192, world_size=1, canonical_lr=1e-4, canonical_bs=4096, anneal_end=50000,
                 igr_weight=0.0001, mask_weight=0.1, depth_weight=0.1, seed=66, fused_optimizer=True, encode_a_bg=True,
                 inside_outside=False):
        """encode_a_bg / inside_outside: NEUCONW.ENCODE_A_BG and SDF_CONFIG.inside_outside (config/train_indoor.yaml sets
        False / True: a background NeRF without appearance codes, and the SDF's geometric init flipped for a scene seen
        from inside)."""
        torch.manual_seed(seed)
        self.device = device
        self.embedding_a = torch.nn.Embedding(n_vocab, n_a).to(device)
        self.neuconw = NeuconW(dict(SDF_CONFIG, inside_outside=bool(inside_outside)), COLOR_CONFIG, dict(init_val=0.3),
                               in_channels_a=n_a, encode_a=True).to(device)
        self.nerf = NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4],
                         encode_appearance=bool(encode_a_bg), in_channels_a=n_a, in_channels_dir=27, use_viewdirs=True).to(device)
        self.renderer = NeuconWRenderer(
            nerf=self.nerf, neuconw=self.neuconw, embeddings={"a": self.embedding_a}, n_samples=n_samples,
            s_val_base=s_val_base, n_importance=n_importance, n_outside=n_outside, up_sample_steps=up_sample_steps,
            perturb=1.0, origin=list(origin), radius=radius, render_bg=True, mesh_mask_list=["sky"],
            depth_loss=True, spc_options=dict(voxel_size=0.1, recontruct_path=None, min_track_length=0),
            sample_range=16, boundary_samples=10, nerf_far_override=False, precision=precision, chunk_rows=chunk_rows)
        self.loss = NeuconWLoss(igr_weight=igr_weight, mask_weight=mask_weight, depth_weight=depth_weight)
        self.params = [p for m in (self.embedding_a, self.neuconw, self.nerf) for p in m.parameters()]
        lr = canonical_lr * (world_size * batch_size / canonical_bs)  # train.py:21-25
        # utils/__init__.py:30 Adam(eps=1e-7) + train.py:61 gradient_clip_val=0.99
        self.fused_optimizer = bool(fused_optimizer)
        if self.fused_optimizer:
            self.optimizer = FusedClipAdam(lr=lr, eps=1e-7, max_norm=0.99)
        else:
            self.optimizer = torch.optim.Adam(self.params, lr=lr, eps=1e-7, weight_decay=0)
        self.anneal_end = anneal_end
        self.global_step = 0
        self.world_size = world_size
        self.ray_mask_ids = [LABEL_IDS[n] for n in ("person", "car", "bicycle", "minibike")]

    def cos_anneal_ratio(self):
        return 1.0 if self.anneal_end == 0 else min(1.0, self.global_step / self.anneal_end)

    def forward(self, rays, ts, label):
        """NeuconWSystem.forward (neuconw_system.py:159-176)."""
        return self.renderer.render(rays, ts, label, background_rgb=torch.zeros([1, 3], device=rays.device),
                                    cos_anneal_ratio=self.cos_anneal_ratio())

    def filter_rays(self, batch):
        """RAY_MASK_LIST black list of training_step (neuconw_system.py:345-355): rays whose semantic label is person /
        car / bicycle / minibike are dropped before rendering.  Batches drawn from nrw.raycache.RayCache arrive already
        filtered and compacted on the device (key "n_valid"); anything else is filtered here with the reference's
        boolean indexing (one device->host sync for the count, as in the reference)."""
        if "n_valid" in batch or not self.ray_mask_ids:
            return batch
        label = batch["label"]
        keep = torch.ones_like(label, dtype=torch.bool)
        for i in self.ray_mask_ids:
            keep &= label != i
        return {k: (v[keep] if torch.is_tensor(v) and v.shape[:1] == label.shape[:1] else v) for k, v in batch.items()}

    def compute_grads(self, batch):
        """forward + loss + backward of one batch; every .grad becomes a view of the flat gradient buffer.
        Returns (detached loss, flat gradient of neuconw+nerf, embedding gradient)."""
        batch = self.filter_rays(batch)
        rays, rgbs, ts, label = batch["rays"], batch["rgbs"], batch["ts"], batch["label"]
        self.renderer.nerf_far_override = False       # training always reads near/far from the cache (neuconw_system.py:345)
        for p in self.params:                  # zero_grad(set_to_none=True)
            p.grad = None
        results = self.forward(rays, ts, label)
        self._mark("forward")
        loss = sum(self.loss(results, rgbs).values())
        if getattr(self, "track_metrics", False):      # device tensors, no host sync (neuconw_system.py:362-371 logs the same)
            with torch.no_grad():
                mse = ((results["color"].detach() - rgbs) ** 2).mean()
                self.last_metrics = {"loss": loss.detach(), "psnr": -10.0 * torch.log10(mse),
                                     "eikonal": results["gradient_error"].detach().mean(), "s_val": results["s_val"].detach().mean()}
        loss.backward()
        self._mark("backward")
        eng = self.renderer.engine
        flat = eng.last_flat_grad
        for k, p in eng.named_params():        # make every .grad a view of the flat gradient buffer
            shape, off, numel = eng.index[k]
            view = flat[off:off + numel].view(shape)
            if k.endswith("deviation_network.variance") and p.grad is not None:
                view.copy_(p.grad)             # reaches the parameter through torch glue (inv_s), not through the engine
            p.grad = view
        return loss.detach(), flat, self.embedding_a.weight.grad

    def reduce_grads(self, flat, emb_grad):
        """DDP semantics: gradient MEAN over ranks (per-rank loss normalisers stay per-rank, SURVEY 8e).  One collective
        for neuconw + nerf (15.6 MB flat buffer, NCCL over NVLink) and one for the dense embedding gradient."""
        if self.world_size > 1 and not _SKIP_REDUCE:
            dist.all_reduce(flat)
            flat.div_(self.world_size)
            if emb_grad is not None:
                dist.all_reduce(emb_grad)
                emb_grad.div_(self.world_size)

    def apply_grads(self, flat, emb_grad):
        eng = self.renderer.engine
        if self.fused_optimizer:
            # the flat buffers hold every neuconw / nerf parameter (the embedding slice of the table is unused there)
            self.optimizer.step([(eng.flat, flat), (self.embedding_a.weight.data, emb_grad)])
        else:
            torch.nn.utils.clip_grad_norm_(self.params, 0.99)
            self.optimizer.step()
        self._mark("optimizer")
        self.global_step += 1

    def _mark(self, name):
        ev = getattr(self, "stage_events", None)       # optional [(name, cuda event)] list for stage timing
        if ev is not None:
            ev.append((name, _rec()))

    def training_step(self, batch):
        """training_step + backward + DDP-mean all-reduce + clip(0.99) + Adam (neuconw_system.py:337-360,
        train.py:61).  Returns the detached loss tensor (device)."""
        self._mark("start")
        loss, flat, eg = self.compute_grads(batch)
        self.reduce_grads(flat, eg)
        self._mark("reduce")
        self.apply_grads(flat, eg)
        return loss


def _rec():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e
