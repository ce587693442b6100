"""Held-out evaluation in the NeRF-W style: fit one appearance code per held-out photograph on the left half of its pixels
against frozen networks, then score the colour rendered on the right half (datasets/phototourism.py:726-748, metrics.py).

    AppearanceCache    the appearance-free prefix of a render of fixed rays (libnrw nrw_appearance_*); callable on codes
                       [R, n_a], differentiable in them
    fit_appearance     Adam over one code per distinct ts with the reference's colour loss (losses.py:26-27)
    evaluate_held_out  per-image and mean PSNR (metrics.py:psnr) over PhototourismDataset(split="eval")

A fitting step runs only the layers that read the code: the sampler, the SDF network, xyz_encoding_final, the NeRF trunk
and the compositing weights are computed once per cache (include/nrw.h).  The networks are frozen: nothing here changes
a network parameter, and only the fitted rows of embedding_a are written.
"""
import ctypes as C

import torch
from torch.autograd.function import once_differentiable

from ._lib import NrwError, check, ptr, stream_ptr
from .engine import make_render_cfg


def _normalised(renderer, rays):
    """renderer.render's ray normalisation (renderer.py:785-800): unit-sphere origins, near / far over the radius."""
    dev = rays.device
    if renderer.origin.device != dev:
        renderer.origin = renderer.origin.to(dev).float()
        renderer.sfm_to_gt = renderer.sfm_to_gt.to(dev).float()
    rays_o = ((rays[:, 0:3] - renderer.origin).float() / renderer.radius).float().contiguous()
    rays_d = rays[:, 3:6].float().contiguous()
    near = (rays[:, 6:7] / renderer.radius).float()
    far = (rays[:, 7:8] / renderer.radius).float()
    return rays_o, rays_d, near, far


class AppearanceCache:
    """Everything of renderer.render(rays, ts, perturb_overwrite=0)["color"] that does not depend on the appearance codes,
    computed once.  cache(codes) with codes [R, n_a] (one per ray) returns color [R, 3]; it equals the render's colour for
    those codes in embedding_a up to the split W [x | a] = W [x | 0] + W_a a, and is differentiable in the codes.

    The networks must not change while the cache is used (calling it after a parameter update raises)."""

    def __init__(self, renderer, rays, ts, background_rgb=None, cos_anneal_ratio=0.0):
        if not rays.is_cuda:
            raise NrwError("AppearanceCache: the nrw path is CUDA-only (rays are on %s)" % rays.device)
        self.renderer, self.eng = renderer, renderer.engine
        self.ts = ts
        dev = rays.device
        self.R = R = int(rays.shape[0])
        if R < 1:
            raise NrwError("AppearanceCache: no rays")
        rays_o, rays_d, near, far = _normalised(renderer, rays)
        with torch.no_grad():
            S, z_vals, z_out, sample_dist, _, _ = renderer.sparse_sampler(rays_o, rays_d, near, far, 0)
        n_out = renderer.n_outside if (renderer.render_bg and renderer.n_outside > 0) else 0
        if z_out is None:
            z_out = torch.empty(R, 0, dtype=torch.float32, device=dev)
        self.S, self.n_outside = int(S), n_out
        self.rcfg = make_render_cfg(R, S, n_out, cos_anneal_ratio, background_rgb, renderer.trim_sphere)
        self._bind(dev)
        self.token = self.eng.packed_version
        L = self.eng.L
        nbytes = int(L.nrw_appearance_cache_bytes(self.eng.ctx, R, self.S, n_out))
        if nbytes < 0:
            check(nbytes, "nrw_appearance_cache_bytes")
        self._buf = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        self.ptr = C.c_void_p((self._buf.data_ptr() + 255) // 256 * 256)
        with torch.no_grad():
            inv_s = renderer.neuconw.inv_s().detach().reshape(1).contiguous().float()
        self._inputs = (rays_o, rays_d, z_vals.contiguous(), z_out.contiguous(), sample_dist.reshape(-1).contiguous(), inv_s)
        check(L.nrw_appearance_prepare(self.eng.ctx, C.byref(self.rcfg), *[ptr(t) for t in self._inputs], self.ptr, nbytes,
                                       stream_ptr()), "nrw_appearance_prepare")

    def _bind(self, dev):
        """a workspace bound with backward that holds one ray (the cache's R is not bounded by it), weights packed"""
        self.eng.ensure(dev, 1, self.S + self.n_outside, 1)
        self.eng.pack(dev)

    def _ready(self, dev):
        self._bind(dev)
        if self.eng.packed_version != self.token:
            raise NrwError("AppearanceCache: the network parameters changed since the cache was prepared; build a new cache")

    def __call__(self, codes):
        if tuple(codes.shape) != (self.R, self.eng.n_a):
            raise NrwError(f"AppearanceCache: codes must be [{self.R}, {self.eng.n_a}], got {tuple(codes.shape)}")
        return _AppearanceFn.apply(self, codes)


class _AppearanceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cache, codes):
        a = codes.detach().contiguous().float()
        dev = a.device
        cache._ready(dev)
        color = torch.empty(cache.R, 3, dtype=torch.float32, device=dev)
        check(cache.eng.L.nrw_appearance_forward(cache.eng.ctx, cache.ptr, ptr(a), ptr(color), stream_ptr()),
              "nrw_appearance_forward")
        ctx.cache = cache
        ctx.dtype = codes.dtype
        ctx.save_for_backward(a)
        return color

    @staticmethod
    @once_differentiable
    def backward(ctx, g_color):
        cache = ctx.cache
        (a,) = ctx.saved_tensors
        cache._ready(a.device)
        g = g_color.contiguous().float()
        ga = torch.empty_like(a)
        check(cache.eng.L.nrw_appearance_backward(cache.eng.ctx, cache.ptr, ptr(a), ptr(g), ptr(ga), stream_ptr()),
              "nrw_appearance_backward")
        return None, ga.to(ctx.dtype)


def color_loss(color, target):
    """losses.py:26-27 without a mask: sum |color - target| / (n + 1e-5)"""
    return (color - target).abs().sum() / (target.shape[0] + 1e-5)


def fit_appearance(renderer, rays, ts, rgbs, steps, lr, seed=0, n_rays=None):
    """Fit one appearance code per distinct value of ts to the colours rgbs [R, 3] of rays [R, >=8] with torch.optim.Adam
    (learning rate lr, `steps` steps), starting from the current rows of renderer.embeddings["a"].  With n_rays < R the fit
    uses n_rays of the rays, drawn without replacement by a torch.Generator seeded with `seed`.  The fitted rows are written
    into embedding_a and returned ([n_codes, n_a], in ascending ts); the networks and every other row are left as they were.
    Each step is deterministic: the same inputs give bit-identical codes."""
    dev = rays.device
    ts = ts.reshape(-1).to(dev)
    rgbs = rgbs.reshape(-1, 3).to(dev).float()
    if n_rays is not None and int(n_rays) < rays.shape[0]:
        g = torch.Generator().manual_seed(int(seed))
        sel = torch.randperm(rays.shape[0], generator=g)[:int(n_rays)].to(dev)
        rays, ts, rgbs = rays[sel], ts[sel], rgbs[sel]
    emb = renderer.embeddings["a"]
    uniq, inv = torch.unique(ts, return_inverse=True)
    # rays -> codes as a one-hot product: its gradient sums each code's rays without atomics
    onehot = (inv[:, None] == torch.arange(len(uniq), device=dev)[None, :]).float()
    codes = emb.weight.detach()[uniq].clone().float().requires_grad_(True)
    cache = AppearanceCache(renderer, rays, ts)
    opt = torch.optim.Adam([codes], lr=lr)
    for _ in range(int(steps)):
        opt.zero_grad(set_to_none=True)
        loss = color_loss(cache(onehot @ codes), rgbs)
        loss.backward()
        opt.step()
    out = codes.detach()
    with torch.no_grad():
        emb.weight[uniq] = out.to(emb.weight.dtype)
    return out


def psnr(image_pred, image_gt):
    """metrics.py:psnr: -10 log10(mean squared error)"""
    return -10 * torch.log10(torch.mean((image_pred - image_gt) ** 2))


def evaluate_held_out(renderer, dataset, steps, lr, n_fit_rays, seed=0, chunk=8192):
    """For each sample of a PhototourismDataset(split="eval"): fit its code on n_fit_rays rays of the left half
    (fit_appearance with `seed`), then render the right half under no_grad, `chunk` rays at a time, with the existing
    renderer.render (perturb 0).  Returns {"psnr": [per image], "mean_psnr": float, "image_name": [...]}."""
    dev = renderer.origin.device if renderer.origin.is_cuda else torch.device("cuda", torch.cuda.current_device())
    out = {"psnr": [], "image_name": []}
    for idx in range(len(dataset)):
        smp = dataset[idx]
        fit_appearance(renderer, smp["rays_train"].to(dev), smp["ts_train"].to(dev), smp["rgbs_train_gt"].to(dev), steps, lr,
                       seed=seed, n_rays=n_fit_rays)
        rays, ts = smp["rays_eval"].to(dev), smp["ts_eval"].to(dev)
        with torch.no_grad():
            color = torch.cat([renderer.render(rays[i:i + chunk], ts[i:i + chunk], None, perturb_overwrite=0)["color"]
                               for i in range(0, rays.shape[0], chunk)])
        out["psnr"].append(float(psnr(color, smp["rgbs_eval_gt"].to(dev).float())))
        out["image_name"].append(smp["image_name"])
    out["mean_psnr"] = sum(out["psnr"]) / len(out["psnr"]) if out["psnr"] else float("nan")
    return out
