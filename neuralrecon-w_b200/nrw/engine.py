"""Host-side engine: owns the flat parameter buffer, the libnrw context and its workspace, and the
autograd bridge for the fused render path.  PyTorch is plumbing here (device memory, streams,
autograd routing); all arithmetic of the hot path happens inside libnrw.so."""
import ctypes as C
import os
import weakref

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import NrwError, RenderCfg, RenderGrads, RenderIO, SamplerCfg, check, ptr, stream_ptr

# name -> nrw_ctx_create precision (include/nrw.h).  "mixed": bf16x3 forward, plain bf16 backward GEMMs.
PRECISIONS = {"bf16": _lib.NRW_PRECISION_BF16, "bf16x3": _lib.NRW_PRECISION_BF16X3, "bf16x6": _lib.NRW_PRECISION_BF16X6,
              "mixed": _lib.NRW_PRECISION_MIXED}


def default_precision():
    return os.environ.get("NRW_PRECISION", "bf16x3")


def default_backend():
    return _lib.NRW_GEMM_SIMT if os.environ.get("NRW_GEMM", "tcgen05").lower() == "simt" else _lib.NRW_GEMM_TCGEN05


class Engine:
    """One per (neuconw, nerf) pair and device.  Parameters of both modules become views of one flat
    fp32 buffer laid out by nrw_param_table (include/nrw.h), so the backward kernels write one flat
    gradient buffer that a single NCCL all-reduce can reduce."""

    def __init__(self, neuconw=None, nerf=None, n_vocab=0, n_a=48, precision=None, backend=None, chunk_rows=None):
        self.L = _lib.lib()
        self.neuconw = neuconw
        self.nerf = nerf
        self.n_vocab = int(n_vocab)
        self.n_a = int(n_a)
        self.precision = precision or default_precision()
        if self.precision not in PRECISIONS:
            raise NrwError(f"unknown precision {self.precision!r}; choose from {sorted(PRECISIONS)}")
        self.backend = default_backend() if backend is None else backend
        self.chunk_rows = int(chunk_rows or os.environ.get("NRW_CHUNK_ROWS", 262144))
        self.table, self.total = _lib.param_table(self.n_vocab, self.n_a)
        self.index = {name: (shape, off, numel) for name, shape, off, numel in self.table}
        self.ctx = C.c_void_p()
        check(self.L.nrw_ctx_create(C.byref(self.ctx), PRECISIONS[self.precision], self.backend, self.n_vocab, self.n_a),
              "nrw_ctx_create")
        if nerf is not None and not nerf.encode_appearance:
            check(self.L.nrw_ctx_set_nerf_appearance(self.ctx, 0), "nrw_ctx_set_nerf_appearance")
        self.flat = None
        self.packed = None
        self.workspace = None
        self.bound = (0, 0, 0, 0)
        self.last_flat_grad = None
        for m in (neuconw, nerf):
            if m is not None:
                m._nrw_engine = weakref.ref(self)

    def __del__(self):
        try:
            if self.ctx:
                self.L.nrw_ctx_destroy(self.ctx)
        except Exception:
            pass

    # ---- parameters -------------------------------------------------------------------------
    def named_params(self):
        out = []
        for prefix, mod in (("neuconw.", self.neuconw), ("nerf.", self.nerf)):
            if mod is None:
                continue
            for k, p in mod.named_parameters():
                out.append((prefix + k, p))
        return out

    def flatten(self, device):
        """(Re)establish that every parameter is a view of self.flat; cheap when already true."""
        named = self.named_params()
        if self.flat is not None and self.flat.device == device:
            base = self.flat.data_ptr()
            if all(p.data_ptr() == base + self.index[k][1] * 4 and p.device == device for k, p in named):
                return named
        flat = torch.zeros(self.total, dtype=torch.float32, device=device)
        for k, p in named:
            if k not in self.index:
                raise NrwError(f"parameter {k} is not part of the supported architecture")
            shape, off, numel = self.index[k]
            if tuple(p.shape) != tuple(shape):
                raise NrwError(f"parameter {k} has shape {tuple(p.shape)}, the CUDA path needs {shape}")
            view = flat[off:off + numel].view(shape)
            view.copy_(p.data.to(device=device, dtype=torch.float32))
            p.data = view
        self.flat = flat
        self.packed_version = None
        return named

    # ---- context / workspace ----------------------------------------------------------------
    def ensure(self, device, max_rays, max_T, with_backward, S=None, chunk_hint=0):
        """(Re)bind the workspace.  With backward enabled, as many chunk slots as the memory budget
        (NRW_SLOT_BUDGET_GB, default 70 % of free HBM) allows keep their forward activations resident so
        the backward pass does not recompute the forward of those chunks (NRW_RECOMPUTE=1: one slot each).

        Bounds only ever grow.  `max_rays x max_T` sizes the PER-RAY scratch of render / sample; point queries
        (sdf, neuconw_forward, nerf_forward) need chunk buffers only and pass `chunk_hint` (rows they would like one
        chunk to hold) instead of inflating the ray bound, so a 1M-point SDF query after a training step neither
        allocates per-ray scratch for 1M rays nor costs the training path its forward slots."""
        b = self.bound
        want_chunk = min(self.chunk_rows, ((max(int(chunk_hint), 0) + 127) // 128) * 128)
        if (self.workspace is not None and self.workspace.device == device and b[0] >= int(max_rays) and b[1] >= int(max_T)
                and b[2] >= int(with_backward) and b[3] >= min(want_chunk, 65536)):     # any bound chunk >= 64k rows serves a query
            return
        max_rays = max(int(max_rays), 1, b[0])
        max_T = max(int(max_T), 2, b[1])
        with_backward = max(int(with_backward), b[2])
        if S:
            self.bound_S = max(int(S), getattr(self, "bound_S", 0))
        # chunk: as large as configured, but never (much) larger than the whole problem
        need_rows = ((max_rays * max_T + 127) // 128) * 128
        chunk = max(min(self.chunk_rows, max(need_rows, 4096, want_chunk)), ((max_T + 127) // 128) * 128, b[3])
        with torch.cuda.device(device):
            if self.packed is None or self.packed.device != device:
                nb = self.L.nrw_packed_bytes(self.ctx)
                self.packed = torch.empty(nb + 1024, dtype=torch.uint8, device=device)
            self.workspace = None
            torch.cuda.empty_cache()
            ns_sdf = ns_nerf = 1
            if with_backward and os.environ.get("NRW_RECOMPUTE", "0") != "1":
                S_eff = getattr(self, "bound_S", 0) or max_T
                free, _total = torch.cuda.mem_get_info(device)
                budget = float(os.environ.get("NRW_SLOT_BUDGET_GB", 0)) * 2 ** 30 or 0.7 * free
                # candidate chunk sizes: the configured one, then a BALANCED one (equal rays per chunk, no nearly-empty
                # last chunk: e.g. 8192 rays x 142 samples = 4.4 chunks of 262144 rows -> 5 chunks of 232,832 rows)
                n_chunks = -(-(max_rays * max_T) // chunk)
                balanced = ((-(-max_rays // n_chunks) * max_T + 127) // 128) * 128
                best = None
                for cand in ([chunk, balanced] if balanced < chunk else [chunk]):
                    want_sdf = -(-max_rays // max(cand // S_eff, 1))
                    want_nerf = -(-max_rays // max(cand // max_T, 1))
                    fits = lambda k_sdf, k_nerf: self.L.nrw_workspace_bytes(
                        self.ctx, cand, with_backward, max_rays, max_T, k_sdf, k_nerf) <= budget
                    # as many chunks as fit (the others are recomputed in the backward), SDF slots first: an SDF chunk's
                    # forward costs more per byte of slot than a NeRF chunk's
                    k_sdf = next((k for k in range(want_sdf, 0, -1) if fits(k, 1)), 0)
                    k_nerf = next((k for k in range(want_nerf, 0, -1) if fits(k_sdf, k)), 0)
                    missing = (want_sdf - k_sdf, want_nerf - k_nerf)
                    if k_sdf and k_nerf and (best is None or missing < best[0]):
                        best = (missing, cand, k_sdf, k_nerf)
                if best is not None:
                    _, chunk, ns_sdf, ns_nerf = best
            wb = self.L.nrw_workspace_bytes(self.ctx, chunk, with_backward, max_rays, max_T, ns_sdf, ns_nerf)
            self.workspace = torch.empty(wb + 2048, dtype=torch.uint8, device=device)
            pk = (self.packed.data_ptr() + 1023) // 1024 * 1024
            ws = (self.workspace.data_ptr() + 1023) // 1024 * 1024
            check(self.L.nrw_ctx_bind(self.ctx, C.c_void_p(pk), self.packed.numel() - (pk - self.packed.data_ptr()),
                                      C.c_void_p(ws), self.workspace.numel() - (ws - self.workspace.data_ptr()),
                                      chunk, with_backward, max_rays, max_T, ns_sdf, ns_nerf, stream_ptr()),
                  "nrw_ctx_bind")
        self.bound = (max_rays, max_T, with_backward, chunk)
        self.slots = (ns_sdf, ns_nerf)
        self.packed_version = None        # the packed area may have moved / been re-created

    def pack(self, device):
        """Weight-norm materialisation + plane split of every layer (nrw_pack_weights), ONCE per parameter version:
        torch bumps the version counter of the flat buffer on every in-place update of a view (optimizer.step,
        load_state_dict, .copy_), FusedClipAdam bumps it explicitly after writing through the raw pointer."""
        named = self.flatten(device)
        # (a Parameter whose .data was re-pointed at a slice of the flat buffer keeps its OWN version counter, so the
        # per-parameter counters are part of the token: torch.optim.* steps bump those, not the flat buffer's)
        token = (self.flat.data_ptr(), self.flat._version, sum(p._version for _, p in named))
        if getattr(self, "packed_version", None) != token:
            check(self.L.nrw_pack_weights(self.ctx, ptr(self.flat), stream_ptr()), "nrw_pack_weights")
            self.packed_version = token
        return named

    # ---- operations -------------------------------------------------------------------------
    # A point query joins autograd when grad mode is on and one of its input tensors requires grad (_query_grad); the
    # parameters then receive gradients too.  Otherwise it is the inference call below, outputs without grad_fn.
    def sdf(self, pts):
        """SDF values for pts [n,3] -> [n] (NeuconWRenderer.sdf, rendering/renderer.py:947-949)."""
        if _query_grad(pts):
            return _NeuconWQueryFn.apply(self, "sdf", pts, None, None, *self._query_params(pts.device))[0]
        return self._sdf(pts)

    def neuconw_forward(self, pts, dirs, a, want_rgb=True):
        """(rgb [n,3] or None, sdf [n], normals [n,3]) of NeuconW at pts [n,3], view directions dirs [n,3] and appearance
        codes a [n,n_a] (dirs and a are read only with want_rgb)."""
        if _query_grad(pts, dirs if want_rgb else None, a if want_rgb else None):
            params = self._query_params(pts.device)
            if want_rgb:
                return tuple(_NeuconWQueryFn.apply(self, "forward", pts, dirs, a, *params))
            return (None, *_NeuconWQueryFn.apply(self, "gradient", pts, None, None, *params))
        return self._neuconw_forward(pts, dirs, a, want_rgb)

    def nerf_forward(self, pts4, dirs, a):
        """(density [n,1], rgb [n,3]) of the background NeRF at pts4 [n,4], dirs [n,3], a [n,n_a] (a is not read without
        the appearance head)."""
        if _query_grad(pts4, dirs, a if self.nerf.encode_appearance else None):
            return tuple(_NeRFQueryFn.apply(self, pts4, dirs, a, *self._query_params(pts4.device)))
        return self._nerf_forward(pts4, dirs, a)

    def _query_params(self, device):
        return [p for _, p in self.flatten(device)]

    def _sdf(self, pts):
        pts = pts.detach().reshape(-1, 3).contiguous().float()
        n, dev = pts.shape[0], pts.device
        self.ensure(dev, 1, 2, 0, chunk_hint=n)
        self.pack(dev)
        out = torch.empty(pts.shape[0], dtype=torch.float32, device=dev)
        check(self.L.nrw_sdf_query(self.ctx, ptr(pts), pts.shape[0], ptr(out), stream_ptr()), "nrw_sdf_query")
        return out

    def _neuconw_forward(self, pts, dirs, a, want_rgb=True):
        pts = pts.detach().reshape(-1, 3).contiguous().float()
        n, dev = pts.shape[0], pts.device
        self.ensure(dev, 1, 2, 0, chunk_hint=n)
        self.pack(dev)
        sdf = torch.empty(n, dtype=torch.float32, device=dev)
        nrm = torch.empty(n, 3, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev) if want_rgb else None
        dirs_c = dirs.detach().reshape(-1, 3).contiguous().float() if want_rgb else None
        a_c = a.detach().reshape(n, -1).contiguous().float() if want_rgb else None
        check(self.L.nrw_neuconw_forward(self.ctx, ptr(pts), ptr(dirs_c), ptr(a_c), n, ptr(rgb), ptr(sdf), ptr(nrm),
                                         stream_ptr()), "nrw_neuconw_forward")
        return rgb, sdf, nrm

    def _nerf_forward(self, pts4, dirs, a):
        pts4 = pts4.detach().reshape(-1, 4).contiguous().float()
        n, dev = pts4.shape[0], pts4.device
        self.ensure(dev, 1, 2, 0, chunk_hint=n)
        self.pack(dev)
        dens = torch.empty(n, 1, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
        # without the appearance head the code is not read (it may be None)
        a_c = a.detach().reshape(n, -1).contiguous().float() if self.nerf.encode_appearance else None
        check(self.L.nrw_nerf_forward(self.ctx, ptr(pts4), ptr(dirs.detach().reshape(-1, 3).contiguous().float()),
                                      ptr(a_c), n, ptr(dens), ptr(rgb), stream_ptr()), "nrw_nerf_forward")
        return dens, rgb

    def sample(self, scfg, o, d, near, far, s_near=None, s_far=None, u_ray=None, u_out=None, trace=False):
        R, dev = o.shape[0], o.device
        fine = s_near is not None
        S = self.L.nrw_samples_per_ray(C.byref(scfg), int(fine))
        self.ensure(dev, R, S + scfg.n_outside, self.bound[2])
        self.pack(dev)
        z = torch.empty(R, S, dtype=torch.float32, device=dev)
        zo = torch.empty(R, max(scfg.n_outside, 0), dtype=torch.float32, device=dev)
        sd = torch.empty(R, dtype=torch.float32, device=dev)
        ti = to = None
        if trace and scfg.n_importance > 0:
            k = scfg.up_sample_steps
            n_new = scfg.n_importance // k
            ti = torch.zeros(k * R * n_new, dtype=torch.int32, device=dev)
            tot = sum(R * (scfg.n_samples + (i + 1) * n_new) for i in range(k))
            to = torch.zeros(tot, dtype=torch.int32, device=dev)
        c = lambda t: None if t is None else t.detach().reshape(-1).contiguous().float()
        args = [c(o.reshape(-1)), c(d.reshape(-1)), c(near), c(far), c(s_near), c(s_far), c(u_ray), c(u_out)]
        check(self.L.nrw_sample(self.ctx, C.byref(scfg), R, *[ptr(t) for t in args], ptr(z), ptr(zo), ptr(sd),
                                ptr(ti), ptr(to), stream_ptr()), "nrw_sample")
        return z, zo, sd, ti, to

    def render(self, rcfg, o, d, z_vals, z_out, sample_dist, a_emb, inv_s):
        """Differentiable fused render core.  Returns a dict of tensors (see _RenderFn)."""
        dev = o.device
        need_grad = torch.is_grad_enabled()
        T = rcfg.S + rcfg.n_outside
        self.ensure(dev, rcfg.R, T, int(need_grad), S=rcfg.S)
        named = self.pack(dev)
        params = [p for _, p in named]
        outs = _RenderFn.apply(self, rcfg, o, d, z_vals, z_out, sample_dist, a_emb, inv_s, *params)
        keys = ["color", "color_sphere", "color_bg", "cdf", "gradients", "weights", "weights_sum", "inside_sphere",
                "depth", "normals", "gradient_error"]
        return dict(zip(keys, outs))


def _io_struct(tensors):
    io = RenderIO()
    for k in _lib._IO_FIELDS:
        setattr(io, k, ptr(tensors.get(k)))
    return io


_OUT_KEYS = ("color", "color_sphere", "color_bg", "cdf", "gradients", "weights", "weights_sum", "inside_sphere",
             "depth", "normals", "gradient_error")


class _RenderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, rcfg, o, d, z_vals, z_out, sample_dist, a_emb, inv_s, *params):
        dev = o.device
        R, S, n_o = rcfg.R, rcfg.S, rcfg.n_outside
        T = S + n_o
        f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        t = dict(o=o.contiguous(), d=d.contiguous(), z_vals=z_vals.contiguous(), z_out=z_out.contiguous(),
                 sample_dist=sample_dist.contiguous(), a_emb=a_emb.detach().contiguous(),
                 inv_s=inv_s.detach().reshape(1).contiguous().float(),
                 color=f(R, 3), color_sphere=f(R, 3), color_bg=f(R, 3), cdf=f(R, S), gradients=f(R, S, 3),
                 weights=f(R, T), weights_sum=f(R), inside_sphere=f(R, S), depth=f(R), normals=f(R, 3),
                 gradient_error=f(1), sv_sdf=f(R, S), sv_rgb=f(R, S, 3), sv_bg_alpha=f(R, T), sv_bg_rgb=f(R, T, 3),
                 sv_z_feed=f(R, T), sv_relax_sum=f(1))
        io = _io_struct(t)
        # generation stamp: the forward activations live in the context's shared slots; render_backward only trusts them
        # when the stamp matches (two grad-enabled renders followed by backward of the first -> recompute path)
        eng.generation = getattr(eng, "generation", 0) + 1
        rcfg.reserved0 = eng.generation
        check(eng.L.nrw_render_forward(eng.ctx, C.byref(rcfg), C.byref(io), stream_ptr()), "nrw_render_forward")
        # The returned tensors must NOT sit in ctx.__dict__: output -> grad_fn -> ctx -> output is a cycle through
        # C++ that Python's gc cannot break (it kept every step's ctx, its tensors and the engine alive).
        # save_for_backward is the cycle-safe way to keep outputs.
        ctx.out_keys = _OUT_KEYS
        ctx.save_for_backward(*[t[k] for k in _OUT_KEYS])
        ctx.eng, ctx.rcfg, ctx.t = eng, rcfg, {k: v for k, v in t.items() if k not in _OUT_KEYS}
        ctx.inv_s_shape = inv_s.shape
        ctx.n_params = len(params)
        ctx.param_meta = [(p.shape, eng.index[k][1], eng.index[k][2]) for (k, _), p in zip(eng.named_params(), params)]
        ctx.mark_non_differentiable(t["inside_sphere"])
        ctx.set_materialize_grads(False)
        return (t["color"], t["color_sphere"], t["color_bg"], t["cdf"], t["gradients"], t["weights"],
                t["weights_sum"], t["inside_sphere"], t["depth"], t["normals"], t["gradient_error"])

    @staticmethod
    def backward(ctx, g_color, g_cs, g_cb, g_cdf, g_grad, g_w, g_ws, g_inside, g_depth, g_normals, g_ge):
        if ctx.t is None:
            raise NrwError("render backward called twice (retain_graph is not supported: the saved per-sample "
                           "tensors are released after the first backward)")
        eng, rcfg = ctx.eng, ctx.rcfg
        t = dict(ctx.t)
        t.update(zip(ctx.out_keys, ctx.saved_tensors))
        dev = t["o"].device
        if eng.bound[2] < 1:
            raise NrwError("render was run under no_grad; cannot backpropagate through it")
        c = lambda g: None if g is None else g.contiguous().float()
        gs = dict(g_color=c(g_color), g_color_sphere=c(g_cs), g_color_bg=c(g_cb), g_cdf=c(g_cdf), g_gradients=c(g_grad),
                  g_weights=c(g_w), g_weights_sum=c(g_ws), g_depth=c(g_depth), g_normals=c(g_normals),
                  g_gradient_error=c(g_ge))
        flat_grad = torch.zeros(eng.total, dtype=torch.float32, device=dev)
        g_a = torch.empty(rcfg.R, eng.n_a, dtype=torch.float32, device=dev)
        g_invs = torch.zeros(1, dtype=torch.float32, device=dev)
        gr = RenderGrads()
        for k, v in gs.items():
            setattr(gr, k, ptr(v))
        gr.grad_params, gr.grad_a_emb, gr.grad_inv_s = ptr(flat_grad), ptr(g_a), ptr(g_invs)
        io = _io_struct(t)
        check(eng.L.nrw_render_backward(eng.ctx, C.byref(rcfg), C.byref(io), C.byref(gr), stream_ptr()),
              "nrw_render_backward")
        eng.last_flat_grad = flat_grad
        ctx.t = None            # release the per-sample saved tensors now, not when the graph is collected
        ctx.eng = None
        pgrads = [flat_grad[off:off + numel].view(shape) for shape, off, numel in ctx.param_meta]
        return (None, None, None, None, None, None, None, g_a, g_invs.reshape(ctx.inv_s_shape), *pgrads)


def _query_grad(*inputs):
    """does a point query join autograd: grad mode on and some input tensor requiring grad."""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in inputs)


def _flat(t, cols):
    return None if t is None else t.detach().reshape(-1, cols).contiguous().float()


def _param_grads(flat_grad, meta):
    return [flat_grad[off:off + numel].view(shape) for shape, off, numel in meta]


def _input_grad(g, like):
    """a gradient in the shape and dtype of its input (like = (shape, dtype))."""
    return None if g is None else g.view(like[0]).to(like[1])


class _QueryFn(torch.autograd.Function):
    """Shared plumbing of the point-query Functions.  The forward is the inference call, so its outputs equal a call under
    no_grad.  Only the inputs are saved: the backward recomputes the query's forward chunk by chunk inside libnrw, so a
    render or another query in between cannot leave it stale activations.  It differentiates the per-layer chain at the
    parameters as packed when the backward runs.  Once-differentiable: differentiating the backward raises."""

    @staticmethod
    def _setup(ctx, eng, params, inputs):
        ctx.eng = eng
        ctx.like = [None if t is None else (t.shape, t.dtype) for t in inputs]
        ctx.param_meta = [(p.shape, eng.index[k][1], eng.index[k][2]) for (k, _), p in zip(eng.named_params(), params)]
        ctx.set_materialize_grads(False)

    @staticmethod
    def _refuse_create_graph():
        # the backward runs with grad mode on only under create_graph=True; its result would be a constant, so a gradient
        # of it (e.g. an eikonal term written as autograd.grad(sdf, x, create_graph=True)) would silently vanish
        if torch.is_grad_enabled():
            raise NrwError("NeuconW / NeRF point queries are once-differentiable: their backward cannot be differentiated "
                           "(create_graph=True); use NeuconW.gradient(x) for the SDF's gradient")

    @staticmethod
    def _bind(eng, dev, n):
        eng.ensure(dev, 1, 2, 1, chunk_hint=n)     # bound for backward; the ray bound does not grow
        eng.pack(dev)
        return torch.zeros(eng.total, dtype=torch.float32, device=dev)


class _NeuconWQueryFn(_QueryFn):
    """NeuconW queries: kind "sdf" -> (sdf,), "gradient" -> (sdf, normals), "forward" -> (rgb, sdf, normals)."""

    @staticmethod
    def forward(ctx, eng, kind, pts, dirs, a, *params):
        if kind == "sdf":
            outs = (eng._sdf(pts),)
        else:
            rgb, sdf, nrm = eng._neuconw_forward(pts, dirs, a, want_rgb=kind == "forward")
            outs = (sdf, nrm) if rgb is None else (rgb, sdf, nrm)
        ctx.kind = kind
        _QueryFn._setup(ctx, eng, params, (pts, dirs, a))
        ctx.save_for_backward(_flat(pts, 3), _flat(dirs, 3), None if a is None else _flat(a, eng.n_a))
        return outs

    @staticmethod
    def backward(ctx, *grads):
        _QueryFn._refuse_create_graph()
        return _NeuconWQueryFn._backward(ctx, *grads)

    @staticmethod
    @once_differentiable
    def _backward(ctx, *grads):
        eng = ctx.eng
        pts, dirs, a = ctx.saved_tensors
        names = {"sdf": ("sdf",), "gradient": ("sdf", "normals"), "forward": ("rgb", "sdf", "normals")}[ctx.kind]
        up = dict(zip(names, grads))
        n, dev = pts.shape[0], pts.device
        c = lambda k, cols: _flat(up.get(k), cols)
        g_sdf, g_nrm, g_rgb = c("sdf", 1), c("normals", 3), c("rgb", 3)
        need = ctx.needs_input_grad
        f = lambda want, cols: torch.empty(n, cols, dtype=torch.float32, device=dev) if want else None
        gp, gd, ga = f(need[2], 3), f(need[3], 3), f(need[4], eng.n_a)
        flat_grad = _QueryFn._bind(eng, dev, n)
        if n:
            check(eng.L.nrw_neuconw_backward(eng.ctx, ptr(pts), ptr(dirs), ptr(a), n, ptr(g_sdf), ptr(g_nrm), ptr(g_rgb),
                                             ptr(flat_grad), ptr(gp), ptr(gd), ptr(ga), stream_ptr()),
                  "nrw_neuconw_backward")
        x_pts, x_dirs, x_a = ctx.like
        return (None, None, _input_grad(gp, x_pts), _input_grad(gd, x_dirs), _input_grad(ga, x_a),
                *_param_grads(flat_grad, ctx.param_meta))


class _NeRFQueryFn(_QueryFn):
    """NeRF.forward: (density [n,1], rgb [n,3]).  Without the appearance head the code gets no gradient."""

    @staticmethod
    def forward(ctx, eng, pts4, dirs, a, *params):
        dens, rgb = eng._nerf_forward(pts4, dirs, a)
        _QueryFn._setup(ctx, eng, params, (pts4, dirs, a))
        app = eng.nerf.encode_appearance
        ctx.save_for_backward(_flat(pts4, 4), _flat(dirs, 3), _flat(a, eng.n_a) if app else None)
        return dens, rgb

    @staticmethod
    def backward(ctx, g_dens, g_rgb):
        _QueryFn._refuse_create_graph()
        return _NeRFQueryFn._backward(ctx, g_dens, g_rgb)

    @staticmethod
    @once_differentiable
    def _backward(ctx, g_dens, g_rgb):
        eng = ctx.eng
        pts4, dirs, a = ctx.saved_tensors
        n, dev = pts4.shape[0], pts4.device
        need = ctx.needs_input_grad
        f = lambda want, cols: torch.empty(n, cols, dtype=torch.float32, device=dev) if want else None
        gp, gd = f(need[1], 4), f(need[2], 3)
        ga = f(need[3] and a is not None, eng.n_a)
        flat_grad = _QueryFn._bind(eng, dev, n)
        if n:
            check(eng.L.nrw_nerf_backward(eng.ctx, ptr(pts4), ptr(dirs), ptr(a), n, ptr(_flat(g_dens, 1)),
                                          ptr(_flat(g_rgb, 3)), ptr(flat_grad), ptr(gp), ptr(gd), ptr(ga), stream_ptr()),
                  "nrw_nerf_backward")
        x_pts, x_dirs, x_a = ctx.like
        return (None, _input_grad(gp, x_pts), _input_grad(gd, x_dirs), _input_grad(ga, x_a),
                *_param_grads(flat_grad, ctx.param_meta))


def make_sampler_cfg(n_samples, n_importance, up_sample_steps, n_outside, s_val_base, boundary_samples, perturb):
    return SamplerCfg(int(n_samples), int(n_importance), int(up_sample_steps), int(n_outside), int(s_val_base),
                      int(boundary_samples or 0), int(bool(perturb)))


def make_render_cfg(R, S, n_outside, cos_anneal_ratio, background_rgb, trim_sphere):
    cfg = RenderCfg()
    cfg.R, cfg.S, cfg.n_outside = int(R), int(S), int(n_outside)
    cfg.cos_anneal_ratio = float(cos_anneal_ratio)
    # device pointer; the caller keeps `background_rgb` alive (it is stashed on the cfg object)
    cfg._bg_keepalive = None
    if background_rgb is not None:
        cfg._bg_keepalive = background_rgb.detach().reshape(-1)[:3].contiguous().float()
        cfg.background_rgb = cfg._bg_keepalive.data_ptr()
    else:
        cfg.background_rgb = None
    cfg.trim_sphere = int(bool(trim_sphere))
    return cfg
