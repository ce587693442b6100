// Appearance-code fitting against frozen networks (include/nrw.h nrw_appearance_*): everything of a render that does not
// depend on the appearance code is computed once, by nrw_appearance_prepare, into a caller-owned cache; a fitting step
// then runs only the layers that do.
//
// The code enters the networks in two places: static_linear_0 of the colour net reads IN1 = [xf | viewPE | a] (layer
// L_CS0, code columns from 539) and static_linear_0 of the NeRF's appearance head reads FEATN = [feature | viewPE | a]
// (L_NS0, code columns from 283).  With perturb = 0 the samples, the SDF, the normals, the alphas and so the compositing
// weights do not read it.  So per sample the cache keeps U = W [x | 0] + b of both layers (fp32, the GEMM's pre-activation
// output), the [pts | normal] columns of the colour layers' input, and the weights that map the per-sample colours to
// `color`; per ray, the rest of `color` (background_rgb (1 - weights_sum), and the background colours of a NeRF without
// the appearance head).  A step computes relu(U + W_a a) (W_a: the code columns, a: the ray's code), the remaining layers
// with the existing GEMMs, and a fixed-weight sum per ray; its backward runs the data half of the same layers back to
// static_linear_0's pre-activation gradient, sums it per ray and maps the 128-wide sum to the code.  No weight gradient is
// formed.  The backward recomputes the step's forward chunk by chunk, so nothing it reads can be stale.
#include "engine.h"

namespace nrw {

static constexpr int CS0_CODE_COL = 539;   // IN1 = [xf 512 | viewPE 27 | a]
static constexpr int NS0_CODE_COL = 283;   // FEATN = [feature 256 | viewPE 27 | a]

// ---- kernels: one block of 128 threads per ray, thread n owns column n of the 128-wide layer -------------------------
// weight W[n, col] of a packed layer as the sum of its first P planes
__device__ __forceinline__ float weight_at(const Planes& W, int P, int n, int col) {
  return planes_load(W, P, (long long)n * W.ld + col);
}

// out[m, n] = relu(U[m, n] + sum_k W[n, col0 + k] a[r, k]) for the spr samples m of ray r, as P planes; with IN2.p also
// IN2[m, 128:192] = [pts 3 | normal 3 | 0] (the colour layers' direct inputs)
__global__ void __launch_bounds__(128) app_preact_kernel(const float* __restrict__ U, Planes W, int Pw, int col0,
                                                         const float* __restrict__ a, int n_a, int spr, int P, Planes out,
                                                         const float* __restrict__ pts, const float* __restrict__ nrm,
                                                         Planes IN2) {
  __shared__ float sa[128];
  const int r = blockIdx.x, n = threadIdx.x;
  if (n < n_a) sa[n] = a[(long long)r * n_a + n];
  __syncthreads();
  float v = 0.0f;
  for (int k = 0; k < n_a; ++k) v = fmaf(weight_at(W, Pw, n, col0 + k), sa[k], v);
  for (int i = 0; i < spr; ++i) {
    const long long m = (long long)r * spr + i;
    planes_store(out, P, m * out.ld + n, fmaxf(U[m * 128 + n] + v, 0.0f));
  }
  if (IN2.p) {
    for (int t = n; t < spr * 64; t += blockDim.x) {
      const long long m = (long long)r * spr + t / 64;
      const int j = t % 64;
      const float x = j < 3 ? pts[m * 3 + j] : j < 6 ? nrm[m * 3 + j - 3] : 0.0f;
      planes_store(IN2, P, m * IN2.ld + 128 + j, x);
    }
  }
}

// grad_a[r, k] += sum_n W[n, col0 + k] sum_i dpre[r * spr + i, n]: the code gradient of static_linear_0 from its
// pre-activation gradient (planes), summed over the ray's samples in sample order (no atomics: reproducible)
__global__ void __launch_bounds__(128) app_code_grad_kernel(Planes dpre, int Pd, int spr, Planes W, int Pw, int col0,
                                                            int n_a, float* __restrict__ grad_a) {
  __shared__ float sv[128];
  const int r = blockIdx.x, n = threadIdx.x;
  float acc = 0.0f;
  for (int i = 0; i < spr; ++i) acc += planes_load(dpre, Pd, ((long long)r * spr + i) * dpre.ld + n);
  sv[n] = acc;
  __syncthreads();
  if (n < n_a) {
    float g = 0.0f;
    for (int j = 0; j < 128; ++j) g = fmaf(weight_at(W, Pw, j, col0 + n), sv[j], g);
    grad_a[(long long)r * n_a + n] += g;
  }
}

// color[r, ch] += sum_i w[r * spr + i] rgb[r * spr + i, ch] over nr rays (one thread per ray and channel)
__global__ void ray_wsum_kernel(const float* __restrict__ rgb, const float* __restrict__ w, int nr, int spr,
                                float* __restrict__ color) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nr * 3) return;
  const int r = t / 3, ch = t % 3;
  float acc = 0.0f;
  for (int i = 0; i < spr; ++i) {
    const long long m = (long long)r * spr + i;
    acc = fmaf(w[m], rgb[m * 3 + ch], acc);
  }
  color[t] += acc;
}

// its transpose: d_rgb[m, ch] = w[m] g_color[m / spr, ch] for M = nr * spr rows
__global__ void ray_wbcast_kernel(const float* __restrict__ g_color, const float* __restrict__ w, long long M, int spr,
                                  float* __restrict__ d_rgb) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M * 3) return;
  const long long m = t / 3;
  d_rgb[t] = w[m] * g_color[(m / spr) * 3 + t % 3];
}

static int launch_ray_wsum(const float* rgb, const float* w, int nr, int spr, float* color, cudaStream_t s) {
  ray_wsum_kernel<<<cdiv((long long)nr * 3, 128), 128, 0, s>>>(rgb, w, nr, spr, color);
  NRW_LAUNCH_OK();
  return NRW_OK;
}
static int launch_ray_wbcast(const float* g_color, const float* w, int nr, int spr, float* d_rgb, cudaStream_t s) {
  const long long M = (long long)nr * spr;
  ray_wbcast_kernel<<<cdiv(M * 3, 256), 256, 0, s>>>(g_color, w, M, spr, d_rgb);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- cache layout --------------------------------------------------------------------------------------------------
// fp32 arrays, each 256-byte aligned.  Per SDF sample: Uc [128], pts [3], nrm [3], w_fg, sdf; per ray: cst [3]; with
// n_outside > 0 per NeRF sample: alpha, z (the merged depths); with the appearance head also Un [128] and w_bg, without it
// the NeRF's colour [3] (folded into cst by the prepare).  sdf, alpha, z and the NeRF colour are the prepare's scratch.
struct AppLayout {
  int R, S, T;
  bool bg, bg_app;
  long long Uc, pts, nrm, wfg, sdf, cst, alpha, zf, Un, wbg, bgrgb, bytes;
};
static AppLayout app_layout(const nrw_ctx& c, int R, int S, int n_outside) {
  AppLayout L{};
  L.R = R; L.S = S; L.T = S + n_outside;
  L.bg = n_outside > 0;
  L.bg_app = L.bg && c.nerf_app;
  const long long RS = (long long)R * S, RT = (long long)R * L.T;
  long long off = 0;
  auto take = [&](long long floats) { const long long o = off; off = round_up(off + floats * 4, 256); return o; };
  L.Uc = take(RS * 128); L.pts = take(RS * 3); L.nrm = take(RS * 3); L.wfg = take(RS); L.sdf = take(RS);
  L.cst = take((long long)R * 3);
  L.alpha = L.zf = L.Un = L.wbg = L.bgrgb = -1;
  if (L.bg) { L.alpha = take(RT); L.zf = take(RT); }
  if (L.bg_app) { L.Un = take(RT * 128); L.wbg = take(RT); }
  if (L.bg && !L.bg_app) L.bgrgb = take(RT * 3);
  L.bytes = off;
  return L;
}
static float* at(const void* cache, long long off) {
  return off < 0 ? nullptr : reinterpret_cast<float*>(const_cast<char*>(reinterpret_cast<const char*>(cache)) + off);
}

long long appearance_cache_bytes(const nrw_ctx& c, int R, int S, int n_outside) {
  return app_layout(c, R, S, n_outside).bytes;
}

static int app_ready(const nrw_ctx& c, int T, bool backward) {
  NRW_CHECK(c.bound && c.packed_valid, NRW_ERR_STATE, "appearance: bind a workspace and pack weights first");
  NRW_CHECK(!backward || c.with_bwd, NRW_ERR_STATE, "appearance_backward: workspace not bound for backward");
  NRW_CHECK(c.Mc >= T, NRW_ERR_WORKSPACE, "appearance: chunk_rows=%d smaller than one ray (%d)", c.Mc, T);
  return NRW_OK;
}

int appearance_prepare(nrw_ctx& c, const nrw_render_cfg& cfg, const float* o, const float* d, const float* z_vals,
                       const float* z_out, const float* sample_dist, const float* inv_s, void* cache, long long cache_bytes,
                       cudaStream_t s) {
  const int R = cfg.R, S = cfg.S, T = cfg.S + cfg.n_outside;
  NRW_TRY(app_ready(c, T, false));
  const AppLayout L = app_layout(c, R, S, cfg.n_outside);
  NRW_CHECK(cache_bytes >= L.bytes, NRW_ERR_WORKSPACE, "appearance_prepare: cache too small: %lld < %lld bytes", cache_bytes,
            L.bytes);
  const int P = c.n_planes;
  c.fwd_cached = false;   // the chunks below overwrite the forward slots of the last render
  float *Uc = at(cache, L.Uc), *pts = at(cache, L.pts), *nrm = at(cache, L.nrm), *sdf = at(cache, L.sdf);
  float *alpha = at(cache, L.alpha), *zf = at(cache, L.zf), *Un = at(cache, L.Un), *bgrgb = at(cache, L.bgrgb);
  if (L.bg) {
    NRW_TRY(launch_merge_sorted(R, S, cfg.n_outside, z_vals, z_out, zf, s));
    NRW_TRY(walk_chunks(c, c.nerf_slots, R, T, false, false, [&](FwdNerfSlot& f, bool, int r0, int nr, int M) -> int {
      // no code: FEATN's code columns are written as zeros
      NRW_TRY(nerf_chunk_forward(c, f, M, o + r0 * 3, d + r0 * 3, zf + (long long)r0 * T, sample_dist + r0, nullptr, nullptr,
                                 T, T, s));
      NRW_CUDA_OK(cudaMemcpyAsync(alpha + (long long)r0 * T, f.c_alpha, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
      if (L.bg_app) {
        Epi e; e.bias = c.bias(L_NS0); e.out_f32 = Un + (long long)r0 * T * 128; e.ld_f32 = 128;
        return mm(c, P, f.FEATN, c.W(L_NS0), M, 128, 384, e, s);
      }
      NRW_CUDA_OK(cudaMemcpyAsync(bgrgb + (long long)r0 * T * 3, f.c_rgbbg, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
      return NRW_OK;
    }));
  }
  NRW_TRY(walk_chunks(c, c.sdf_slots, R, S, false, false, [&](FwdSdfSlot& f, bool, int r0, int nr, int M) -> int {
    const long long m0 = (long long)r0 * S;
    NRW_TRY(launch_points(o + r0 * 3, d + r0 * 3, z_vals + m0, sample_dist + r0, nr, S, 1, f.PTS, s));
    NRW_TRY(sdf_chunk_forward(c, f, M, f.PTS, true, true, s));
    NRW_TRY(launch_color_embed(d + r0 * 3, nullptr, 0, S, f.PTS, f.c_nrm, M, P, f.IN1, f.IN2, s));   // code columns: 0
    { Epi e; e.bias = c.bias(L_CX); e.out_pl = f.IN1; NRW_TRY(mm(c, P, f.FEAT, c.W(L_CX), M, 512, 512, e, s)); }
    { Epi e; e.bias = c.bias(L_CS0); e.out_f32 = Uc + m0 * 128; e.ld_f32 = 128; NRW_TRY(mm(c, P, f.IN1, c.W(L_CS0), M, 128, 640, e, s)); }
    NRW_CUDA_OK(cudaMemcpyAsync(pts + m0 * 3, f.PTS, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    NRW_CUDA_OK(cudaMemcpyAsync(nrm + m0 * 3, f.c_nrm, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    NRW_CUDA_OK(cudaMemcpyAsync(sdf + m0, f.c_sdf, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
    return NRW_OK;
  }));
  nrw_render_io io{};
  io.o = o; io.d = d; io.z_vals = z_vals; io.z_out = z_out; io.sample_dist = sample_dist; io.inv_s = inv_s;
  NRW_TRY(composite_weights(cfg, io, sdf, nrm, alpha, bgrgb, at(cache, L.wfg), at(cache, L.wbg), at(cache, L.cst), s));
  c.app_caches[cache] = AppCacheDims{R, S, cfg.n_outside};
  return NRW_OK;
}

static int app_lookup(const nrw_ctx& c, const void* cache, AppLayout& L) {
  const auto it = c.app_caches.find(cache);
  NRW_CHECK(it != c.app_caches.end(), NRW_ERR_STATE, "appearance: the cache was not prepared on this context");
  L = app_layout(c, it->second.R, it->second.S, it->second.n_outside);
  return NRW_OK;
}

// the code-dependent layers of rays [r0, r0 + nr): SDF samples -> f.c_rgb, NeRF samples -> f.c_rgbbg
static int app_color_chunk(nrw_ctx& c, FwdSdfSlot& f, const AppLayout& L, const void* cache, const float* a, int r0, int nr,
                           int M, cudaStream_t s) {
  const long long m0 = (long long)r0 * L.S;
  app_preact_kernel<<<nr, 128, 0, s>>>(at(cache, L.Uc) + m0 * 128, c.W(L_CS0), c.n_planes, CS0_CODE_COL, a + (long long)r0 * c.n_a,
                                       c.n_a, L.S, c.n_planes, f.H1, at(cache, L.pts) + m0 * 3, at(cache, L.nrm) + m0 * 3, f.IN2);
  NRW_LAUNCH_OK();
  return color_chunk_tail(c, f, M, s);
}
static int app_nerf_chunk(nrw_ctx& c, FwdNerfSlot& f, const AppLayout& L, const void* cache, const float* a, int r0, int nr,
                          int M, cudaStream_t s) {
  const long long m0 = (long long)r0 * L.T;
  app_preact_kernel<<<nr, 128, 0, s>>>(at(cache, L.Un) + m0 * 128, c.W(L_NS0), c.n_planes, NS0_CODE_COL, a + (long long)r0 * c.n_a,
                                       c.n_a, L.T, c.n_planes, f.AP[1], nullptr, nullptr, Planes{nullptr, 0, 0});
  NRW_LAUNCH_OK();
  return nerf_rgb_tail(c, f, M, s);
}

int appearance_forward(nrw_ctx& c, const void* cache, const float* a_emb, float* color, cudaStream_t s) {
  AppLayout L;
  NRW_TRY(app_lookup(c, cache, L));
  NRW_TRY(app_ready(c, L.T, false));
  c.fwd_cached = false;
  NRW_CUDA_OK(cudaMemcpyAsync(color, at(cache, L.cst), (size_t)L.R * 12, cudaMemcpyDeviceToDevice, s));
  const float* wfg = at(cache, L.wfg);
  NRW_TRY(walk_chunks(c, c.sdf_slots, L.R, L.S, false, false, [&](FwdSdfSlot& f, bool, int r0, int nr, int M) -> int {
    NRW_TRY(app_color_chunk(c, f, L, cache, a_emb, r0, nr, M, s));
    return launch_ray_wsum(f.c_rgb, wfg + (long long)r0 * L.S, nr, L.S, color + r0 * 3, s);
  }));
  if (!L.bg_app) return NRW_OK;
  const float* wbg = at(cache, L.wbg);
  return walk_chunks(c, c.nerf_slots, L.R, L.T, false, false, [&](FwdNerfSlot& f, bool, int r0, int nr, int M) -> int {
    NRW_TRY(app_nerf_chunk(c, f, L, cache, a_emb, r0, nr, M, s));
    return launch_ray_wsum(f.c_rgbbg, wbg + (long long)r0 * L.T, nr, L.T, color + r0 * 3, s);
  });
}

// Each chunk recomputes its forward, then runs the data GEMMs of the same layers (ReLU-gated, c.bwd_planes) back to
// static_linear_0's pre-activation gradient.  The heads' own weight-gradient partials land in the gradient scratch c.gs,
// which every backward clears before it uses it.
int appearance_backward(nrw_ctx& c, const void* cache, const float* a_emb, const float* g_color, float* grad_a_emb,
                        cudaStream_t s) {
  AppLayout L;
  NRW_TRY(app_lookup(c, cache, L));
  NRW_TRY(app_ready(c, L.T, true));
  c.fwd_cached = false;
  const int P = c.bwd_planes;
  const Heads& H = c.pm.heads;
  NRW_CUDA_OK(cudaMemsetAsync(grad_a_emb, 0, (size_t)L.R * c.n_a * 4, s));
  const float* wfg = at(cache, L.wfg);
  NRW_TRY(walk_chunks(c, c.sdf_slots, L.R, L.S, false, false, [&](FwdSdfSlot& f, bool, int r0, int nr, int M) -> int {
    NRW_TRY(app_color_chunk(c, f, L, cache, a_emb, r0, nr, M, s));
    NRW_TRY(launch_ray_wbcast(g_color + r0 * 3, wfg + (long long)r0 * L.S, nr, L.S, c.c_dn, s));
    NRW_TRY(launch_head_bwd(3, f.X[4], P, 256, M, c.f_area + H.cl4_w, c.c_dn, f.c_rgb, nullptr, 1, c.dX[0], nullptr,
                            c.gs + H.d_cl4_w, c.gs + H.d_cl4_b, s));
    int cur = 0;
    for (int l = 3; l >= 1; --l) {
      Epi e; e.aux_relu = f.X[l].p; e.ld_relu = 256; e.out_pl = c.dX[1 - cur];
      NRW_TRY(mm(c, P, c.dX[cur], c.WT(L_CL0 + l), M, 256, 256, e, s));
      cur = 1 - cur;
    }
    { Epi e; e.aux_relu = f.IN2.p; e.ld_relu = 192; e.out_pl = c.dH2; NRW_TRY(mm(c, P, c.dX[cur], c.WT(L_CL0), M, 128, 256, e, s)); }
    { Epi e; e.aux_relu = f.H1.p; e.ld_relu = 128; e.out_pl = c.dH1; NRW_TRY(mm(c, P, c.dH2, c.WT(L_CS1), M, 128, 128, e, s)); }
    app_code_grad_kernel<<<nr, 128, 0, s>>>(c.dH1, P, L.S, c.W(L_CS0), P, CS0_CODE_COL, c.n_a, grad_a_emb + (long long)r0 * c.n_a);
    NRW_LAUNCH_OK();
    return NRW_OK;
  }));
  if (!L.bg_app) return NRW_OK;
  const float* wbg = at(cache, L.wbg);
  return walk_chunks(c, c.nerf_slots, L.R, L.T, false, false, [&](FwdNerfSlot& f, bool, int r0, int nr, int M) -> int {
    NRW_TRY(app_nerf_chunk(c, f, L, cache, a_emb, r0, nr, M, s));
    NRW_TRY(launch_ray_wbcast(g_color + r0 * 3, wbg + (long long)r0 * L.T, nr, L.T, c.c_dn, s));
    NRW_TRY(launch_head_bwd(3, f.AP[4], P, 128, M, c.f_area + H.nr_w, c.c_dn, nullptr, nullptr, 0, c.dNA[0], nullptr,
                            c.gs + H.d_nr_w, c.gs + H.d_nr_b, s));
    int cur = 0;
    for (int l = 3; l >= 1; --l) {
      Epi e; e.aux_relu = f.AP[l].p; e.ld_relu = 128; e.out_pl = c.dNA[1 - cur];
      NRW_TRY(mm(c, P, c.dNA[cur], c.WT(L_NS0 + l), M, 128, 128, e, s));
      cur = 1 - cur;
    }
    app_code_grad_kernel<<<nr, 128, 0, s>>>(c.dNA[cur], P, L.T, c.W(L_NS0), P, NS0_CODE_COL, c.n_a, grad_a_emb + (long long)r0 * c.n_a);
    NRW_LAUNCH_OK();
    return NRW_OK;
  });
}

}  // namespace nrw
