// extern "C" surface of libnrw.so (include/nrw.h).  No exceptions cross this boundary.
#include <stdlib.h>
#include <new>

#include "engine.h"
#include "octree.h"

using namespace nrw;

#define NRW_GUARD_BEGIN try {
#define NRW_GUARD_END                                          \
  } catch (const std::exception& e) {                          \
    set_last_error("C++ exception: %s", e.what());             \
    return NRW_ERR_ARG;                                        \
  } catch (...) {                                              \
    set_last_error("unknown C++ exception");                   \
    return NRW_ERR_ARG;                                        \
  }

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

const char* nrw_last_error(void) { return last_error_cstr(); }
int nrw_version(void) { return 100; }

int nrw_param_count(void) { return PI_COUNT; }
int nrw_param_table(int n_vocab, int n_a, nrw_param_info* out) {
  NRW_GUARD_BEGIN
  static thread_local std::vector<ParamInfo> tab;
  tab = build_param_table(n_vocab, n_a);
  for (int i = 0; i < PI_COUNT; ++i) {
    out[i].name = tab[i].name.c_str();
    out[i].rows = tab[i].rows;
    out[i].cols = tab[i].cols;
    out[i].offset = tab[i].offset;
    out[i].numel = tab[i].numel;
  }
  return NRW_OK;
  NRW_GUARD_END
}
long long nrw_param_total(int n_vocab, int n_a) {
  auto tab = build_param_table(n_vocab, n_a);
  return tab.back().offset + round_up(tab.back().numel, 4);
}

int nrw_ctx_create(nrw_ctx** out, int precision, int gemm_backend, int n_vocab, int n_a) {
  NRW_GUARD_BEGIN
  NRW_CHECK(out != nullptr, NRW_ERR_ARG, "ctx_create: out is null");
  NRW_CHECK(precision >= NRW_PRECISION_BF16 && precision <= NRW_PRECISION_MIXED, NRW_ERR_ARG,
            "ctx_create: precision must be 1 (bf16), 2 (bf16x3), 3 (bf16x6) or 4 (mixed) (got %d)", precision);
  NRW_CHECK(gemm_backend == NRW_GEMM_TCGEN05 || gemm_backend == NRW_GEMM_SIMT, NRW_ERR_ARG, "ctx_create: backend %d", gemm_backend);
  NRW_CHECK(n_a >= 1 && n_a <= 96, NRW_ERR_ARG, "ctx_create: n_a=%d unsupported (1..96)", n_a);
  nrw_ctx* c = new (std::nothrow) nrw_ctx();
  NRW_CHECK(c != nullptr, NRW_ERR_ARG, "ctx_create: out of host memory");
  const bool mixed = precision == NRW_PRECISION_MIXED;
  c->n_planes = mixed ? 2 : precision;
  c->bwd_planes = mixed ? 1 : precision;
  c->backend = gemm_backend; c->n_vocab = n_vocab; c->n_a = n_a;
  c->tab = build_param_table(n_vocab, n_a);
  c->pm = build_packed_model(c->tab, c->n_planes, true);
  *out = c;
  return NRW_OK;
  NRW_GUARD_END
}
int nrw_ctx_set_nerf_appearance(nrw_ctx* ctx, int on) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && (on == 0 || on == 1), NRW_ERR_ARG, "set_nerf_appearance: on=%d must be 0 or 1", on);
  NRW_CHECK(!ctx->bound, NRW_ERR_STATE,
            "set_nerf_appearance: call before nrw_ctx_bind (it changes the packed layout and the workspace)");
  ctx->nerf_app = on;
  ctx->pm = build_packed_model(ctx->tab, ctx->n_planes, on != 0);
  return NRW_OK;
  NRW_GUARD_END
}
int nrw_ctx_destroy(nrw_ctx* ctx) {
  delete ctx;
  return NRW_OK;
}
long long nrw_packed_bytes(const nrw_ctx* ctx) { return ctx ? ctx->pm.total_bytes : 0; }
long long nrw_workspace_bytes(const nrw_ctx* ctx, int chunk_rows, int with_backward, int max_rays, int max_T,
                              int n_slots_sdf, int n_slots_nerf) {
  if (!ctx) return 0;
  return workspace_bytes(*ctx, chunk_rows, with_backward, max_rays, max_T, n_slots_sdf, n_slots_nerf);
}
int nrw_ctx_bind(nrw_ctx* ctx, void* packed, long long packed_bytes, void* workspace, long long ws_bytes,
                 int chunk_rows, int with_backward, int max_rays, int max_T, int n_slots_sdf, int n_slots_nerf,
                 void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && packed && workspace, NRW_ERR_ARG, "ctx_bind: null argument");
  NRW_CHECK(packed_bytes >= ctx->pm.total_bytes, NRW_ERR_WORKSPACE, "ctx_bind: packed buffer %lld < %lld", packed_bytes,
            ctx->pm.total_bytes);
  NRW_CHECK((reinterpret_cast<uintptr_t>(packed) & 1023) == 0, NRW_ERR_ARG, "ctx_bind: packed buffer must be 1024B aligned");
  ctx->packed = reinterpret_cast<char*>(packed);
  ctx->bf_area = reinterpret_cast<bf16*>(ctx->packed + ctx->pm.bf16_off_bytes);
  ctx->f_area = reinterpret_cast<float*>(ctx->packed + ctx->pm.f32_off_bytes);
  NRW_CUDA_OK(cudaMemcpyAsync(ctx->packed, ctx->pm.layers, sizeof(PackedLayer) * L_COUNT, cudaMemcpyHostToDevice, S(stream)));
  NRW_CUDA_OK(cudaStreamSynchronize(S(stream)));  // pm.layers is pageable host memory
  ctx->packed_valid = false;
  return carve_workspace(*ctx, workspace, ws_bytes, chunk_rows, with_backward, max_rays, max_T, n_slots_sdf,
                         n_slots_nerf, S(stream));
  NRW_GUARD_END
}
int nrw_pack_weights(nrw_ctx* ctx, const float* params, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && ctx->packed, NRW_ERR_STATE, "pack_weights: context not bound");
  NRW_TRY(pack_weights(ctx->pm, ctx->tab, ctx->n_planes, params, ctx->packed, S(stream)));
  ctx->params = params;
  ctx->packed_valid = true;
  return NRW_OK;
  NRW_GUARD_END
}

int nrw_sdf_query(nrw_ctx* ctx, const float* pts, long long n, float* sdf, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && ctx->bound && ctx->packed_valid, NRW_ERR_STATE, "sdf_query: bind + pack first");
  if (n == 0) return NRW_OK;
  return sdf_query(*ctx, pts, n, sdf, S(stream));
  NRW_GUARD_END
}

int nrw_neuconw_forward(nrw_ctx* ctx, const float* pts, const float* dirs, const float* a, long long n, float* rgb,
                        float* sdf, float* normals, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && ctx->bound && ctx->packed_valid, NRW_ERR_STATE, "neuconw_forward: bind + pack first");
  return neuconw_query(*ctx, pts, dirs, a, n, rgb, sdf, normals, S(stream));
  NRW_GUARD_END
}

int nrw_nerf_forward(nrw_ctx* ctx, const float* pts4, const float* dirs, const float* a, long long n, float* density,
                     float* rgb, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && ctx->bound && ctx->packed_valid, NRW_ERR_STATE, "nerf_forward: bind + pack first");
  return nerf_query(*ctx, pts4, dirs, a, n, density, rgb, S(stream));
  NRW_GUARD_END
}

int nrw_neuconw_backward(nrw_ctx* ctx, const float* pts, const float* dirs, const float* a, long long n, const float* g_sdf,
                         const float* g_normals, const float* g_rgb, float* grad_params, float* grad_pts, float* grad_dirs,
                         float* grad_a, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx != nullptr && n >= 0, NRW_ERR_ARG, "neuconw_backward: null context or n=%lld < 0", n);
  NRW_CHECK(n == 0 || (pts && grad_params), NRW_ERR_ARG, "neuconw_backward: null pts or grad_params");
  NRW_CHECK(!g_rgb || (dirs && a), NRW_ERR_ARG, "neuconw_backward: g_rgb needs dirs and a");
  if (n == 0) return NRW_OK;
  NRW_CHECK(ctx->bound && ctx->packed_valid && ctx->with_bwd, NRW_ERR_STATE,
            "neuconw_backward: bind a workspace with backward and pack first");
  return neuconw_query_backward(*ctx, pts, dirs, a, n, g_sdf, g_normals, g_rgb, grad_params, grad_pts, grad_dirs, grad_a,
                                S(stream));
  NRW_GUARD_END
}

int nrw_nerf_backward(nrw_ctx* ctx, const float* pts4, const float* dirs, const float* a, long long n, const float* g_density,
                      const float* g_rgb, float* grad_params, float* grad_pts4, float* grad_dirs, float* grad_a,
                      void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx != nullptr && n >= 0, NRW_ERR_ARG, "nerf_backward: null context or n=%lld < 0", n);
  NRW_CHECK(n == 0 || (pts4 && dirs && grad_params), NRW_ERR_ARG, "nerf_backward: null pts4, dirs or grad_params");
  NRW_CHECK(!g_rgb || !ctx->nerf_app || a, NRW_ERR_ARG, "nerf_backward: g_rgb needs a (appearance head)");
  NRW_CHECK(!grad_a || ctx->nerf_app, NRW_ERR_ARG, "nerf_backward: grad_a requested from a NeRF without the appearance head");
  if (n == 0) return NRW_OK;
  NRW_CHECK(ctx->bound && ctx->packed_valid && ctx->with_bwd, NRW_ERR_STATE,
            "nerf_backward: bind a workspace with backward and pack first");
  return nerf_query_backward(*ctx, pts4, dirs, a, n, g_density, g_rgb, grad_params, grad_pts4, grad_dirs, grad_a, S(stream));
  NRW_GUARD_END
}

int nrw_samples_per_ray(const nrw_sampler_cfg* cfg, int with_fine_octree) {
  const int k = cfg->up_sample_steps;
  const int n_new = (cfg->n_importance > 0 && k > 0) ? cfg->n_importance / k : 0;
  return cfg->n_samples + k * n_new + ((with_fine_octree && cfg->boundary_samples > 0) ? cfg->boundary_samples : 0);
}

int nrw_sample(nrw_ctx* ctx, const nrw_sampler_cfg* cfg, int R, const float* o, const float* d, const float* near,
               const float* far, const float* sample_near, const float* sample_far, const float* u_ray,
               const float* u_out, float* z_vals, float* z_out, float* sample_dist, int32_t* trace_inds,
               int32_t* trace_order, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && ctx->bound && ctx->packed_valid, NRW_ERR_STATE, "sample: bind + pack first");
  NRW_CHECK(cfg->n_samples >= 2, NRW_ERR_ARG, "sample: n_samples must be >= 2");
  if (R == 0) return NRW_OK;
  return sample(*ctx, *cfg, R, o, d, near, far, sample_near, sample_far, u_ray, u_out, z_vals, z_out, sample_dist,
                trace_inds, trace_order, S(stream));
  NRW_GUARD_END
}

int nrw_upsample_round(int R, int m, int n_new, float inv_s, const float* o, const float* d, const float* z,
                       const float* sdf, float* cdf_scratch, float* z_new, float* z_merged, int32_t* inds,
                       int32_t* order, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(cdf_scratch && z_new && z_merged, NRW_ERR_ARG, "upsample_round: null output/scratch");
  if (R == 0) return NRW_OK;
  return launch_upsample_round(R, m, n_new, inv_s, o, d, z, sdf, cdf_scratch, z_new, z_merged, inds, order, S(stream));
  NRW_GUARD_END
}

int nrw_boundary_samples(int R, int S0, int nb, const float* near, const float* far, const float* z, float* out,
                         void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(S0 >= 1 && nb >= 0, NRW_ERR_ARG, "boundary_samples: S0=%d nb=%d", S0, nb);
  if (R == 0) return NRW_OK;
  NRW_CHECK(near && far && z && out, NRW_ERR_ARG, "boundary_samples: null pointer");
  return launch_boundary(R, S0, nb, near, far, z, out, S(stream));
  NRW_GUARD_END
}

int nrw_render_forward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cfg && io, NRW_ERR_ARG, "render_forward: null argument");
  if (cfg->R == 0) return NRW_OK;
  return render_forward(*ctx, *cfg, *io, S(stream));
  NRW_GUARD_END
}
int nrw_render_backward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io, const nrw_render_grads* g,
                        void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cfg && io && g && g->grad_params && g->grad_a_emb && g->grad_inv_s, NRW_ERR_ARG,
            "render_backward: null argument");
  if (cfg->R == 0) return NRW_OK;
  return render_backward(*ctx, *cfg, *io, *g, S(stream));
  NRW_GUARD_END
}

int nrw_composite_forward(const nrw_render_cfg* cfg, const nrw_render_io* io, const float* sdf, const float* nrm,
                          const float* rgb, const float* bg_alpha, const float* bg_rgb, float* scratch2, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(cfg && io && scratch2, NRW_ERR_ARG, "composite_forward: null argument");
  return composite_forward(*cfg, *io, sdf, nrm, rgb, bg_alpha, bg_rgb, scratch2, S(stream));
  NRW_GUARD_END
}
int nrw_composite_backward(const nrw_render_cfg* cfg, const nrw_render_io* io, const nrw_render_grads* g,
                           const float* nrm, float* d_sdf, float* d_nrm, float* d_rgb, float* d_bg_alpha,
                           float* d_bg_rgb, void* stream) {
  NRW_GUARD_BEGIN
  const bool bg = cfg->n_outside > 0;
  return composite_backward(*cfg, *io, *g, io->sv_sdf, nrm, io->sv_rgb, bg ? io->sv_bg_alpha : nullptr,
                            bg ? io->sv_bg_rgb : nullptr, d_sdf, d_nrm, d_rgb, d_bg_alpha, d_bg_rgb, g->grad_inv_s,
                            S(stream));
  NRW_GUARD_END
}
int nrw_network_backward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io, const float* d_sdf,
                         const float* d_normals, const float* d_rgb, const float* d_bg_alpha, const float* d_bg_rgb,
                         float* grad_params, float* grad_a_emb, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cfg && io && grad_params && grad_a_emb, NRW_ERR_ARG, "network_backward: null argument");
  NRW_CHECK(d_sdf && d_normals && d_rgb, NRW_ERR_ARG, "network_backward: null upstream gradient");
  NRW_CHECK(cfg->n_outside <= 0 || (d_bg_alpha && d_bg_rgb), NRW_ERR_ARG,
            "network_backward: n_outside=%d needs both background upstream gradients", cfg->n_outside);
  if (cfg->R == 0) return NRW_OK;
  return network_backward(*ctx, *cfg, *io, d_sdf, d_normals, d_rgb, d_bg_alpha, d_bg_rgb, grad_params, grad_a_emb,
                          S(stream));
  NRW_GUARD_END
}

long long nrw_appearance_cache_bytes(const nrw_ctx* ctx, int R, int S, int n_outside) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && R > 0 && S >= 1 && n_outside >= 0, NRW_ERR_ARG,
            "appearance_cache_bytes: null context or R=%d S=%d n_outside=%d out of range", R, S, n_outside);
  return appearance_cache_bytes(*ctx, R, S, n_outside);
  NRW_GUARD_END
}
int nrw_appearance_prepare(nrw_ctx* ctx, const nrw_render_cfg* cfg, const float* o, const float* d, const float* z_vals,
                           const float* z_out, const float* sample_dist, const float* inv_s, void* cache, long long cache_bytes,
                           void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cfg && o && d && z_vals && sample_dist && inv_s && cache, NRW_ERR_ARG, "appearance_prepare: null argument");
  NRW_CHECK(cfg->R > 0 && cfg->S >= 1 && cfg->n_outside >= 0, NRW_ERR_ARG, "appearance_prepare: R=%d S=%d n_outside=%d",
            cfg->R, cfg->S, cfg->n_outside);
  NRW_CHECK(cfg->n_outside == 0 || z_out, NRW_ERR_ARG, "appearance_prepare: n_outside=%d needs z_out", cfg->n_outside);
  NRW_CHECK((reinterpret_cast<uintptr_t>(cache) & 255) == 0, NRW_ERR_ARG, "appearance_prepare: cache must be 256B aligned");
  return appearance_prepare(*ctx, *cfg, o, d, z_vals, z_out, sample_dist, inv_s, cache, cache_bytes, S(stream));
  NRW_GUARD_END
}
int nrw_appearance_forward(nrw_ctx* ctx, const void* cache, const float* a_emb, float* color, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cache && a_emb && color, NRW_ERR_ARG, "appearance_forward: null argument");
  return appearance_forward(*ctx, cache, a_emb, color, S(stream));
  NRW_GUARD_END
}
int nrw_appearance_backward(nrw_ctx* ctx, const void* cache, const float* a_emb, const float* g_color, float* grad_a_emb,
                            void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(ctx && cache && a_emb && g_color && grad_a_emb, NRW_ERR_ARG, "appearance_backward: null argument");
  return appearance_backward(*ctx, cache, a_emb, g_color, grad_a_emb, S(stream));
  NRW_GUARD_END
}

int nrw_octree_near_far(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                        const float* rays_o, const float* rays_d, int R, const float scene_origin[3], float scale,
                        float* near, float* far, int32_t* pid, int32_t* count, void* stream) {
  NRW_GUARD_BEGIN
  if (R == 0) return NRW_OK;
  return octree_near_far(octree, prefix, pyramid_host, level, rays_o, rays_d, R, scene_origin, scale, near, far, pid,
                         count, S(stream));
  NRW_GUARD_END
}
int nrw_octree_hits(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                    const float* rays_o, const float* rays_d, int R, const float scene_origin[3], float scale,
                    const int64_t* offsets, int32_t* ray_index, int32_t* point_index, float* depth, void* stream) {
  NRW_GUARD_BEGIN
  if (R == 0) return NRW_OK;
  return octree_hits(octree, prefix, pyramid_host, level, rays_o, rays_d, R, scene_origin, scale, offsets, ray_index,
                     point_index, depth, S(stream));
  NRW_GUARD_END
}

long long nrw_octree_build_scratch_bytes(int n_points, int level, int cap_nonleaf) {
  return octree_build_scratch_bytes(n_points, level, cap_nonleaf);
}
int nrw_octree_build(const void* points, int points_are_f64, int n_points, int level, uint8_t* octree, int32_t* prefix,
                     int32_t* pyramid, int16_t* points_out, int cap_nonleaf, int cap_total, int32_t* counts_out,
                     void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(octree && prefix && pyramid && points_out && counts_out && scratch, NRW_ERR_ARG, "nrw_octree_build: null output");
  NRW_CHECK(n_points == 0 || points, NRW_ERR_ARG, "nrw_octree_build: null points");
  return octree_build(points, points_are_f64, n_points, level, octree, prefix, pyramid, points_out, cap_nonleaf, cap_total,
                      counts_out, scratch, S(stream));
  NRW_GUARD_END
}

int nrw_grad_sumsq(const float* grad, long long n, double* acc, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(acc && (n == 0 || grad), NRW_ERR_ARG, "nrw_grad_sumsq: null pointer");
  return grad_sumsq(grad, n, acc, S(stream));
  NRW_GUARD_END
}
int nrw_adam_clip_step(float* p, const float* grad, float* m, float* v, long long n, const double* sumsq, double max_norm,
                       double lr, double beta1, double beta2, double eps, int step, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(n == 0 || (p && grad && m && v), NRW_ERR_ARG, "nrw_adam_clip_step: null pointer");
  return adam_clip_step(p, grad, m, v, n, sumsq, max_norm, lr, beta1, beta2, eps, step, S(stream));
  NRW_GUARD_END
}

long long nrw_compact_scratch_bytes(long long n) { return compact_scratch_bytes(n); }
int nrw_raycache_gather(const float* cache_rays, const float* cache_rgbs, long long n_cache, const int64_t* index, int batch,
                        const int32_t* mask_labels_host, int n_mask, float* rays, float* rgbs, int64_t* ts, float* label,
                        int64_t* n_valid, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(batch == 0 || (cache_rays && cache_rgbs && index && rays && rgbs && ts && label && n_valid && scratch), NRW_ERR_ARG,
            "nrw_raycache_gather: null pointer");
  return raycache_gather(cache_rays, cache_rgbs, n_cache, index, batch, mask_labels_host, n_mask, rays, rgbs, ts, label, n_valid,
                         scratch, S(stream));
  NRW_GUARD_END
}
int nrw_threshold_compact(const float* sdf, const float* xyz, long long n, float threshold, float* out, int64_t* count,
                          void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(n == 0 || (sdf && xyz && out && count && scratch), NRW_ERR_ARG, "nrw_threshold_compact: null pointer");
  return threshold_compact(sdf, xyz, n, threshold, out, count, scratch, S(stream));
  NRW_GUARD_END
}
int nrw_grid_points_dense(int dim, const float lo[3], const float hi[3], long long i0, long long n, float* out, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(n == 0 || (lo && hi && out), NRW_ERR_ARG, "nrw_grid_points_dense: null pointer");
  return grid_points_dense(dim, lo, hi, i0, n, out, S(stream));
  NRW_GUARD_END
}
int nrw_grid_points_sparse(const int16_t* leaves, long long n_leaves, int up_times, float voxel_size, const float vol_origin[3],
                           const float scene_origin[3], float scene_radius, long long i0, long long n, float* xyz_sfm,
                           float* xyz_train, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(n == 0 || (leaves && vol_origin && scene_origin && xyz_train), NRW_ERR_ARG, "nrw_grid_points_sparse: null pointer");
  return grid_points_sparse(leaves, n_leaves, up_times, voxel_size, vol_origin, scene_origin, scene_radius, i0, n, xyz_sfm, xyz_train,
                            S(stream));
  NRW_GUARD_END
}

long long nrw_mc_scratch_bytes(int d0, int d1, int d2) {
  NRW_CHECK(d0 >= 2 && d1 >= 2 && d2 >= 2, NRW_ERR_ARG, "nrw_mc_scratch_bytes: every dimension must be >= 2 (got %d x %d x %d)", d0, d1, d2);
  return mc_scratch_bytes(d0, d1, d2);
}
int nrw_mc_count(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask, void* scratch, long long* counts,
                 void* stream) {
  NRW_GUARD_BEGIN
  return mc_count(vol, d0, d1, d2, level, mask, scratch, reinterpret_cast<int64_t*>(counts), S(stream));
  NRW_GUARD_END
}
int nrw_mc_emit(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask, const void* scratch, long long n_verts,
                long long n_faces, float* verts, float* normals, int32_t* faces, void* stream) {
  NRW_GUARD_BEGIN
  return mc_emit(vol, d0, d1, d2, level, mask, scratch, n_verts, n_faces, verts, normals, faces, S(stream));
  NRW_GUARD_END
}

long long nrw_nn_index_bytes(long long n_ref) { return nn_index_bytes(n_ref); }
int nrw_nn_build(const double* ref, long long n_ref, void* index, void* stream) {
  NRW_GUARD_BEGIN
  return nn_build(ref, n_ref, index, S(stream));
  NRW_GUARD_END
}
long long nrw_nn_query_scratch_bytes(long long n_query) { return nn_query_scratch_bytes(n_query); }
int nrw_nn_query(const void* index, long long n_ref, const double* queries, long long n_query, double* dist, int64_t* idx,
                 void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  return nn_query(index, n_ref, queries, n_query, dist, idx, scratch, S(stream));
  NRW_GUARD_END
}
long long nrw_mesh_sample_scratch_bytes(long long n_faces) { return mesh_sample_scratch_bytes(n_faces); }
int nrw_mesh_sample(const double* verts, long long n_verts, const int64_t* faces, long long n_faces, long long n_samples,
                    unsigned long long seed, double* out, int64_t* face_id, int32_t* status, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  return mesh_sample(verts, n_verts, faces, n_faces, n_samples, seed, out, face_id, status, scratch, S(stream));
  NRW_GUARD_END
}

long long nrw_raster_scratch_bytes(long long n_verts, long long n_faces, int height, int width) {
  return raster_scratch_bytes(n_verts, n_faces, height, width);
}
int nrw_raster_depth(const double* verts, long long n_verts, const int64_t* faces, long long n_faces, const double* world_to_cam,
                     double fx, double fy, double cx, double cy, int height, int width, double znear, double zfar, int cull_back,
                     float* depth, int32_t* status, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  return raster_depth(verts, n_verts, faces, n_faces, world_to_cam, fx, fy, cx, cy, height, width, znear, zfar, cull_back, depth,
                      status, scratch, S(stream));
  NRW_GUARD_END
}
long long nrw_reproject_scratch_bytes(int height, int width) { return reproject_scratch_bytes(height, width); }
int nrw_reproject_mark(const float* depth, int height, int width, double fx, double fy, double cx, double cy,
                       const double* cam_to_world, const void* index, long long n_ref, double threshold, uint8_t* visible,
                       long long* n_valid, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  return reproject_mark(depth, height, width, fx, fy, cx, cy, cam_to_world, index, n_ref, threshold, visible, n_valid, scratch,
                        S(stream));
  NRW_GUARD_END
}

long long nrw_raygen_capacity(int height, int width, double depth_percent) {
  return raygen_capacity(height, width, depth_percent);
}
long long nrw_raygen_scratch_bytes(int height, int width, int with_label, long long n_keypoints, long long out_cap) {
  return raygen_scratch_bytes(height, width, with_label, n_keypoints, out_cap);
}
int nrw_raygen_image(const nrw_raygen_cfg* cfg, const uint8_t* rgb8, const float* semantic, const double* xys,
                     const int64_t* point3d_ids, long long n_keypoints, const double* point_xyz, const double* point_error,
                     long long n_points, float* rows, float* rgbs, long long out_cap, int64_t* counts, int32_t* status,
                     void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(cfg != nullptr, NRW_ERR_ARG, "nrw_raygen_image: null cfg");
  return raygen_image(*cfg, rgb8, semantic, xys, point3d_ids, n_keypoints, point_xyz, point_error, n_points, rows, rgbs, out_cap,
                      counts, status, scratch, S(stream));
  NRW_GUARD_END
}
long long nrw_depth_range_scratch_bytes(long long n_points, int n_images) { return depth_range_scratch_bytes(n_points, n_images); }
int nrw_depth_range(const double* xyz, long long n_points, const double* w2c, int n_images, double q_lo, double q_hi, double* out,
                    int64_t* n_front, int32_t* status, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  return depth_range(xyz, n_points, w2c, n_images, q_lo, q_hi, out, n_front, status, scratch, S(stream));
  NRW_GUARD_END
}

int nrw_voxel_cast(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                   const float scene_origin[3], float scale, const double* cam_to_world, float fx, float fy, float cx,
                   float cy, int height, int width, uint8_t* visible, float* depth, int32_t* leaf, int64_t* n_hit,
                   void* stream) {
  NRW_GUARD_BEGIN
  return voxel_cast(octree, prefix, pyramid_host, level, scene_origin, scale, cam_to_world, fx, fy, cx, cy, height, width,
                    visible, depth, leaf, n_hit, S(stream));
  NRW_GUARD_END
}
int nrw_voxel_lookup(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                     const double* points, long long n_points, int32_t* leaf, int32_t* status, void* stream) {
  NRW_GUARD_BEGIN
  return voxel_lookup(octree, prefix, pyramid_host, level, points, n_points, leaf, status, S(stream));
  NRW_GUARD_END
}

int nrw_view_roi_count(const float* views, const int32_t* hw, int n_views, long long max_hw, const float scene_origin[3],
                       float radius, int64_t* counts, void* stream) {
  NRW_GUARD_BEGIN
  return view_roi_count(views, hw, n_views, max_hw, scene_origin, radius, counts, S(stream));
  NRW_GUARD_END
}
int nrw_label_static_count(const float* labels, long long n, const int32_t* ids_host, int n_ids, int64_t* count, void* stream) {
  NRW_GUARD_BEGIN
  return label_static_count(labels, n, ids_host, n_ids, count, S(stream));
  NRW_GUARD_END
}

long long nrw_gemm_test_scratch_bytes(int M, int N, int K) {
  const long long a = round_up((long long)M * K, 512), b = round_up((long long)N * K, 512);
  return (a + b) * 3 * 2 + 4096;
}
long long nrw_first_hit_scratch_bytes(long long n_queries, long long map_pixels) {
  return first_hit_scratch_bytes(n_queries, map_pixels);
}
int nrw_first_hit(const float* points, long long n_points, const double* views_host, const int32_t* boxes_host, int n_views,
                  const int32_t* q_view, const float* q_xy, long long n_queries, int64_t* hit, int32_t* status,
                  void* scratch, long long scratch_bytes, void* stream) {
  NRW_GUARD_BEGIN
  return first_hit(points, n_points, views_host, boxes_host, n_views, q_view, q_xy, n_queries, hit, status, scratch,
                   scratch_bytes, S(stream));
  NRW_GUARD_END
}
int nrw_obs_reproj_error(const double* X, const int32_t* view, const double* xy, long long n, const double* P, int n_views,
                         double* err, double* uv, void* stream) {
  NRW_GUARD_BEGIN
  return obs_reproj_error(X, view, xy, n, P, n_views, err, uv, S(stream));
  NRW_GUARD_END
}
int nrw_gemm_test(int backend, int n_planes, int mn_major, int k_slices, int M, int N, int K, const float* A,
                  const float* B, const float* bias, int act, float* D, void* scratch, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK((reinterpret_cast<uintptr_t>(scratch) & 1023) == 0, NRW_ERR_ARG, "gemm_test: scratch must be 1024B aligned");
  bf16* sp = reinterpret_cast<bf16*>(scratch);
  const long long a = round_up((long long)M * K, 512), b = round_up((long long)N * K, 512);
  // operand storage: mn_major=0: A [M,K], B [N,K];  mn_major=1: A [K,M], B [K,N]
  Planes PA{sp, a, mn_major ? M : K};
  Planes PB{sp + 3 * a, b, mn_major ? N : K};
  NRW_TRY(launch_split_planes(A, mn_major ? K : M, mn_major ? M : K, mn_major ? M : K, n_planes, PA, S(stream)));
  NRW_TRY(launch_split_planes(B, mn_major ? K : N, mn_major ? N : K, mn_major ? N : K, n_planes, PB, S(stream)));
  GemmDesc g;
  g.A = PA; g.B = PB; g.n_planes = n_planes; g.M = M; g.N = N; g.K = K; g.mn_major = mn_major; g.k_slices = k_slices;
  g.epi.bias = bias; g.epi.act = act; g.epi.out_f32 = D; g.epi.ld_f32 = N; g.epi.atomic = k_slices > 1 ? 1 : 0;
  if (getenv("NRW_GEMM_TEST_LAYER") && !mn_major && k_slices == 1 && N <= K) {
    // tuning: the SDF forward-layer store pattern (fp32 pre-activation + split planes of the activation, written over A)
    g.epi.out_f32 = nullptr; g.epi.out_pre = side_f32(D, N);
    g.epi.out_pl = PA; g.epi.n_planes = n_planes; g.epi.n_store = N;
  }
  return gemm(backend, g, S(stream));
  NRW_GUARD_END
}
int nrw_gemm_pair_test(int paired, int kind, int M, int N, int K, int Mw, int Nw, int Kw, int k_slices, const void* A,
                       const void* B, const void* dY, const void* X, const void* side_h, const float* side_f,
                       const float* rowvec, const float* colvec, float scale, int n_store, void* out_pl, float* out_f32,
                       float* out2, float* colsum, float* dW, void* stream) {
  NRW_GUARD_BEGIN
  NRW_CHECK(kind >= 0 && kind <= 3 && k_slices >= 1 && scale != 0.0f, NRW_ERR_ARG, "gemm_pair_test: kind=%d k_slices=%d", kind,
            k_slices);
  auto plane = [](const void* p, long long rows, int ld) { return Planes{reinterpret_cast<bf16*>(const_cast<void*>(p)), rows * ld, ld}; };
  GemmPair pr;
  GemmDesc& d = pr.data;
  d.A = plane(A, M, K); d.B = plane(B, N, K); d.n_planes = 1; d.M = M; d.N = N; d.K = K;
  Epi& e = d.epi;
  e.scale = scale; e.n_store = n_store; e.rowvec = rowvec; e.colvec = rowvec ? colvec : nullptr;
  if (kind == 1 || kind == 2) {   // gates from one bf16 plane of u (x 1/scale: the skip layer's input)
    e.aux_u = plane(side_h, M, N); e.aux_u_planes = 1; e.aux_u_scale = 1.0f / scale;
  }
  if (kind == 1) {
    e.aux_q = side_f ? side_f32(side_f, N) : side_f32(colvec, 0);
    e.aux_q_bcast = side_f ? 0 : 1;
    e.out2 = side_f32(out2, N);
    e.rowvec = e.colvec = nullptr;
  }
  if (kind == 2) e.aux_add = side_f32(side_f, N);
  if (kind == 3) { e.aux_relu = reinterpret_cast<const bf16*>(side_h); e.ld_relu = N; }
  if (kind == 1 && out_f32) { e.out_f32 = out_f32; e.ld_f32 = N; }
  else { e.out_pl = plane(out_pl, M, N); e.n_planes = 1; }
  if (kind != 1) e.colsum = colsum;
  GemmDesc& w = pr.dw;
  w.A = plane(dY, Kw, Mw); w.B = plane(X, Kw, Nw); w.n_planes = 1; w.M = Mw; w.N = Nw; w.K = Kw; w.mn_major = 1;
  w.k_slices = k_slices;
  w.epi.out_f32 = dW; w.epi.ld_f32 = Nw; w.epi.atomic = 1;
  if (paired) return gemm_tc_pair(pr, S(stream));
  NRW_TRY(gemm_tc(w, S(stream)));
  return gemm_tc(d, S(stream));
  NRW_GUARD_END
}
long long nrw_launch_count(void) { return g_kernel_launches; }
int nrw_gemm_timing(int enable, double* out5 /* host: ms, algorithmic FLOP, MMA FLOP, launches, algorithmic HBM bytes; may be NULL */) {
  NRW_GUARD_BEGIN
  if (out5) {
    long long n = 0;
    NRW_TRY(gemm_tc_timing_read(&out5[0], &out5[1], &out5[2], &n, &out5[4]));
    out5[3] = (double)n;
  }
  gemm_tc_timing_enable(enable != 0);
  return NRW_OK;
  NRW_GUARD_END
}
int nrw_debug_gemm_profile(void* device_buf_u64_sms_x16) {
  gemm_tc_set_profile_buffer(reinterpret_cast<unsigned long long*>(device_buf_u64_sms_x16));
  return NRW_OK;
}

}  // extern "C"
