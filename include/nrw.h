/* nrw.h - C ABI of the H100-native NeuralRecon-W per-ray training core (libnrw.so).
 *
 * The reference (zju3dv/NeuralRecon-W) is pure Python: its seam for this path is the
 * duck-typed Python object NeuconWRenderer (rendering/renderer.py:51-961) plus the
 * nn.Modules NeuconW (models/neuconw.py:299-376) and NeRF (models/nerf.py:86-184).  This
 * header declares what a reference-side binding (ctypes, see INTEGRATION.md) would bind for
 * each of those entry points.  Conventions:
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless marked host;
 *   - the caller (PyTorch) owns all memory; the library never allocates device memory;
 *     scratch is passed in through nrw_ctx_bind and sized by nrw_*_bytes();
 *   - every call is asynchronous on the cudaStream_t passed as `stream` (a void*);
 *   - return 0 (NRW_OK) or a negative nrw_status; message via nrw_last_error() (thread-local);
 *   - one process per GPU; a context is bound to the device current at creation.
 */
#ifndef NRW_H_
#define NRW_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define NRW_API __attribute__((visibility("default")))
#else
#define NRW_API
#endif

typedef enum {
  NRW_OK = 0,
  NRW_ERR_ARG = -1,       /* bad argument / unsupported configuration */
  NRW_ERR_CUDA = -2,      /* CUDA runtime or driver error */
  NRW_ERR_WORKSPACE = -3, /* bound workspace / packed-weight buffer too small */
  NRW_ERR_STATE = -4      /* call order violated (e.g. render before pack) */
} nrw_status;

typedef struct nrw_ctx nrw_ctx;

/* GEMM backends: 0 = wgmma tensor cores (product path; the name NRW_GEMM_TCGEN05 is historical), 1 = fp32 CUDA cores (verification). */
#define NRW_GEMM_TCGEN05 0
#define NRW_GEMM_SIMT 1

NRW_API const char* nrw_last_error(void);
NRW_API int nrw_version(void);

/* ---- parameter layout ------------------------------------------------------------------
 * All trainable tensors of NeuconWSystem (embedding_a, neuconw, nerf; SURVEY.md 9.4 /
 * lightning_modules/neuconw_system.py:74-103) live in ONE flat fp32 buffer; gradients in a
 * second buffer with the same layout (single NCCL all-reduce).  The table below is the
 * single source of truth for names / shapes / offsets (in floats). */
typedef struct {
  const char* name; /* reference state_dict key, e.g. "neuconw.sdf_net.lin0.weight_v" */
  int rows, cols;   /* cols == 0 for 1-D tensors, rows == cols == 0 for scalars */
  long long offset; /* float offset into the flat buffer */
  long long numel;
} nrw_param_info;
NRW_API int nrw_param_count(void);
NRW_API int nrw_param_table(int n_vocab, int n_a, nrw_param_info* out /* host, nrw_param_count() */);
NRW_API long long nrw_param_total(int n_vocab, int n_a);

/* ---- context ---------------------------------------------------------------------------
 * precision: how every fp32 GEMM operand is split into bf16 planes (values 1..3 are the plane count).
 *   NRW_PRECISION_BF16    forward and backward GEMMs on one bf16 plane per operand: one product per
 *                         multiply-add, plain bf16 outputs and gradients.
 *   NRW_PRECISION_BF16X3  forward and backward GEMMs on two planes (hi, lo): the three products
 *                         hi.hi + hi.lo + lo.hi, accumulated in fp32.
 *   NRW_PRECISION_BF16X6  forward and backward GEMMs on three planes: all six products of weight >= 2^-16,
 *                         about fp32 accuracy.
 *   NRW_PRECISION_MIXED   forward as bf16x3, so every rendered output and normal keeps split-bf16 accuracy;
 *                         the backward GEMMs and their softplus gates read the hi plane only (bf16 gradients).
 * Anything else is NRW_ERR_ARG.  chunk_rows: samples per MLP chunk (multiple of 128). */
#define NRW_PRECISION_BF16 1
#define NRW_PRECISION_BF16X3 2
#define NRW_PRECISION_BF16X6 3
#define NRW_PRECISION_MIXED 4
NRW_API int nrw_ctx_create(nrw_ctx** out, int precision, int gemm_backend, int n_vocab, int n_a);
NRW_API int nrw_ctx_destroy(nrw_ctx* ctx);
/* on = 0: the background NeRF has no appearance head (models/nerf.py encode_appearance=False): its colour branch is
 * relu(views_linears.0([feature, viewPE])) -> rgb_linear, the appearance code is neither read nor differentiated, and the
 * nerf.apperence_encoding.* slots of the parameter table are unused (their gradient stays 0).  Default 1.  Call before
 * nrw_ctx_bind: it changes the packed layout and the workspace (NRW_ERR_STATE after a bind). */
NRW_API int nrw_ctx_set_nerf_appearance(nrw_ctx* ctx, int on);
NRW_API long long nrw_packed_bytes(const nrw_ctx* ctx);
/* n_slots_sdf / n_slots_nerf: how many chunks keep their forward activations resident for the backward pass
 * (>= number of chunks of a batch: no forward recompute in backward; 1: recompute, minimum memory). */
NRW_API long long nrw_workspace_bytes(const nrw_ctx* ctx, int chunk_rows, int with_backward, int max_rays,
                                      int max_samples_per_ray, int n_slots_sdf, int n_slots_nerf);
NRW_API int nrw_ctx_bind(nrw_ctx* ctx, void* packed, long long packed_bytes, void* workspace,
                         long long workspace_bytes, int chunk_rows, int with_backward, int max_rays,
                         int max_samples_per_ray, int n_slots_sdf, int n_slots_nerf, void* stream);
/* weight-norm materialisation + bf16 plane split + transposes of every layer (replaces what
 * torch.nn.utils.weight_norm recomputes on every call, models/neuconw.py:104-105,256-257). */
NRW_API int nrw_pack_weights(nrw_ctx* ctx, const float* params, void* stream);

/* ---- NeuconWRenderer.sdf / NeuconW.sdf  (rendering/renderer.py:947-949) -----------------
 * With two-plane operands on the tensor-core backend the whole query is ONE launch of the fused on-chip chain (encoding, 8 layers,
 * head; 12 B in / 4 B out of HBM per point) and touches no workspace; otherwise it runs chunk by chunk through the bound
 * workspace.  Results do not depend on how the caller batches the points. */
NRW_API int nrw_sdf_query(nrw_ctx* ctx, const float* pts /*[n,3]*/, long long n, float* sdf /*[n]*/,
                          void* stream);
/* NeuconW.forward pieces (models/neuconw.py:339-376): sdf, features' consumer rgb, normals. */
NRW_API int nrw_neuconw_forward(nrw_ctx* ctx, const float* pts /*[n,3]*/, const float* dirs /*[n,3]*/,
                                const float* a /*[n,n_a]*/, long long n, float* rgb /*[n,3]*/,
                                float* sdf /*[n]*/, float* normals /*[n,3]*/, void* stream);
/* NeRF.forward (models/nerf.py:156-182): pts4 [n,4], dirs [n,3], a [n,n_a] -> density[n], rgb[n,3] */
NRW_API int nrw_nerf_forward(nrw_ctx* ctx, const float* pts4, const float* dirs, const float* a,
                             long long n, float* density, float* rgb, void* stream);
/* Backward of the three queries above (models/neuconw.py:284-296, models/nerf.py:156-182): the gradients of
 * L = <g_sdf, sdf> + <g_normals, normals> + <g_rgb, rgb> (NeuconW) or <g_density, density> + <g_rgb, rgb> (NeRF) with
 * respect to the parameters, the points, the view directions and the appearance codes.  A NULL upstream gradient is zero
 * and the work it would feed is skipped; a NULL output is not wanted.  grad_params (flat layout) is ACCUMULATED into, every
 * other output is written.  The query's forward is recomputed chunk by chunk (nothing of the forward call is kept), so the
 * gradients belong to the parameters as packed now; the SDF value is differentiated on the per-layer chain.  The normals'
 * point gradient is a Hessian-vector product; rgb's includes the path through the normal.  Needs a workspace bound with
 * with_backward (NRW_ERR_STATE otherwise).  NeuconW: dirs and a are needed with g_rgb.  NeRF: dirs always, a with g_rgb
 * when the appearance head is on; grad_a from a NeRF without the appearance head is NRW_ERR_ARG.  n == 0 does nothing. */
NRW_API int nrw_neuconw_backward(nrw_ctx* ctx, const float* pts /*[n,3]*/, const float* dirs /*[n,3] or NULL*/,
                                 const float* a /*[n,n_a] or NULL*/, long long n, const float* g_sdf /*[n]*/,
                                 const float* g_normals /*[n,3]*/, const float* g_rgb /*[n,3]*/, float* grad_params,
                                 float* grad_pts /*[n,3]*/, float* grad_dirs /*[n,3]*/, float* grad_a /*[n,n_a]*/,
                                 void* stream);
NRW_API int nrw_nerf_backward(nrw_ctx* ctx, const float* pts4 /*[n,4]*/, const float* dirs /*[n,3]*/,
                              const float* a /*[n,n_a] or NULL*/, long long n, const float* g_density /*[n]*/,
                              const float* g_rgb /*[n,3]*/, float* grad_params, float* grad_pts4 /*[n,4]*/,
                              float* grad_dirs /*[n,3]*/, float* grad_a /*[n,n_a]*/, void* stream);

/* ---- NeuconWRenderer.sparse_sampler (rendering/renderer.py:458-568) ---------------------- */
typedef struct {
  int n_samples, n_importance, up_sample_steps, n_outside, s_val_base;
  int boundary_samples; /* only used when sample_near/sample_far are given */
  int perturb;          /* 0/1: u_ray / u_out must be given when 1 */
} nrw_sampler_cfg;
/* o,d [R,3] (unit-sphere frame), near,far [R]; sample_near/sample_far [R] or NULL (no fine octree);
 * u_ray [R], u_out [R,n_outside] uniform draws or NULL.  Outputs: z_vals [R,S], z_out [R,n_outside],
 * sample_dist [R].  Optional trace (may be NULL): inds int32 [steps,R,n_imp/steps] (searchsorted
 * indices), order int32 [steps,R,S_round_max] (merge permutation). */
NRW_API int nrw_sample(nrw_ctx* ctx, const nrw_sampler_cfg* cfg, int R, const float* o, const float* d,
                       const float* near, const float* far, const float* sample_near,
                       const float* sample_far, const float* u_ray, const float* u_out, float* z_vals,
                       float* z_out, float* sample_dist, int32_t* trace_inds, int32_t* trace_order,
                       void* stream);
NRW_API int nrw_samples_per_ray(const nrw_sampler_cfg* cfg, int with_fine_octree);
/* one up-sampling round with injected sdf (stage-wise bit-exactness test; renderer.py:257-363) */
NRW_API int nrw_upsample_round(int R, int m, int n_new, float inv_s, const float* o, const float* d,
                               const float* z /*[R,m]*/, const float* sdf /*[R,m]*/,
                               float* cdf_scratch /*[R,m]*/, float* z_new /*[R,n_new]*/,
                               float* z_merged /*[R,m+n_new]*/, int32_t* inds /*[R,n_new]*/,
                               int32_t* order /*[R,m+n_new]*/, void* stream);

/* boundary samples of the fine-sampling branch (stage-wise bit-exactness test; renderer.py:546-566):
 * z [R,S0] ascending -> out [R,S0+nb] = sort(cat(nb/2 samples on [near,z_0), nb-nb/2 on (z_last,far], z)) */
NRW_API int nrw_boundary_samples(int R, int S0, int nb, const float* near, const float* far, const float* z,
                                 float* out, void* stream);

/* ---- NeuconWRenderer.render core (rendering/renderer.py:157-228,570-783) ----------------- */
typedef struct {
  int R, S, n_outside;        /* T = S + n_outside */
  float cos_anneal_ratio;
  const float* background_rgb; /* device [3] or NULL (renderer.py:753-754) */
  int reserved0;               /* generation stamp: render_backward reuses the cached forward activations only when
                                  it equals the stamp of the render_forward call that produced them (else recompute) */
  int trim_sphere;
} nrw_render_cfg;

/* Device pointers of one render call.  Inputs first, then outputs, then the small per-sample
 * tensors the backward pass needs ("saved", caller-allocated like everything else). */
typedef struct {
  /* inputs */
  const float* o;           /* [R,3] */
  const float* d;           /* [R,3] */
  const float* z_vals;      /* [R,S] */
  const float* z_out;       /* [R,n_outside] */
  const float* sample_dist; /* [R] */
  const float* a_emb;       /* [R,n_a] */
  const float* inv_s;       /* [1] */
  /* outputs (16-key dict of renderer.py:899-916, minus the loss-side glue kept in torch) */
  float* color;             /* [R,3] */
  float* color_sphere;      /* [R,3] */
  float* color_bg;          /* [R,3] */
  float* cdf;               /* [R,S] */
  float* gradients;         /* [R,S,3] */
  float* weights;           /* [R,T] */
  float* weights_sum;       /* [R] */
  float* inside_sphere;     /* [R,S] */
  float* depth;             /* [R] */
  float* normals;           /* [R,3] */
  float* gradient_error;    /* [1] */
  /* saved for backward */
  float* sv_sdf;            /* [R,S] */
  float* sv_rgb;            /* [R,S,3] */
  float* sv_bg_alpha;       /* [R,T] */
  float* sv_bg_rgb;         /* [R,T,3] */
  float* sv_z_feed;         /* [R,T] */
  float* sv_relax_sum;      /* [1] */
} nrw_render_io;

NRW_API int nrw_render_forward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io, void* stream);

/* upstream gradients (NULL = zero) and gradient outputs */
typedef struct {
  const float* g_color;        /* [R,3] */
  const float* g_color_sphere; /* [R,3] */
  const float* g_color_bg;     /* [R,3] */
  const float* g_cdf;          /* [R,S] */
  const float* g_gradients;    /* [R,S,3] */
  const float* g_weights;      /* [R,T] */
  const float* g_weights_sum;  /* [R] */
  const float* g_depth;        /* [R] */
  const float* g_normals;      /* [R,3] */
  const float* g_gradient_error; /* [1] */
  float* grad_params;          /* flat, same layout as params; ACCUMULATED into */
  float* grad_a_emb;           /* [R,n_a] (written) */
  float* grad_inv_s;           /* [1] (written) */
} nrw_render_grads;
NRW_API int nrw_render_backward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io,
                                const nrw_render_grads* g, void* stream);

/* stage-wise compositing (K4) with injected per-sample inputs, for parity tests */
NRW_API int nrw_composite_forward(const nrw_render_cfg* cfg, const nrw_render_io* io, const float* sdf,
                                  const float* normals_ps /*[R,S,3]*/, const float* rgb /*[R,S,3]*/,
                                  const float* bg_alpha, const float* bg_rgb, float* scratch2 /*[2]*/,
                                  void* stream);
NRW_API int nrw_composite_backward(const nrw_render_cfg* cfg, const nrw_render_io* io,
                                   const nrw_render_grads* g, const float* normals_ps, float* d_sdf,
                                   float* d_normals_ps, float* d_rgb, float* d_bg_alpha, float* d_bg_rgb,
                                   void* stream);
/* the network half of nrw_render_backward with injected per-sample upstream gradients: d_sdf [R,S], d_normals [R,S,3],
 * d_rgb [R,S,3], and when n_outside > 0 d_bg_alpha [R,T], d_bg_rgb [R,T,3] in sv_z_feed order (all required, none
 * means zero).  Reuses the forward that nrw_render_forward left in the context under the generation-stamp and
 * recompute rules of nrw_render_backward; grad_params is ACCUMULATED into, grad_a_emb [R,n_a] is written. */
NRW_API int nrw_network_backward(nrw_ctx* ctx, const nrw_render_cfg* cfg, const nrw_render_io* io, const float* d_sdf,
                                 const float* d_normals, const float* d_rgb, const float* d_bg_alpha,
                                 const float* d_bg_rgb, float* grad_params, float* grad_a_emb, void* stream);

/* ---- appearance codes of held-out photographs against frozen networks (NeRF-W evaluation; rules in csrc/appearance.cu)
 * nrw_appearance_prepare runs the appearance-free part of nrw_render_forward for the rays of cfg (o, d, z_vals [R,S],
 * z_out [R,n_outside] (may be NULL when n_outside = 0), sample_dist [R], inv_s [1], as for the render; cfg's
 * cos_anneal_ratio, background_rgb and trim_sphere apply, reserved0 is not read) and stores into `cache` (caller-owned,
 * 256-byte aligned, nrw_appearance_cache_bytes(ctx, R, S, n_outside) bytes) everything of `color` that does not depend on
 * the appearance code: per sample static_linear_0's pre-activation without the code columns (colour net, and the NeRF's
 * appearance head), the colour layers' [pts | normal] inputs and the compositing weights of the colours; per ray the
 * constant rest.  nrw_appearance_forward then writes color [R,3], equal to nrw_render_forward's color for the codes
 * a_emb [R,n_a] up to the split W [x | a] = W [x | 0] + W_a a; nrw_appearance_backward writes grad_a_emb [R,n_a] for the
 * upstream g_color [R,3] (per-ray sums in a fixed order: reproducible).  Neither forms a weight gradient or runs the SDF
 * network, xyz_encoding_final or the NeRF trunk.  The cache holds the networks as packed at the prepare (prepare again
 * after nrw_pack_weights with new weights); the context remembers each prepared cache by its address, and R is not bounded
 * by the bound max_rays.  Forward and backward run chunk by chunk through the bound workspace (the backward recomputes its
 * forward; it needs a bind with backward) and invalidate the forward a render left for its backward, which then
 * recomputes it.  Status: NRW_ERR_ARG for R <= 0 or a NULL required pointer, NRW_ERR_STATE before bind + pack, for a cache
 * not prepared on this context or a backward without a backward bind, NRW_ERR_WORKSPACE for a cache smaller than
 * nrw_appearance_cache_bytes.  nrw_appearance_cache_bytes returns a negative nrw_status for sizes out of range. */
NRW_API long long nrw_appearance_cache_bytes(const nrw_ctx* ctx, int R, int S, int n_outside);
NRW_API int nrw_appearance_prepare(nrw_ctx* ctx, const nrw_render_cfg* cfg, const float* o, const float* d,
                                   const float* z_vals, const float* z_out, const float* sample_dist, const float* inv_s,
                                   void* cache, long long cache_bytes, void* stream);
NRW_API int nrw_appearance_forward(nrw_ctx* ctx, const void* cache, const float* a_emb /*[R,n_a]*/, float* color /*[R,3]*/,
                                   void* stream);
NRW_API int nrw_appearance_backward(nrw_ctx* ctx, const void* cache, const float* a_emb, const float* g_color /*[R,3]*/,
                                    float* grad_a_emb /*[R,n_a], written*/, void* stream);

/* ---- octree near/far (tools/prepare_data/generate_voxel.py:311-439) ---------------------- */
/* octree bytes (breadth-first, one per non-leaf), prefix = exclusive popcount sum (#nodes entries),
 * pyramid int32 [2, level+2].  rays in the SfM frame.  Outputs near,far [R] (already * scale),
 * pid int32 [R] (-1 = miss), count int32 [R] (# leaf voxels hit). */
NRW_API int nrw_octree_near_far(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host,
                                int level, const float* rays_o, const float* rays_d, int R,
                                const float scene_origin[3], float scale, float* near, float* far,
                                int32_t* pid, int32_t* count, void* stream);
/* compacted hit list (ray_index, point_index, depth) front-to-back per ray; offsets = exclusive scan of count */
NRW_API int nrw_octree_hits(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host,
                            int level, const float* rays_o, const float* rays_d, int R,
                            const float scene_origin[3], float scale, const int64_t* offsets,
                            int32_t* ray_index, int32_t* point_index, float* depth, void* stream);

/* ---- octree build (K0; tools/prepare_data/generate_voxel.py:149-150 quantize_points + unbatched_points_to_octree,
 *      :173-178 scan_octrees + generate_points; called by get_octree renderer.py:137-155 and octree_update
 *      neuconw_system.py:268-312) ------------------------------------------------------------------------------- */
/* points [n,3] (float32, or float64 when points_are_f64) already normalised to the open cube (-1,1)
 * (generate_voxel.py:113-127).  Device outputs: octree uint8 [cap_nonleaf] (breadth-first child masks, zero padded),
 * prefix int32 [cap_nonleaf] (exclusive popcount sum), pyramid int32 [2, level+2], points_out int16 [cap_total,3]
 * (node coordinates of every level, breadth-first), counts_out int32 [2] = {#non-leaf nodes, #nodes}.  Nothing is
 * written out of bounds when a capacity is too small: compare counts_out with the capacities after synchronising
 * (n_points * level / n_points * (level+1) always suffice).  scratch: nrw_octree_build_scratch_bytes, 256-byte aligned. */
NRW_API long long nrw_octree_build_scratch_bytes(int n_points, int level, int cap_nonleaf);
NRW_API int nrw_octree_build(const void* points, int points_are_f64, int n_points, int level, uint8_t* octree,
                             int32_t* prefix, int32_t* pyramid, int16_t* points_out, int cap_nonleaf, int cap_total,
                             int32_t* counts_out, void* scratch, void* stream);

/* ---- fused clip + Adam on flat fp32 buffers (train.py:61 gradient_clip_val -> clip_grad_norm_;
 *      utils/__init__.py:30 torch.optim.Adam(eps=1e-7)) ---------------------------------------------------------- */
/* acc[0] (device double, zeroed by the caller) += sum g^2; call once per gradient buffer of the clipped group */
NRW_API int nrw_grad_sumsq(const float* grad, long long n, double* acc, void* stream);
/* one Adam step (t = step >= 1) on p with moments m, v; the gradient is scaled by min(1, max_norm/(sqrt(*sumsq)+1e-6))
 * when sumsq != NULL and max_norm > 0 (torch.nn.utils.clip_grad_norm_).  Nothing is read back to the host. */
NRW_API int nrw_adam_clip_step(float* p, const float* grad, float* m, float* v, long long n, const double* sumsq,
                               double max_norm, double lr, double beta1, double beta2, double eps, int step,
                               void* stream);

/* ---- ray-cache batch gather (SURVEY 8f-3): PhototourismDataset.__getitem__ with semantics over an index vector
 *      (datasets/phototourism.py:709-724) fused with training_step's RAY_MASK_LIST filter
 *      (lightning_modules/neuconw_system.py:345-355).  cache_rays [n,12] = o3,d3,near,far,ts,label,depth,weight and
 *      cache_rgbs [n,3] are the reference's cache arrays (tools/prepare_data/prepare_data_cache.py:128-151) resident in HBM.
 *      Rows whose label equals one of mask_labels_host[0..n_mask) (<= 8 ids, host array) are dropped; kept rows are
 *      written in index order: rays [m,10] = row[0:8] ++ row[10:12], rgbs [m,3], ts [m] int64, label [m]; n_valid[0] = m
 *      (device int64).  scratch: nrw_compact_scratch_bytes(batch) bytes, 256-byte aligned. ---------------------------- */
NRW_API long long nrw_compact_scratch_bytes(long long n);
NRW_API int nrw_raycache_gather(const float* cache_rays, const float* cache_rgbs, long long n_cache, const int64_t* index,
                                int batch, const int32_t* mask_labels_host, int n_mask, float* rays, float* rgbs, int64_t* ts,
                                float* label, int64_t* n_valid, void* scratch, void* stream);
/* ---- mesh-extraction / octree-refresh query pipeline (SURVEY 8f-1, 8f-2) ------------------------------------------------
 * dense lattice of utils/visualization.py:42-52: out[t] = (lin_x[i], lin_y[j], lin_z[k]) for linear index i0+t =
 * (i*dim + j)*dim + k, lin_c = torch.linspace(lo[c], hi[c], dim) (float32). */
NRW_API int nrw_grid_points_dense(int dim, const float lo[3], const float hi[3], long long i0, long long n, float* out /*[n,3]*/,
                                  void* stream);
/* up-sampled sparse lattice of tools/extract_mesh.py:73-95 / neuconw_system.py:213-234: candidate i0+t -> leaf (i0+t)/up^3
 * (leaves int16 [n_leaves,3], lexicographic = torch.nonzero order), sub-voxel unravel((i0+t)%up^3); xyz_sfm (optional) =
 * float32(index)*voxel_size + vol_origin, xyz_train = (xyz_sfm - scene_origin)/scene_radius. */
NRW_API int nrw_grid_points_sparse(const int16_t* leaves, long long n_leaves, int up_times, float voxel_size,
                                   const float vol_origin[3], const float scene_origin[3], float scene_radius, long long i0,
                                   long long n, float* xyz_sfm, float* xyz_train, void* stream);
/* stable compaction xyz[sdf <= threshold] (neuconw_system.py:259), appended at out[count[0]...]; count (device int64) is
 * increased by the number of rows kept.  scratch: nrw_compact_scratch_bytes(n). */
NRW_API int nrw_threshold_compact(const float* sdf, const float* xyz /*[n,3]*/, long long n, float threshold, float* out,
                                  int64_t* count, void* scratch, void* stream);

/* ---- masked marching cubes (the mesh step of utils/visualization.py::extract_mesh; rules in csrc/mcubes.cu) -------------
 * vol: contiguous fp32 [d0,d1,d2] (C order), every d >= 2; mask: uint8 [d0,d1,d2] or NULL, cell (i,j,k) is meshed only
 * when mask[i+1,j+1,k+1] != 0 (and its 8 corners are finite).  nrw_mc_count writes counts (device int64[2]) = {n_verts,
 * n_faces} and fills scratch (nrw_mc_scratch_bytes, 256-byte aligned); nrw_mc_emit, given the same volume, level, mask and
 * scratch and the two counts read back by the caller, writes verts fp32 [n_verts,3] (index coordinates, axis 0 first),
 * normals fp32 [n_verts,3] and faces int32 [n_faces,3].  n_verts must be <= INT32_MAX.  nrw_mc_scratch_bytes returns a
 * negative nrw_status for a dimension below 2. */
NRW_API long long nrw_mc_scratch_bytes(int d0, int d1, int d2);
NRW_API int nrw_mc_count(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask /*nullable*/,
                         void* scratch, long long* counts /*device int64[2]: n_verts, n_faces*/, void* stream);
NRW_API int nrw_mc_emit(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask, const void* scratch,
                        long long n_verts, long long n_faces, float* verts, float* normals, int32_t* faces, void* stream);

/* ---- exact nearest neighbour and surface sampling in fp64 (utils/eval_utils.py; rules in csrc/nnsearch.cu) ----------
 * nrw_nn_build indexes ref f64 [n_ref,3] (1 <= n_ref <= INT32_MAX, finite) into `index` (nrw_nn_index_bytes(n_ref) bytes,
 * 256-byte aligned; it also serves as the build's scratch).  nrw_nn_query writes, for every query q of queries f64
 * [n_query,3], the smallest (squared distance, index) pair over the indexed points: dist f64 [n_query] = sqrt of the
 * squared distance, idx int64 [n_query].  n_ref must be the count the index was built for (the index holds its own copy of
 * the points, so `ref` may be freed after the build).  scratch:
 * nrw_nn_query_scratch_bytes(n_query), 256-byte aligned.  The *_bytes functions return a negative nrw_status for a size
 * outside their range. */
NRW_API long long nrw_nn_index_bytes(long long n_ref);
NRW_API int nrw_nn_build(const double* ref, long long n_ref, void* index, void* stream);
NRW_API long long nrw_nn_query_scratch_bytes(long long n_query);
NRW_API int nrw_nn_query(const void* index, long long n_ref, const double* queries, long long n_query, double* dist,
                         int64_t* idx, void* scratch, void* stream);
/* Area-weighted uniform samples of the triangle mesh verts f64 [n_verts,3], faces int64 [n_faces,3]: out f64
 * [n_samples,3], face_id int64 [n_samples] (nullable).  Sample s depends only on (seed, s).  status (device int32[1]) is
 * written by the call: bit 0 = a face index outside [0, n_verts), bit 1 = total area not positive and finite; when it is
 * non-zero nothing is sampled.  scratch: nrw_mesh_sample_scratch_bytes(n_faces), 256-byte aligned. */
NRW_API long long nrw_mesh_sample_scratch_bytes(long long n_faces);
NRW_API int nrw_mesh_sample(const double* verts, long long n_verts, const int64_t* faces, long long n_faces, long long n_samples,
                            unsigned long long seed, double* out, int64_t* face_id /*nullable*/, int32_t* status,
                            void* scratch, void* stream);

/* ---- mesh depth rasterisation and back-projection (utils/reproj_filter.py; rules in csrc/raster.cu) ----------------
 * nrw_raster_depth renders the depth of the mesh verts f64 [n_verts,3] (finite), faces int64 [n_faces,3] seen through
 * world_to_cam (HOST f64 [3,4] row-major, COLMAP axes: z forward, y down) and the pinhole fx, fy, cx, cy into depth f32
 * [height,width] (the camera z of the nearest hit with znear <= z <= zfar, 0 where nothing is hit).  cull_back = 1 drops
 * faces whose right-hand normal points away from the camera.  status (device int32[1]) is written by the call: bit 0 = a
 * face index outside [0, n_verts) (such faces are skipped).  scratch: nrw_raster_scratch_bytes(n_verts, n_faces, height,
 * width), 256-byte aligned.  Needs FLT_MIN <= znear <= zfar <= FLT_MAX, fx, fy > 0, height * width <= INT32_MAX.
 * nrw_reproject_mark back-projects every pixel with depth > 0 from its integer coordinate (c, r) through the pinhole
 * and cam_to_world (HOST f64 [3,4]) and sets visible[i] = 1 (uint8 [n_ref], not cleared) for the nearest point i of an
 * nrw_nn_build index over n_ref points when its distance is < threshold.  n_valid (device int64[1], nullable) is
 * increased by the number of pixels with depth > 0.  scratch: nrw_reproject_scratch_bytes(height, width), 256-byte
 * aligned.  Neither call reads anything back to the host.  The *_bytes functions return a negative nrw_status for
 * sizes outside their range. */
NRW_API long long nrw_raster_scratch_bytes(long long n_verts, long long n_faces, int height, int width);
NRW_API int nrw_raster_depth(const double* verts, long long n_verts, const int64_t* faces, long long n_faces,
                             const double* world_to_cam, double fx, double fy, double cx, double cy, int height, int width,
                             double znear, double zfar, int cull_back, float* depth, int32_t* status, void* scratch,
                             void* stream);
NRW_API long long nrw_reproject_scratch_bytes(int height, int width);
NRW_API int nrw_reproject_mark(const float* depth, int height, int width, double fx, double fy, double cx, double cy,
                               const double* cam_to_world, const void* index, long long n_ref, double threshold,
                               uint8_t* visible, long long* n_valid /*nullable*/, void* scratch, void* stream);

/* ---- training ray-cache generation (datasets/phototourism.py::read_meta; rules in csrc/raygen.cu) -------------------
 * nrw_raygen_image writes one image's cache rows: rows f32 [out_cap, 12] (o3, d3, near, far, ts, label, depth, weight;
 * 11 columns without the label when with_label = 0) and rgbs f32 [out_cap, 3], the kept pixels in raster order, then the
 * depth_percent padding and a seeded permutation.  Inputs: rgb8 uint8 [height, width, 3]; semantic f32
 * [sem_height, sem_width] (with_label only); the image's keypoints xys f64 [n_keypoints, 2] (full-resolution pixels) and
 * point3d_ids int64 [n_keypoints] (-1 = none); the point table point_xyz f64 [n_points, 3] and point_error f64 [n_points]
 * indexed by point3D id.  counts (device int64[4]) = {rows written, kept rows, depth-valid kept rows, padding rows};
 * status (device int32[1]): bit 0 = a point3D id past the table, bit 1 = out_cap too small for the padding.  out_cap >=
 * nrw_raygen_capacity(height, width, depth_percent); scratch: nrw_raygen_scratch_bytes, 256-byte aligned.  Nothing is
 * read back to the host; the caller reads counts[0] to size its copy.
 * nrw_depth_range writes, for every image i of w2c f64 [n_images, 3, 4] (device), out f64 [n_images, 2] =
 * np.percentile(z, (q_lo, q_hi)) of the camera z of the points xyz f64 [n_points, 3] with z > 0, n_front int64
 * [n_images] (nullable) = their count; status bit 0 = an image with no point in front.  n_points * n_images <=
 * INT32_MAX; scratch: nrw_depth_range_scratch_bytes.  nrw_raygen_capacity and the *_bytes functions return a negative
 * nrw_status for sizes, or a depth_percent outside [0, 1), out of range. */
typedef struct {
  const uint8_t* octree; /* device: breadth-first child masks */
  const int32_t* prefix; /* device: exclusive popcount sum */
  int level;             /* 1..16 */
  float scene_origin[3]; /* fp32, SfM frame */
  float scale;           /* > 0 */
} nrw_octree_ref;
typedef struct {
  int height, width;       /* image after the downscale */
  int img_downscale;       /* >= 1: keypoints are divided by it, the semantic map is read at size // it */
  float fx, fy, cx, cy;    /* K of the downscaled image, finite, fx, fy != 0 */
  float c2w[12];           /* fp32 [3,4] row-major, columns 1:2 negated (read_meta) */
  double w2c_z[4];         /* fp64 third row of COLMAP's [R | t] */
  int image_id;            /* ts column and the padding stream */
  int with_label, sem_height, sem_width;
  int use_voxel;           /* 1: near/far and the kept set from the two octrees; 0: constant near/far, every row kept */
  float near, far;         /* use_voxel = 0 */
  float voxel_size;        /* added to the expanded octree's far */
  nrw_octree_ref sfm;      /* expand 1, radius 1: decides which rows are kept */
  nrw_octree_ref expanded; /* expand 2, radius 1.5: the stored near/far */
  double depth_percent;    /* [0, 1) */
  unsigned long long seed;
} nrw_raygen_cfg;
NRW_API long long nrw_raygen_capacity(int height, int width, double depth_percent);
NRW_API long long nrw_raygen_scratch_bytes(int height, int width, int with_label, long long n_keypoints, long long out_cap);
NRW_API int nrw_raygen_image(const nrw_raygen_cfg* cfg, const uint8_t* rgb8, const float* semantic, const double* xys,
                             const int64_t* point3d_ids, long long n_keypoints, const double* point_xyz,
                             const double* point_error, long long n_points, float* rows, float* rgbs, long long out_cap,
                             int64_t* counts, int32_t* status, void* scratch, void* stream);
NRW_API long long nrw_depth_range_scratch_bytes(long long n_points, int n_images);
NRW_API int nrw_depth_range(const double* xyz, long long n_points, const double* w2c, int n_images, double q_lo, double q_hi,
                            double* out, int64_t* n_front, int32_t* status, void* scratch, void* stream);

/* ---- point-cloud visibility through its voxel octree (utils/kaolin_renderer.py; rules in csrc/voxelvis.cu) -----------
 * nrw_voxel_cast casts one ray per pixel of a height x width pinhole view (fx, fy, cx, cy in fp32, pixel (c, r) from the
 * integer grid) from cam_to_world (host f64 [3,4] row-major, rounded to fp32) through an octree of nrw_octree_build
 * (octree, prefix on the device, pyramid_host [2, level+2] on the host; level 1..16), normalised by scene_origin and
 * scale as get_near_far does, and takes the first leaf each ray hits.  Outputs, each nullable: visible u8 [n_leaf]
 * set to 1 at every hit leaf (never cleared, so views accumulate), depth f32 [height, width] = near * scale / |d|
 * (0 on a miss), leaf i32 [height, width] (-1 on a miss), n_hit (device int64) increased by the number of hit pixels.
 * nrw_voxel_lookup maps points f64 [n_points, 3], already normalised ((x - origin) / scale), to their leaf index
 * (-1 outside the open cube (-1, 1)^3); a quantised cell that is not a leaf also gives -1 and sets bit 0 of status
 * (device int32, cleared first).  Every argument is checked before any launch; nothing is read back to the host. */
NRW_API int nrw_voxel_cast(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                           const float scene_origin[3], float scale, const double* cam_to_world, float fx, float fy,
                           float cx, float cy, int height, int width, uint8_t* visible, float* depth, int32_t* leaf,
                           int64_t* n_hit, void* stream);
NRW_API int nrw_voxel_lookup(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                             const double* points, long long n_points, int32_t* leaf, int32_t* status, void* stream);

/* ---- training-view selection of the scene split (tools/prepare_data/dataset_filter_utils.py; rules in csrc/viewsel.cu) --
 * nrw_view_roi_count counts, for every view of one launch, the pixels whose ray passes through the scene sphere
 * (view_selection's ROI test): views f32 [n_views, 16] = fx, fy, cx, cy, c2w[12] (fp32 [3,4] row-major, columns 1:2
 * negated as read_meta makes them), hw int32 [n_views, 2] = height, width, both on the device; scene_origin (host f32[3])
 * and radius (finite, > 0) in fp32.  counts (device int64 [n_views]) is overwritten; a view with height or width < 1, or
 * height * width > max_hw (1 .. INT32_MAX, the caller's largest view), gets -1.  Rays follow the ray-cache pass's fp32
 * rule.
 * nrw_label_static_count adds to count (device int64, not cleared) the number of labels f32 [n] that equal none of the
 * n_ids <= 8 ids (host int32, each 0 .. 2^24 - 1).  Every host argument is checked before any launch; nothing is read
 * back to the host. */
NRW_API int nrw_view_roi_count(const float* views, const int32_t* hw, int n_views, long long max_hw, const float scene_origin[3],
                               float radius, int64_t* counts, void* stream);
NRW_API int nrw_label_static_count(const float* labels, long long n, const int32_t* ids_host, int n_ids, int64_t* count,
                                   void* stream);

/* ---- ground-truth alignment check (tools/reproj_error.py; rules in csrc/gtproj.cu) -------------------------------
 * nrw_first_hit writes hit (device int64 [n_queries]): for each query (q_view int32, q_xy f32 [n_queries, 2], both on
 * the device) the index of the point (f32 [n_points, 3], n_points < 2^32) with the smallest fp32 camera depth > 0 whose
 * fp64 projection rounds to the query's pixel (rint of its xy), the smaller index on equal depths, or -1.  views (HOST
 * f64 [n_views, 16]) = world->camera [3, 4] row-major, fx, fy, cx, cy; boxes (HOST int32 [n_views, 4]) = x0, y0, width,
 * height of the bounding box of each view's query pixels (width or height 0 for a view without queries).  A query whose
 * view is out of range or whose pixel lies outside its box gets -1 and sets bit 0 of status (device int32, cleared).
 * scratch (256-byte aligned) of scratch_bytes >= nrw_first_hit_scratch_bytes(n_queries, largest box area); a larger
 * scratch fits more views into one pass over the points.  The result does not depend on the pass layout.
 * nrw_obs_reproj_error writes err (device f64 [n]): the distance of the projection of X (f64 [n, 3]) by the P = K [R|t]
 * (device f64 [n_views, 12]) of view[i] (int32 [n]) to xy (f64 [n, 2]); uv (f64 [n, 2], nullable) receives the
 * projection.  An out-of-range view gives NaN.  Every argument is checked before any launch; nothing is read back. */
NRW_API long long nrw_first_hit_scratch_bytes(long long n_queries, long long map_pixels);
NRW_API int nrw_first_hit(const float* points, long long n_points, const double* views_host, const int32_t* boxes_host,
                          int n_views, const int32_t* q_view, const float* q_xy, long long n_queries, int64_t* hit,
                          int32_t* status, void* scratch, long long scratch_bytes, void* stream);
NRW_API int nrw_obs_reproj_error(const double* X, const int32_t* view, const double* xy, long long n, const double* P,
                                 int n_views, double* err, double* uv, void* stream);

/* ---- unit-test hooks ---------------------------------------------------------------------- */
/* D[M,N] = (sum planes of A)[M,K] * (sum planes of B)[N,K]^T from fp32 inputs: splits into planes in
 * scratch (caller-provided, nrw_gemm_test_scratch_bytes) and runs the selected backend. */
NRW_API long long nrw_gemm_test_scratch_bytes(int M, int N, int K);
NRW_API int nrw_gemm_test(int backend, int n_planes, int mn_major, int k_slices, int M, int N, int K,
                          const float* A, const float* B, const float* bias, int act, float* D,
                          void* scratch, void* stream);
/* A backward layer's data GEMM and weight gradient in one paired tensor-core launch (paired = 1; the launch must be eligible,
 * else NRW_ERR_ARG), or as two launches, weight gradient first (paired = 0).  One-plane bf16 operands:
 *   data  out[M, N] = epilogue(A[M, K] B[N, K]^T) of kind `kind`, all side streams [M, N] with ld N:
 *         0 GENERIC   planes out_pl, column sums into colsum (if non-NULL)
 *         1 TANGENT   gate from the bf16 plane side_h (u / scale), aux_q = side_f (NULL: colvec broadcast), out2 (fp32),
 *                     planes out_pl, or out_f32 when non-NULL
 *         2 REVERSE   [+ rowvec (x) colvec], gate from side_h, + side_f, planes out_pl, colsum
 *         3 RELU_BWD  [+ rowvec (x) colvec], mask by the bf16 side_h > 0, planes out_pl, colsum
 *         with the output scale `scale` and the column bound n_store;
 *   dW    dW[Mw, Nw] (fp32) += dY[Kw, Mw]^T X[Kw, Nw], split into k_slices K-slices. */
NRW_API int nrw_gemm_pair_test(int paired, int kind, int M, int N, int K, int Mw, int Nw, int Kw, int k_slices,
                               const void* A, const void* B, const void* dY, const void* X, const void* side_h,
                               const float* side_f, const float* rowvec, const float* colvec, float scale, int n_store,
                               void* out_pl, float* out_f32, float* out2, float* colsum, float* dW, void* stream);
NRW_API long long nrw_launch_count(void);
/* measurement: while enabled, every tensor-core GEMM launch is bracketed by CUDA events on its stream; a call with
 * out5 != NULL synchronises those events and returns {sum of kernel ms, algorithmic FLOP (2MNK), MMA FLOP
 * (x plane products), launches, algorithmic HBM bytes (operands + epilogue streams)} since the last read
 * (bench.py roofline). */
NRW_API int nrw_gemm_timing(int enable, double* out5_host);
/* debug: per-CTA cycle attribution of the tensor-core GEMM (u64 [SMs,16], zeroed by the caller; NULL = off) */
NRW_API int nrw_debug_gemm_profile(void* device_buf_u64);

#ifdef __cplusplus
}
#endif
#endif /* NRW_H_ */
