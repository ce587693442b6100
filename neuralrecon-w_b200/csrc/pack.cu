// Parameter table, weight packing (weight-norm materialisation + bf16 plane split + transposes)
// and the inverse map for gradients (incl. weight-norm backward).
#include <stdarg.h>

#include "params.h"

namespace nrw {

long long g_kernel_launches = 0;
static thread_local char g_err[1024] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error_cstr() { return g_err; }

// ---------------------------------------------------------------------------------------------
std::vector<ParamInfo> build_param_table(int n_vocab, int n_a) {
  std::vector<ParamInfo> t;
  auto add = [&](const std::string& n, int r, int c) { t.push_back(ParamInfo{n, r, c, 0, 0}); };
  add("embedding_a.weight", n_vocab, n_a);
  const int sdf_o[9] = {512, 512, 512, 473, 512, 512, 512, 512, 513};
  const int sdf_i[9] = {39, 512, 512, 512, 512, 512, 512, 512, 512};
  for (int l = 0; l < 9; ++l) {
    std::string p = "neuconw.sdf_net.lin" + std::to_string(l) + ".";
    add(p + "weight_v", sdf_o[l], sdf_i[l]);
    add(p + "weight_g", sdf_o[l], 1);
    add(p + "bias", sdf_o[l], 0);
  }
  add("neuconw.xyz_encoding_final.weight", 512, 512);
  add("neuconw.xyz_encoding_final.bias", 512, 0);
  add("neuconw.deviation_network.variance", 0, 0);
  const int col_o[5] = {256, 256, 256, 256, 3};
  const int col_i[5] = {134, 256, 256, 256, 256};
  for (int l = 0; l < 5; ++l) {
    std::string p = "neuconw.color_net.lin" + std::to_string(l) + ".";
    add(p + "weight_v", col_o[l], col_i[l]);
    add(p + "weight_g", col_o[l], 1);
    add(p + "bias", col_o[l], 0);
  }
  add("neuconw.color_net.static_encoding.static_linear_0.weight", 128, 512 + 27 + n_a);
  add("neuconw.color_net.static_encoding.static_linear_0.bias", 128, 0);
  add("neuconw.color_net.static_encoding.static_linear_1.weight", 128, 128);
  add("neuconw.color_net.static_encoding.static_linear_1.bias", 128, 0);
  add("neuconw.color_net.xyz_encoding_final.weight", 512, 512);
  add("neuconw.color_net.xyz_encoding_final.bias", 512, 0);
  for (int i = 0; i < 8; ++i) {
    std::string p = "nerf.pts_linears." + std::to_string(i) + ".";
    add(p + "weight", 256, i == 0 ? 84 : (i == 5 ? 340 : 256));
    add(p + "bias", 256, 0);
  }
  for (int s = 0; s < 4; ++s) {
    std::string p = "nerf.apperence_encoding.static_linear_" + std::to_string(s) + ".";
    add(p + "weight", 128, s == 0 ? 256 + 27 + n_a : 128);
    add(p + "bias", 128, 0);
  }
  add("nerf.views_linears.0.weight", 128, 283);
  add("nerf.views_linears.0.bias", 128, 0);
  add("nerf.feature_linear.weight", 256, 256);
  add("nerf.feature_linear.bias", 256, 0);
  add("nerf.alpha_linear.weight", 1, 256);
  add("nerf.alpha_linear.bias", 1, 0);
  add("nerf.rgb_linear.weight", 3, 128);
  add("nerf.rgb_linear.bias", 3, 0);
  long long off = 0;
  for (auto& p : t) {
    p.numel = (p.rows == 0 && p.cols == 0) ? 1 : (long long)p.rows * (p.cols == 0 ? 1 : p.cols);
    p.offset = off;
    off += round_up(p.numel, 4);
  }
  return t;
}

// ---------------------------------------------------------------------------------------------
static void init_layer(PackedLayer& L, const std::vector<ParamInfo>& tab, int w, int g, int b, int row_off,
                       int n_rows, int Np, int Kp) {
  memset(&L, 0, sizeof(L));
  L.w_off = tab[w].offset;
  L.g_off = g >= 0 ? tab[g].offset : -1;
  L.b_off = tab[b].offset;
  L.src_rows = tab[w].rows;
  L.src_cols = tab[w].cols;
  L.row_off = row_off;
  L.n_rows = n_rows;
  L.Np = Np;
  L.Kp = Kp;
  for (int j = 0; j < MAX_KP; ++j) L.colmap[j] = -1;
  for (int c = 0; c < MAX_SRC_COLS; ++c) L.colinv[c] = -1;
  for (int j = 0; j < L.src_cols && j < Kp; ++j) L.colmap[j] = (short)j;  // identity by default
}
static void finish_layer(PackedLayer& L) {
  for (int j = 0; j < L.Kp; ++j)
    if (L.colmap[j] >= 0) L.colinv[L.colmap[j]] = (short)j;
}

PackedModel build_packed_model(const std::vector<ParamInfo>& tab, int n_planes, bool nerf_app) {
  PackedModel pm;
  memset(&pm, 0, sizeof(pm));
  PackedLayer* L = pm.layers;
  // SDF net: lin0 K 39->64; lin3 473 rows -> 512; lin8 rows 1..512 (row 0 is the sdf head)
  init_layer(L[L_SDF0], tab, pi_sdf_v(0), pi_sdf_g(0), pi_sdf_b(0), 0, 512, 512, 64);
  for (int l = 1; l < 8; ++l)
    init_layer(L[L_SDF0 + l], tab, pi_sdf_v(l), pi_sdf_g(l), pi_sdf_b(l), 0, l == 3 ? 473 : 512, 512, 512);
  init_layer(L[L_SDF8F], tab, pi_sdf_v(8), pi_sdf_g(8), pi_sdf_b(8), 1, 512, 512, 512);
  // colour net
  init_layer(L[L_CX], tab, PI_CX_W, -1, PI_CX_B, 0, 512, 512, 512);
  init_layer(L[L_CS0], tab, PI_CS0_W, -1, PI_CS0_B, 0, 128, 128, 640);   // [xf512 | viewPE27 | a | pad]
  init_layer(L[L_CS1], tab, PI_CS1_W, -1, PI_CS1_B, 0, 128, 128, 128);
  init_layer(L[L_CL0], tab, pi_col_v(0), pi_col_g(0), pi_col_b(0), 0, 256, 256, 192);
  {  // packed [h2(128) | pts(3) | normals(3) | pad]  <-  source [pts3, normals3, dir_encoding128]
    PackedLayer& c = L[L_CL0];
    for (int j = 0; j < MAX_KP; ++j) c.colmap[j] = -1;
    for (int j = 0; j < 128; ++j) c.colmap[j] = (short)(6 + j);
    for (int j = 0; j < 6; ++j) c.colmap[128 + j] = (short)j;
  }
  for (int l = 1; l < 4; ++l)
    init_layer(L[L_CL0 + l], tab, pi_col_v(l), pi_col_g(l), pi_col_b(l), 0, 256, 256, 256);
  // background NeRF
  init_layer(L[L_N0], tab, PI_NPTS_BASE, -1, PI_NPTS_BASE + 1, 0, 256, 256, 128);
  for (int i = 1; i < 8; ++i)
    init_layer(L[L_N0 + i], tab, PI_NPTS_BASE + 2 * i, -1, PI_NPTS_BASE + 2 * i + 1, 0, 256, 256, i == 5 ? 384 : 256);
  {  // packed [h(256) | pe(84) | pad]  <-  source [pe84, h256]
    PackedLayer& c = L[L_N0 + 5];
    for (int j = 0; j < MAX_KP; ++j) c.colmap[j] = -1;
    for (int j = 0; j < 256; ++j) c.colmap[j] = (short)(84 + j);
    for (int j = 0; j < 84; ++j) c.colmap[256 + j] = (short)j;
  }
  init_layer(L[L_NF], tab, PI_NF_W, -1, PI_NF_B, 0, 256, 256, 256);
  if (nerf_app)
    init_layer(L[L_NS0], tab, PI_NAPP_BASE, -1, PI_NAPP_BASE + 1, 0, 128, 128, 384);  // [feat256|viewPE27|a|pad]
  else   // views_linears.0 over [feat256|viewPE27]: the a and pad columns of FEATN meet zero weights
    init_layer(L[L_NS0], tab, PI_NVIEWS_W, -1, PI_NVIEWS_B, 0, 128, 128, 384);
  for (int s = 1; s < 4; ++s)   // (no rows without appearance: packed as zeros, no gradient unpacked)
    init_layer(L[L_NS0 + s], tab, PI_NAPP_BASE + 2 * s, -1, PI_NAPP_BASE + 2 * s + 1, 0, nerf_app ? 128 : 0, 128, 128);
  for (int i = 0; i < L_COUNT; ++i) finish_layer(L[i]);

  // packed buffer layout: [device copy of layer table][bf16 area][fp32 area]
  pm.table_bytes = round_up((long long)sizeof(PackedLayer) * L_COUNT, 1024);
  long long bf = 0;
  for (int i = 0; i < L_COUNT; ++i) {
    const long long sz = (long long)L[i].Np * L[i].Kp;
    pm.plane_stride[i] = sz;
    L[i].W_off = bf;  bf += round_up(sz * n_planes, 512);
    L[i].WT_off = bf; bf += round_up(sz * n_planes, 512);
  }
  pm.bf16_off_bytes = pm.table_bytes;
  pm.f32_off_bytes = round_up(pm.bf16_off_bytes + bf * 2, 1024);
  long long f = 0, gsz = 0;
  auto falloc = [&](long long n) { long long o = f; f += round_up(n, 4); return o; };
  auto galloc = [&](long long n) { long long o = gsz; gsz += round_up(n, 4); return o; };
  for (int i = 0; i < L_COUNT; ++i) {
    L[i].bias_off = falloc(L[i].Np);
    L[i].rnorm_off = falloc(L[i].Np);
    L[i].dW_off = galloc((long long)L[i].Np * L[i].Kp);
    L[i].db_off = galloc(L[i].Np);
  }
  Heads& H = pm.heads;
  H.sdf_w0 = falloc(512); H.sdf_b0 = falloc(1); H.cl4_w = falloc(3 * 256); H.cl4_b = falloc(3);
  H.na_w = falloc(256); H.na_b = falloc(1); H.nr_w = falloc(3 * 128); H.nr_b = falloc(3);
  H.sdf_rn0 = falloc(1); H.cl4_rn = falloc(3);
  H.d_sdf_w0 = galloc(512); H.d_sdf_b0 = galloc(1); H.d_cl4_w = galloc(3 * 256); H.d_cl4_b = galloc(3);
  H.d_na_w = galloc(256); H.d_na_b = galloc(1); H.d_nr_w = galloc(3 * 128); H.d_nr_b = galloc(3);
  pm.total_bytes = round_up(pm.f32_off_bytes + f * 4, 1024);
  pm.grad_floats = gsz;
  return pm;
}

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = 0.0f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}

// grid (512, L_COUNT): one block per packed row
__global__ void __launch_bounds__(256) pack_kernel(const PackedLayer* __restrict__ table, int n_planes,
                                                   const float* __restrict__ params, bf16* __restrict__ bf_area,
                                                   float* __restrict__ f_area) {
  __shared__ float red[8];
  const PackedLayer& L = table[blockIdx.y];
  const int n = blockIdx.x;
  if (n >= L.Np) return;
  const bool valid = n < L.n_rows;
  const int r = n + L.row_off;
  const float* src = params + L.w_off + (long long)r * L.src_cols;
  float scale = 1.0f;
  if (L.g_off >= 0) {
    float ss = 0.0f;
    if (valid)
      for (int c = threadIdx.x; c < L.src_cols; c += blockDim.x) ss += src[c] * src[c];
    ss = block_sum(ss, red);
    const float rn = valid ? rsqrtf(ss) : 0.0f;
    // torch: g * v / norm ; keep the same evaluation order: (v * g) / norm is not what torch does,
    // _weight_norm computes v * (g / norm)
    scale = valid ? params[L.g_off + r] / sqrtf(ss) : 0.0f;
    if (threadIdx.x == 0) f_area[L.rnorm_off + n] = valid ? 1.0f / sqrtf(ss) : 0.0f;
    (void)rn;
  }
  const long long ps = (long long)L.Np * L.Kp;
  for (int j = threadIdx.x; j < L.Kp; j += blockDim.x) {
    const int c = L.colmap[j];
    float v = (valid && c >= 0) ? src[c] * scale : 0.0f;
    bf16 p0, p1, p2;
    split3(v, p0, p1, p2);
    const long long wi = L.W_off + (long long)n * L.Kp + j;
    const long long ti = L.WT_off + (long long)j * L.Np + n;
    bf_area[wi] = p0; bf_area[ti] = p0;
    if (n_planes > 1) { bf_area[wi + ps] = p1; bf_area[ti + ps] = p1; }
    if (n_planes > 2) { bf_area[wi + 2 * ps] = p2; bf_area[ti + 2 * ps] = p2; }
  }
  if (threadIdx.x == 0) f_area[L.bias_off + n] = valid ? params[L.b_off + r] : 0.0f;
}

struct HeadSrc {
  long long w_off, g_off, b_off;   // param offsets
  int src_cols, row;               // source row index
  long long dst_w, dst_b, dst_rn;  // float offsets in f_area (dst_rn = -1 if none)
};
struct HeadTable { HeadSrc h[8]; };

__global__ void __launch_bounds__(256) pack_heads_kernel(HeadTable T, const float* __restrict__ params,
                                                         float* __restrict__ f_area) {
  __shared__ float red[8];
  const HeadSrc& h = T.h[blockIdx.x];
  const float* src = params + h.w_off + (long long)h.row * h.src_cols;
  float scale = 1.0f;
  if (h.g_off >= 0) {
    float ss = 0.0f;
    for (int c = threadIdx.x; c < h.src_cols; c += blockDim.x) ss += src[c] * src[c];
    ss = block_sum(ss, red);
    scale = params[h.g_off + h.row] / sqrtf(ss);
    if (threadIdx.x == 0 && h.dst_rn >= 0) f_area[h.dst_rn] = 1.0f / sqrtf(ss);
  }
  for (int c = threadIdx.x; c < h.src_cols; c += blockDim.x) f_area[h.dst_w + c] = src[c] * scale;
  if (threadIdx.x == 0) f_area[h.dst_b] = params[h.b_off + h.row];
}

static HeadTable make_head_table(const PackedModel& pm, const std::vector<ParamInfo>& tab) {
  HeadTable T;
  const Heads& H = pm.heads;
  T.h[0] = HeadSrc{tab[pi_sdf_v(8)].offset, tab[pi_sdf_g(8)].offset, tab[pi_sdf_b(8)].offset, 512, 0,
                   H.sdf_w0, H.sdf_b0, H.sdf_rn0};
  for (int c = 0; c < 3; ++c)
    T.h[1 + c] = HeadSrc{tab[pi_col_v(4)].offset, tab[pi_col_g(4)].offset, tab[pi_col_b(4)].offset, 256, c,
                         H.cl4_w + 256 * c, H.cl4_b + c, H.cl4_rn + c};
  T.h[4] = HeadSrc{tab[PI_NA_W].offset, -1, tab[PI_NA_B].offset, 256, 0, H.na_w, H.na_b, -1};
  for (int c = 0; c < 3; ++c)
    T.h[5 + c] = HeadSrc{tab[PI_NR_W].offset, -1, tab[PI_NR_B].offset, 128, c, H.nr_w + 128 * c, H.nr_b + c, -1};
  return T;
}

int pack_weights(const PackedModel& pm, const std::vector<ParamInfo>& tab, int n_planes, const float* params,
                 void* packed_base, cudaStream_t s) {
  const PackedLayer* table = reinterpret_cast<const PackedLayer*>(packed_base);
  bf16* bf_area = reinterpret_cast<bf16*>(reinterpret_cast<char*>(packed_base) + pm.bf16_off_bytes);
  float* f_area = reinterpret_cast<float*>(reinterpret_cast<char*>(packed_base) + pm.f32_off_bytes);
  pack_kernel<<<dim3(512, L_COUNT), 256, 0, s>>>(table, n_planes, params, bf_area, f_area);
  NRW_LAUNCH_OK();
  HeadTable T = make_head_table(pm, tab);
  pack_heads_kernel<<<8, 256, 0, s>>>(T, params, f_area);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// grid (513, L_COUNT): one block per SOURCE row; accumulates into grad_params
__global__ void __launch_bounds__(256) unpack_kernel(const PackedLayer* __restrict__ table,
                                                     const float* __restrict__ params,
                                                     const float* __restrict__ f_area,
                                                     const float* __restrict__ gs, float* __restrict__ gp) {
  __shared__ float red[8];
  const PackedLayer& L = table[blockIdx.y];
  const int r = blockIdx.x;
  const int n = r - L.row_off;
  if (r >= L.src_rows || n < 0 || n >= L.n_rows) return;
  const float* dWp = gs + L.dW_off + (long long)n * L.Kp;
  const float* v = params + L.w_off + (long long)r * L.src_cols;
  float* dv = gp + L.w_off + (long long)r * L.src_cols;
  if (L.g_off >= 0) {
    float dot = 0.0f;
    for (int c = threadIdx.x; c < L.src_cols; c += blockDim.x) dot += dWp[L.colinv[c]] * v[c];
    dot = block_sum(dot, red);
    const float rn = f_area[L.rnorm_off + n];
    const float g = params[L.g_off + r];
    for (int c = threadIdx.x; c < L.src_cols; c += blockDim.x)
      dv[c] += g * rn * (dWp[L.colinv[c]] - v[c] * dot * rn * rn);
    if (threadIdx.x == 0) gp[L.g_off + r] += dot * rn;
  } else {
    for (int c = threadIdx.x; c < L.src_cols; c += blockDim.x) dv[c] += dWp[L.colinv[c]];
  }
  if (threadIdx.x == 0) gp[L.b_off + r] += gs[L.db_off + n];
}

struct HeadGrad {
  long long w_off, g_off, b_off;
  int src_cols, row;
  long long src_dw, src_db, rn;   // float offsets: gradient scratch / f_area
};
struct HeadGradTable { HeadGrad h[8]; };

__global__ void __launch_bounds__(256) unpack_heads_kernel(HeadGradTable T, const float* __restrict__ params,
                                                           const float* __restrict__ f_area,
                                                           const float* __restrict__ gs, float* __restrict__ gp) {
  __shared__ float red[8];
  const HeadGrad& h = T.h[blockIdx.x];
  const float* dW = gs + h.src_dw;
  const float* v = params + h.w_off + (long long)h.row * h.src_cols;
  float* dv = gp + h.w_off + (long long)h.row * h.src_cols;
  if (h.g_off >= 0) {
    float dot = 0.0f;
    for (int c = threadIdx.x; c < h.src_cols; c += blockDim.x) dot += dW[c] * v[c];
    dot = block_sum(dot, red);
    const float rn = f_area[h.rn];
    const float g = params[h.g_off + h.row];
    for (int c = threadIdx.x; c < h.src_cols; c += blockDim.x) dv[c] += g * rn * (dW[c] - v[c] * dot * rn * rn);
    if (threadIdx.x == 0) gp[h.g_off + h.row] += dot * rn;
  } else {
    for (int c = threadIdx.x; c < h.src_cols; c += blockDim.x) dv[c] += dW[c];
  }
  if (threadIdx.x == 0) gp[h.b_off + h.row] += gs[h.src_db];
}

int unpack_grads(const PackedModel& pm, const std::vector<ParamInfo>& tab, const float* params,
                 const void* packed_base, const float* gs, float* gp, cudaStream_t s) {
  const PackedLayer* table = reinterpret_cast<const PackedLayer*>(packed_base);
  const float* f_area = reinterpret_cast<const float*>(reinterpret_cast<const char*>(packed_base) + pm.f32_off_bytes);
  unpack_kernel<<<dim3(513, L_COUNT), 256, 0, s>>>(table, params, f_area, gs, gp);
  NRW_LAUNCH_OK();
  const Heads& H = pm.heads;
  HeadGradTable T;
  T.h[0] = HeadGrad{tab[pi_sdf_v(8)].offset, tab[pi_sdf_g(8)].offset, tab[pi_sdf_b(8)].offset, 512, 0,
                    H.d_sdf_w0, H.d_sdf_b0, H.sdf_rn0};
  for (int c = 0; c < 3; ++c)
    T.h[1 + c] = HeadGrad{tab[pi_col_v(4)].offset, tab[pi_col_g(4)].offset, tab[pi_col_b(4)].offset, 256, c,
                          H.d_cl4_w + 256 * c, H.d_cl4_b + c, H.cl4_rn + c};
  T.h[4] = HeadGrad{tab[PI_NA_W].offset, -1, tab[PI_NA_B].offset, 256, 0, H.d_na_w, H.d_na_b, 0};
  for (int c = 0; c < 3; ++c)
    T.h[5 + c] = HeadGrad{tab[PI_NR_W].offset, -1, tab[PI_NR_B].offset, 128, c, H.d_nr_w + 128 * c, H.d_nr_b + c, 0};
  unpack_heads_kernel<<<8, 256, 0, s>>>(T, params, f_area, gs, gp);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
