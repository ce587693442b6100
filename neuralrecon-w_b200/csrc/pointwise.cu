// Memory-bound helper kernels around the GEMM chain: positional encodings (and their Jacobians),
// the narrow output heads (N <= 3) and their backward, column sums for bias gradients.
#include "pointwise.h"

namespace nrw {

static constexpr float INV_SQRT2 = 0.70710678118654752440f;

// pts[m] = o[r] + d[r] * t,  t = z (use_mid = 0) or z + 0.5 * dist (use_mid = 1; renderer.py:586-593)
// explicit _rn ops: torch evaluates mul and add separately (no FMA contraction).
__global__ void points_kernel(const float* __restrict__ o, const float* __restrict__ d,
                              const float* __restrict__ z, const float* __restrict__ sample_dist, int R,
                              int S, int use_mid, float* __restrict__ pts) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= (long long)R * S) return;
  const int r = (int)(m / S), i = (int)(m % S);
  float t = z[m];
  if (use_mid) {
    const float dist = (i + 1 < S) ? __fsub_rn(z[m + 1], t) : sample_dist[r];
    t = __fadd_rn(t, __fmul_rn(dist, 0.5f));
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) pts[m * 3 + c] = __fadd_rn(o[r * 3 + c], __fmul_rn(d[r * 3 + c], t));
}
int launch_points(const float* o, const float* d, const float* z, const float* sample_dist, int R, int S,
                  int use_mid, float* pts, cudaStream_t s) {
  const long long M = (long long)R * S;
  if (M == 0) return NRW_OK;
  points_kernel<<<cdiv(M, 256), 256, 0, s>>>(o, d, z, sample_dist, R, S, use_mid, pts);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- SDF head: sdf = u8 . w0 + b0 with u8 = softplus(a7) read from its planes; optional gbar7 = softplus'(a7) * w0 ----
// warp per row, lane j handles columns 4j..4j+3 of each 128-column group: 8-byte plane loads / stores
__global__ void __launch_bounds__(256) sdf_head_kernel(Planes U8, int M, const float* __restrict__ w0,
                                                       const float* __restrict__ b0, float* __restrict__ sdf,
                                                       int n_planes, Planes G7) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= M) return;
  const long long row = (long long)warp * U8.ld;
  float acc = 0.0f;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int j = g * 128 + lane * 4;
    float u[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int pl = 0; pl < n_planes; ++pl) {
      const uint2 t = __ldg(reinterpret_cast<const uint2*>(U8.plane(pl) + row + j));
      u[0] += __uint_as_float(t.x << 16); u[1] += __uint_as_float(t.x & 0xFFFF0000u);
      u[2] += __uint_as_float(t.y << 16); u[3] += __uint_as_float(t.y & 0xFFFF0000u);
    }
    const float4 w = __ldg(reinterpret_cast<const float4*>(w0 + j));
    const float wv[4] = {w.x, w.y, w.z, w.w};
    float gq[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      acc = fmaf(u[k], wv[k], acc);
      float s1, s2;
      softplus100_d12_from_u(u[k], s1, s2);
      gq[k] = s1 * wv[k];
    }
    if (G7.p) {
      const long long grow = (long long)warp * G7.ld + j;
      for (int pl = 0; pl < n_planes; ++pl) {
        uint32_t pk[2];
        split_plane<4>(gq, pk);
        *reinterpret_cast<uint2*>(G7.plane(pl) + grow) = make_uint2(pk[0], pk[1]);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) sdf[warp] = acc + b0[0];
}
int launch_sdf_head(Planes U8, int M, const float* w0, const float* b0, float* sdf, int n_planes, Planes G7, cudaStream_t s) {
  NRW_CHECK(U8.ld == 512 && (G7.p == nullptr || G7.ld == 512) && (U8.pstride & 3) == 0, NRW_ERR_ARG, "sdf_head: 512-wide planes expected");
  sdf_head_kernel<<<cdiv((long long)M * 32, 256), 256, 0, s>>>(U8, M, w0, b0, sdf, n_planes, G7);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// sdf = b0 + the 8 row partials the fused-head epilogue left (fixed summation order: deterministic)
__global__ void sdf_head_sum_kernel(const float* __restrict__ hp, int M, const float* __restrict__ b0, float* __restrict__ sdf) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float4 a = __ldg(reinterpret_cast<const float4*>(hp + (long long)m * 8)), b = __ldg(reinterpret_cast<const float4*>(hp + (long long)m * 8 + 4));
  sdf[m] = (((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w))) + b0[0];
}
int launch_sdf_head_sum(const float* hp, int M, const float* b0, float* sdf, cudaStream_t s) {
  sdf_head_sum_kernel<<<cdiv(M, 256), 256, 0, s>>>(hp, M, b0, sdf);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- normal = J_PE(x)^T (q0[:39] + q4[473:512] / sqrt2)  (SURVEY 9.2) -----------------------------
__global__ void sdf_normal_kernel(const float* __restrict__ pts, const float* __restrict__ Q0,
                                  const float* __restrict__ Q4, int M, float* __restrict__ nrm) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float v[39];
  for (int j = 0; j < 39; ++j) v[j] = Q0[(long long)m * 64 + j] + Q4[(long long)m * 512 + 473 + j] * INV_SQRT2;
  float out[3] = {v[0], v[1], v[2]};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = pts[m * 3 + c];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float f = (float)(1 << k);
      float sn, cs;
      sincosf(x * f, &sn, &cs);
      out[c] += v[3 + 6 * k + c] * f * cs - v[6 + 6 * k + c] * f * sn;
    }
  }
  nrm[m * 3] = out[0]; nrm[m * 3 + 1] = out[1]; nrm[m * 3 + 2] = out[2];
}
int launch_sdf_normal(const float* pts, const float* Q0, const float* Q4, int M, float* nrm, cudaStream_t s) {
  sdf_normal_kernel<<<cdiv(M, 128), 128, 0, s>>>(pts, Q0, Q4, M, nrm);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// backward of the above w.r.t. (q0, q4 tail): t = J_PE(x) dn
__global__ void sdf_normal_bwd_kernel(const float* __restrict__ pts, const float* __restrict__ dn, int M,
                                      int n_planes, Planes DQ0, Planes DQ4) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float t[39];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = pts[m * 3 + c], g = dn[m * 3 + c];
    t[c] = g;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float f = (float)(1 << k);
      float sn, cs;
      sincosf(x * f, &sn, &cs);
      t[3 + 6 * k + c] = g * f * cs;
      t[6 + 6 * k + c] = -g * f * sn;
    }
  }
  for (int j = 0; j < 64; ++j) planes_store(DQ0, n_planes, (long long)m * DQ0.ld + j, j < 39 ? t[j] : 0.0f);
  for (int j = 0; j < 39; ++j) planes_store(DQ4, n_planes, (long long)m * DQ4.ld + 473 + j, t[j] * INV_SQRT2);
}
int launch_sdf_normal_bwd(const float* pts, const float* dn, int M, int n_planes, Planes DQ0, Planes DQ4,
                          cudaStream_t s) {
  sdf_normal_bwd_kernel<<<cdiv(M, 128), 128, 0, s>>>(pts, dn, M, n_planes, DQ0, DQ4);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- input gradients of point queries ---------------------------------------------------------------------------
// The encodings [x, sin(f x), cos(f x)]_{f = 2^k} are separable per coordinate: coordinate c feeds column c and the
// sin / cos columns D + 2Dk + c, D + 2Dk + D + c.  One thread per (row, coordinate).
//
// out[m,c] (+)= J_PE(x)^T dE:  dE[m,c] + sum_k f (cos(f x) dE[m, sin_k] - sin(f x) dE[m, cos_k])
__global__ void pe_bwd_kernel(const float* __restrict__ x, int D, int n_freq, const float* __restrict__ dE, int ld, int M,
                              float* __restrict__ out, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * D) return;
  const long long m = i / D;
  const int c = (int)(i % D);
  const float xv = x[i];
  const float* g = dE + m * ld;
  float acc = g[c];
  for (int k = 0; k < n_freq; ++k) {
    const float f = (float)(1 << k);
    float sn, cs;
    sincosf(xv * f, &sn, &cs);
    acc += f * (cs * g[D + 2 * D * k + c] - sn * g[2 * D + 2 * D * k + c]);
  }
  out[i] = accumulate ? out[i] + acc : acc;
}
int launch_pe_bwd(const float* x, int D, int n_freq, const float* dE, int ld, int M, float* out, int accumulate,
                  cudaStream_t s) {
  NRW_CHECK(ld >= D * (2 * n_freq + 1), NRW_ERR_ARG, "pe_bwd: ld=%d < %d encoding columns", ld, D * (2 * n_freq + 1));
  if (M == 0) return NRW_OK;
  pe_bwd_kernel<<<cdiv((long long)M * D, 256), 256, 0, s>>>(x, D, n_freq, dE, ld, M, out, accumulate);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// Point gradient of an SDF query, the mirror of sdf_normal_kernel.  With E = PE6(x):
//   d_E = dE0[:39] + dE4[25:64] / sqrt2     (the reverse sweep's DA_0 W_0 and the skip layer's E columns of DA_4 W_4)
//   v   = q0[:39] + q4[473:512] / sqrt2     (d sdf / d E, which the normal contracts with J_PE)
//   out[m,c] (+)= J_PE(x)^T d_E  +  dn[m,c] sum_j v_j E_j''(x_c)     (the Hessian of E is diagonal)
__global__ void sdf_point_bwd_kernel(const float* __restrict__ pts, const float* __restrict__ Q0, const float* __restrict__ Q4,
                                     const float* __restrict__ dn, const float* __restrict__ dE, int M, float* __restrict__ out,
                                     int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * 3) return;
  const long long m = i / 3;
  const int c = (int)(i % 3);
  const float xv = pts[i], g = dn[i];
  const float* e0 = dE + m * 128 + 64;   // DA_0 W_0, columns 0..63
  const float* e4 = dE + m * 128 + 25;   // DA_4 W_4 rows 448..511: the E columns 473.. start at 25
  const float* q0 = Q0 + m * 64;
  const float* q4 = Q4 + m * 512 + 473;
  float acc = e0[c] + e4[c] * INV_SQRT2;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const float f = (float)(1 << k);
    const int js = 3 + 6 * k + c, jc = js + 3;
    float sn, cs;
    sincosf(xv * f, &sn, &cs);
    const float ds = e0[js] + e4[js] * INV_SQRT2, dc = e0[jc] + e4[jc] * INV_SQRT2;
    const float vs = q0[js] + q4[js] * INV_SQRT2, vc = q0[jc] + q4[jc] * INV_SQRT2;
    acc += f * (cs * ds - sn * dc) - f * f * g * (sn * vs + cs * vc);
  }
  out[i] = accumulate ? out[i] + acc : acc;
}
int launch_sdf_point_bwd(const float* pts, const float* Q0, const float* Q4, const float* dn, const float* dE, int M,
                         float* out, int accumulate, cudaStream_t s) {
  if (M == 0) return NRW_OK;
  sdf_point_bwd_kernel<<<cdiv((long long)M * 3, 256), 256, 0, s>>>(pts, Q0, Q4, dn, dE, M, out, accumulate);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- narrow heads: out[m,c] = act(X[m,:] . W[c,:] + b[c]),  NOUT in {1,3} --------------------------
// act: 0 none, 3 sigmoid.  For the NeRF alpha head (NOUT=1) `dists` turns density into
// alpha = 1 - exp(-softplus(density) * dist) (renderer.py:205-207); density is kept in out2.
template <int NOUT>
__global__ void __launch_bounds__(256) head_kernel(Planes X, int n_planes, int K, int M,
                                                   const float* __restrict__ W, const float* __restrict__ b,
                                                   int act, const float* __restrict__ dists,
                                                   float* __restrict__ out, float* __restrict__ out2) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= M) return;
  float acc[NOUT];
#pragma unroll
  for (int c = 0; c < NOUT; ++c) acc[c] = 0.0f;
  for (int j = lane; j < K; j += 32) {
    const float x = planes_load(X, n_planes, (long long)warp * X.ld + j);
#pragma unroll
    for (int c = 0; c < NOUT; ++c) acc[c] = fmaf(x, W[c * K + j], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < NOUT; ++c)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < NOUT; ++c) {
      float v = acc[c] + b[c];
      if (act == ACT_SIGMOID) v = sigmoidf_(v);
      if (NOUT == 1 && dists) {
        if (out2) out2[warp] = v;
        const float sp = v > 20.0f ? v : log1pf(expf(v));
        v = 1.0f - expf(-sp * dists[warp]);
      }
      out[(long long)warp * NOUT + c] = v;
    }
  }
}
int launch_head(int nout, Planes X, int n_planes, int K, int M, const float* W, const float* b, int act,
                const float* dists, float* out, float* out2, cudaStream_t s) {
  const int grid = cdiv((long long)M * 32, 256);
  if (nout == 1) head_kernel<1><<<grid, 256, 0, s>>>(X, n_planes, K, M, W, b, act, dists, out, out2);
  else head_kernel<3><<<grid, 256, 0, s>>>(X, n_planes, K, M, W, b, act, dists, out, out2);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// backward of a narrow head.  dpre[m,c] is formed on the fly:
//   mode 0: dpre = g_out                      (linear head)
//   mode 1: dpre = g_out * y * (1-y)          (sigmoid head; y = forward output)
//   mode 2: NeRF alpha head: dpre = g_alpha * exp(-softplus(density)*dist) * dist * sigmoid(density)
// writes dX[m,k] = relu'(X[m,k]) * sum_c dpre[m,c] W[c,k] as planes (or, when dX.p == null, only dpre to
// dpre_out), and accumulates dW[c,k] += sum_m dpre X, db[c] += sum_m dpre with block-level partials.
// One block = HB_ROWS rows; thread t owns the column PAIR (2t, 2t+1) (4-byte bf16x2 accesses, K/2 threads): the per-row
// pre-activation gradients dpre sit in shared memory, the dW partials of the block stay in registers and leave with one
// global atomic per (column, output) - no shared-memory atomics (the first version spent 3 of them per element).
static constexpr int HB_ROWS = 128;
template <int NOUT>
__global__ void __launch_bounds__(128) head_bwd_kernel(Planes X, int n_planes, int K, int M,
                                                       const float* __restrict__ W,
                                                       const float* __restrict__ g_out,
                                                       const float* __restrict__ y_or_density,
                                                       const float* __restrict__ dists, int mode, Planes dX,
                                                       float* __restrict__ dpre_out, float* __restrict__ dW,
                                                       float* __restrict__ db) {
  __shared__ float sdp[HB_ROWS][NOUT];
  const int row0 = blockIdx.x * HB_ROWS;
  const int nrows = min(HB_ROWS, M - row0);
  for (int i = threadIdx.x; i < HB_ROWS * NOUT; i += blockDim.x) {
    const int r = i / NOUT, c = i % NOUT;
    float g = 0.0f;
    if (r < nrows) {
      const int m = row0 + r;
      g = g_out[(long long)m * NOUT + c];
      if (mode == 1) {
        const float y = y_or_density[(long long)m * NOUT + c];
        g = g * y * (1.0f - y);
      } else if (mode == 2) {
        const float dens = y_or_density[m];
        const float sp = dens > 20.0f ? dens : log1pf(expf(dens));
        const float dsp = dens > 20.0f ? 1.0f : sigmoidf_(dens);
        g = g * expf(-sp * dists[m]) * dists[m] * dsp;
      }
      if (dpre_out) dpre_out[(long long)m * NOUT + c] = g;
    }
    sdp[r][c] = g;
  }
  __syncthreads();
  if (threadIdx.x < NOUT) {                       // bias gradient of this block
    float sacc = 0.0f;
    for (int r = 0; r < nrows; ++r) sacc += sdp[r][threadIdx.x];
    atomicAdd(&db[threadIdx.x], sacc);
  }
  const int j = threadIdx.x * 2;
  if (j >= K) return;
  float w0[NOUT], w1[NOUT], a0[NOUT], a1[NOUT];
#pragma unroll
  for (int c = 0; c < NOUT; ++c) { w0[c] = W[c * K + j]; w1[c] = W[c * K + j + 1]; a0[c] = a1[c] = 0.0f; }
  for (int r = 0; r < nrows; ++r) {
    const long long off = (long long)(row0 + r) * X.ld + j;
    float x0 = 0.0f, x1 = 0.0f;
    for (int pl = 0; pl < n_planes; ++pl) {
      const uint32_t t = __ldg(reinterpret_cast<const uint32_t*>(X.plane(pl) + off));
      x0 += __uint_as_float(t << 16);
      x1 += __uint_as_float(t & 0xFFFF0000u);
    }
    float d0 = 0.0f, d1 = 0.0f;
#pragma unroll
    for (int c = 0; c < NOUT; ++c) {
      const float dp = sdp[r][c];
      d0 = fmaf(dp, w0[c], d0); d1 = fmaf(dp, w1[c], d1);
      a0[c] = fmaf(dp, x0, a0[c]); a1[c] = fmaf(dp, x1, a1[c]);
    }
    if (dX.p) {
      float v[2] = {x0 > 0.0f ? d0 : 0.0f, x1 > 0.0f ? d1 : 0.0f};
      const long long doff = (long long)(row0 + r) * dX.ld + j;
      for (int pl = 0; pl < n_planes; ++pl) {
        uint32_t pk[1];
        split_plane<2>(v, pk);
        *reinterpret_cast<uint32_t*>(dX.plane(pl) + doff) = pk[0];
      }
    }
  }
#pragma unroll
  for (int c = 0; c < NOUT; ++c) { atomicAdd(&dW[c * K + j], a0[c]); atomicAdd(&dW[c * K + j + 1], a1[c]); }
}
int launch_head_bwd(int nout, Planes X, int n_planes, int K, int M, const float* W, const float* g_out,
                    const float* y_or_density, const float* dists, int mode, Planes dX, float* dpre_out,
                    float* dW, float* db, cudaStream_t s) {
  NRW_CHECK(K % 2 == 0 && K <= 256 && (X.ld & 1) == 0 && (dX.p == nullptr || (dX.ld & 1) == 0), NRW_ERR_ARG, "head_bwd: K=%d", K);
  const int grid = cdiv(M, HB_ROWS);
  if (nout == 1)
    head_bwd_kernel<1><<<grid, 128, 0, s>>>(X, n_planes, K, M, W, g_out, y_or_density, dists, mode, dX, dpre_out, dW, db);
  else
    head_bwd_kernel<3><<<grid, 128, 0, s>>>(X, n_planes, K, M, W, g_out, y_or_density, dists, mode, dX, dpre_out, dW, db);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// generic small utilities
__global__ void fill_kernel(float* p, long long n, float v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
int launch_fill(float* p, long long n, float v, cudaStream_t s) {
  if (n == 0) return NRW_OK;
  fill_kernel<<<cdiv(n, 256), 256, 0, s>>>(p, n, v);
  NRW_LAUNCH_OK();
  return NRW_OK;
}
__global__ void add3_kernel(float* dst, const float* a, const float* b, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = a[i] + (b ? b[i] : 0.0f);
}
int launch_add(float* dst, const float* a, const float* b, long long n, cudaStream_t s) {
  if (n == 0) return NRW_OK;
  add3_kernel<<<cdiv(n, 256), 256, 0, s>>>(dst, a, b, n);
  NRW_LAUNCH_OK();
  return NRW_OK;
}
// split an fp32 matrix [rows, cols] (ld_src) into planes (ld = P.ld), zero padding cols..ld
__global__ void split_planes_kernel(const float* __restrict__ src, long long rows, int cols, int ld_src,
                                    int n_planes, Planes P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * P.ld) return;
  const long long r = i / P.ld;
  const int c = (int)(i % P.ld);
  planes_store(P, n_planes, i, c < cols ? src[r * ld_src + c] : 0.0f);
}
int launch_split_planes(const float* src, long long rows, int cols, int ld_src, int n_planes, Planes P,
                        cudaStream_t s) {
  split_planes_kernel<<<cdiv(rows * P.ld, 256), 256, 0, s>>>(src, rows, cols, ld_src, n_planes, P);
  NRW_LAUNCH_OK();
  return NRW_OK;
}
// per-ray segment sum: out[r, c] = sum_{i<S} X[(r*S+i), c]   (appearance-code gradient)
__global__ void segsum_kernel(const float* __restrict__ X, int ld, int col0, int ncols, int R, int S,
                              float* __restrict__ out, int accumulate) {
  const int r = blockIdx.x;
  for (int c = threadIdx.x; c < ncols; c += blockDim.x) {
    float acc = 0.0f;
    for (int i = 0; i < S; ++i) acc += X[((long long)r * S + i) * ld + col0 + c];
    if (accumulate) out[(long long)r * ncols + c] += acc; else out[(long long)r * ncols + c] = acc;
  }
}
int launch_segsum(const float* X, int ld, int col0, int ncols, int R, int S, float* out, int accumulate,
                  cudaStream_t s) {
  if (R == 0) return NRW_OK;
  segsum_kernel<<<R, 64, 0, s>>>(X, ld, col0, ncols, R, S, out, accumulate);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
