// Input encodings of the three MLPs and column sums, one thread per OUTPUT element so every store is
// coalesced (the sample-per-thread versions were 10x slower: strided 2-byte stores).
#include "pointwise.h"

namespace nrw {

static constexpr float INV_SQRT2 = 0.70710678118654752440f;

// value j of the 3-D positional encoding [x, sin(2^k x), cos(2^k x)]_k (models/neuconw.py:7-55)
__device__ __forceinline__ float pe3(const float* x, int j) {
  if (j < 3) return x[j];
  const int k = (j - 3) / 6, r = (j - 3) % 6, c = r % 3;
  const float t = x[c] * (float)(1 << k);
  return r >= 3 ? cosf(t) : sinf(t);
}
// 4-D variant (models/nerf.py:8-39)
__device__ __forceinline__ float pe4(const float* x, int j) {
  if (j < 4) return x[j];
  const int k = (j - 4) / 8, r = (j - 4) % 8, c = r % 4;
  const float t = x[c] * (float)(1 << k);
  return r >= 4 ? cosf(t) : sinf(t);
}

// ---- staged encoders -------------------------------------------------------------------------------------------------
// A block of 128 threads owns ER = 32 consecutive rows.  Phase 1: one thread per (row, coordinate) evaluates sincosf ONCE per
// frequency (one sinf or cosf per OUTPUT element makes the kernel SFU / issue bound) and leaves the fp32 feature rows in shared memory.  Phase 2: all threads write
// the bf16 planes with 4-byte bf16x2 stores, a warp per 128-byte row segment.
static constexpr int ER = 32;

// planes of a [ER x ncols] fp32 tile in shared memory (row pitch `pitch`) -> dst columns [c0, c0 + ncols) of rows m0.., ncols even
__device__ __forceinline__ void store_tile_planes(const float* tile, int pitch, int ncols, int rows, Planes P, int n_planes,
                                                  long long m0, int c0) {
  const int pairs = ncols >> 1;
  for (int i = threadIdx.x; i < rows * pairs; i += blockDim.x) {
    const int r = i / pairs, q = i % pairs;
    float v[2] = {tile[r * pitch + 2 * q], tile[r * pitch + 2 * q + 1]};
    const long long off = (m0 + r) * P.ld + c0 + 2 * q;
    for (int pl = 0; pl < n_planes; ++pl) {
      uint32_t pk[1];
      split_plane<2>(v, pk);
      *reinterpret_cast<uint32_t*>(P.plane(pl) + off) = pk[0];
    }
  }
}

// U0[m, 0:64] = [PE6(x) 39 | 0];  U4[m, 473:512] = PE6(x) / sqrt(2)
__global__ void __launch_bounds__(128) sdf_embed_kernel(const float* __restrict__ pts, int M, int n_planes, Planes U0,
                                                        Planes U4) {
  __shared__ float pe[ER][64];
  const int m0 = blockIdx.x * ER;
  const int rows = min(ER, M - m0);
  for (int i = threadIdx.x; i < ER * 64; i += blockDim.x) (&pe[0][0])[i] = 0.0f;
  __syncthreads();
  if (threadIdx.x < rows * 3) {
    const int r = threadIdx.x / 3, c = threadIdx.x % 3;
    const float x = pts[(long long)(m0 + r) * 3 + c];
    pe[r][c] = x;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float sn, cs;
      sincosf(x * (float)(1 << k), &sn, &cs);
      pe[r][3 + 6 * k + c] = sn;
      pe[r][3 + 6 * k + 3 + c] = cs;
    }
  }
  __syncthreads();
  store_tile_planes(&pe[0][0], 64, 64, rows, U0, n_planes, m0, 0);
  if (U4.p) {   // 39 columns starting at the odd column 473: scalar bf16 stores
    for (int i = threadIdx.x; i < rows * 39; i += blockDim.x) {
      const int r = i / 39, j = i % 39;
      planes_store(U4, n_planes, (long long)(m0 + r) * U4.ld + 473 + j, pe[r][j] * INV_SQRT2);
    }
  }
}
int launch_sdf_embed(const float* pts, int M, int n_planes, Planes U0, Planes U4, cudaStream_t s) {
  NRW_CHECK((U0.ld & 1) == 0 && (U0.pstride & 1) == 0, NRW_ERR_ARG, "sdf_embed: even leading dimension expected");
  sdf_embed_kernel<<<cdiv(M, ER), 128, 0, s>>>(pts, M, n_planes, U0, U4);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// IN1[m, 512:640] = [viewPE4(d) 27 | a n_a | 0];  IN2[m, 128:192] = [pts 3 | normal 3 | 0]
__global__ void __launch_bounds__(128) color_embed_kernel(const float* __restrict__ dirs, const float* __restrict__ a,
                                                          int n_a, int rows_per_src, const float* __restrict__ pts,
                                                          const float* __restrict__ nrm, int M, int n_planes, Planes IN1,
                                                          Planes IN2) {
  __shared__ float t1[ER][128];
  __shared__ float t2[ER][64];
  const int m0 = blockIdx.x * ER;
  const int rows = min(ER, M - m0);
  for (int i = threadIdx.x; i < ER * 128; i += blockDim.x) (&t1[0][0])[i] = 0.0f;
  for (int i = threadIdx.x; i < ER * 64; i += blockDim.x) (&t2[0][0])[i] = 0.0f;
  __syncthreads();
  if (threadIdx.x < rows * 3) {
    const int r = threadIdx.x / 3, c = threadIdx.x % 3;
    const int m = m0 + r, src = m / rows_per_src;
    const float x = dirs[src * 3 + c];
    t1[r][c] = x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float sn, cs;
      sincosf(x * (float)(1 << k), &sn, &cs);
      t1[r][3 + 6 * k + c] = sn;
      t1[r][3 + 6 * k + 3 + c] = cs;
    }
    t2[r][c] = pts[m * 3 + c];
    t2[r][3 + c] = nrm[m * 3 + c];
  }
  for (int i = threadIdx.x; i < rows * n_a; i += blockDim.x) {
    const int r = i / n_a, j = i % n_a;
    t1[r][27 + j] = a[(long long)((m0 + r) / rows_per_src) * n_a + j];
  }
  __syncthreads();
  store_tile_planes(&t1[0][0], 128, 128, rows, IN1, n_planes, m0, 512);
  store_tile_planes(&t2[0][0], 64, 64, rows, IN2, n_planes, m0, 128);
}
int launch_color_embed(const float* dirs, const float* a, int n_a, int rows_per_src, const float* pts,
                       const float* nrm, int M, int n_planes, Planes IN1, Planes IN2, cudaStream_t s) {
  NRW_CHECK(n_a >= 0 && 27 + n_a <= 128 && (IN1.ld & 1) == 0 && (IN2.ld & 1) == 0, NRW_ERR_ARG, "color_embed: n_a=%d", n_a);
  color_embed_kernel<<<cdiv(M, ER), 128, 0, s>>>(dirs, a, n_a, rows_per_src, pts, nrm, M, n_planes, IN1, IN2);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// Background NeRF inputs (renderer.py:157-203; models/nerf.py:156-160):
// IN0[m, 0:128] and IN5[m, 256:384] = [PE10(pts4) 84 | 0];  FEATN[m, 256:384] = [viewPE 27 | a | 0]
__global__ void __launch_bounds__(128) nerf_embed_kernel(const float* __restrict__ o, const float* __restrict__ d,
                                                         const float* __restrict__ z,
                                                         const float* __restrict__ sample_dist,
                                                         const float* __restrict__ pts4_in, const float* __restrict__ a,
                                                         int n_a, int T, int rows_per_src, int M, int n_planes, Planes IN0,
                                                         Planes IN5, Planes FEATN, float* __restrict__ dists_out) {
  __shared__ float t0[ER][128];
  __shared__ float tv[ER][128];
  __shared__ float p4s[ER][4];
  const int m0 = blockIdx.x * ER;
  const int rows = min(ER, M - m0);
  for (int i = threadIdx.x; i < ER * 128; i += blockDim.x) { (&t0[0][0])[i] = 0.0f; (&tv[0][0])[i] = 0.0f; }
  if (threadIdx.x < rows) {      // the inverted-sphere point of this sample (same operation order as before)
    const int r = threadIdx.x, m = m0 + r, src = m / rows_per_src;
    float p4[4];
    if (pts4_in) {
#pragma unroll
      for (int c = 0; c < 4; ++c) p4[c] = pts4_in[(long long)m * 4 + c];
    } else {
      const int i = m % T;
      const float t0z = z[m];
      const float dist = (i + 1 < T) ? __fsub_rn(z[m + 1], t0z) : sample_dist[src];
      const float mid = __fadd_rn(t0z, __fmul_rn(dist, 0.5f));
      float p[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[src * 3 + c], __fmul_rn(d[src * 3 + c], mid));
      float nr = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
      nr = fminf(fmaxf(nr, 1.0f), 1e10f);
      p4[0] = p[0] / nr; p4[1] = p[1] / nr; p4[2] = p[2] / nr; p4[3] = 1.0f / nr;
      if (dists_out) dists_out[m] = dist;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) p4s[r][c] = p4[c];
  }
  __syncthreads();
  if (threadIdx.x < rows * 4) {  // PE10 of the 4-D point: one thread per (row, coordinate)
    const int r = threadIdx.x >> 2, c = threadIdx.x & 3;
    const float x = p4s[r][c];
    t0[r][c] = x;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      float sn, cs;
      sincosf(x * (float)(1 << k), &sn, &cs);
      t0[r][4 + 8 * k + c] = sn;
      t0[r][4 + 8 * k + 4 + c] = cs;
    }
  }
  if (threadIdx.x < rows * 3) {  // view encoding
    const int r = threadIdx.x / 3, c = threadIdx.x % 3;
    const float x = d[((m0 + r) / rows_per_src) * 3 + c];
    tv[r][c] = x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float sn, cs;
      sincosf(x * (float)(1 << k), &sn, &cs);
      tv[r][3 + 6 * k + c] = sn;
      tv[r][3 + 6 * k + 3 + c] = cs;
    }
  }
  for (int i = threadIdx.x; i < rows * n_a; i += blockDim.x) {
    const int r = i / n_a, j = i % n_a;
    tv[r][27 + j] = a[(long long)((m0 + r) / rows_per_src) * n_a + j];
  }
  __syncthreads();
  store_tile_planes(&t0[0][0], 128, 128, rows, IN0, n_planes, m0, 0);
  store_tile_planes(&t0[0][0], 128, 128, rows, IN5, n_planes, m0, 256);
  store_tile_planes(&tv[0][0], 128, 128, rows, FEATN, n_planes, m0, 256);
}
int launch_nerf_embed(const float* o, const float* d, const float* z, const float* sample_dist,
                      const float* pts4_in, const float* a, int n_a, int T, int rows_per_src, int M,
                      int n_planes, Planes IN0, Planes IN5, Planes FEATN, float* dists_out, cudaStream_t s) {
  NRW_CHECK(n_a >= 0 && 27 + n_a <= 128, NRW_ERR_ARG, "nerf_embed: n_a=%d", n_a);
  nerf_embed_kernel<<<cdiv(M, ER), 128, 0, s>>>(o, d, z, sample_dist, pts4_in, a, n_a, T, rows_per_src, M, n_planes, IN0, IN5,
                                                FEATN, dists_out);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- column sums: out[n] += sum_m rowscale[m] * X[m,n]  (bias gradients, sdf-head weight gradient) ----------
// X is either bf16 planes or fp32.  A block owns ROWS rows; a thread owns 8 consecutive columns (16-byte loads)
// of every (256 / (N/8))-th row; partial sums are combined in shared memory, then one atomicAdd per column.
static constexpr int CS_ROWS = 128;
__global__ void __launch_bounds__(256) colsum_kernel(Planes X, int n_planes, const float* __restrict__ Xf, int ld, int M,
                                                     int N, const float* __restrict__ rowscale, float* __restrict__ out,
                                                     float* __restrict__ out_rs) {
  __shared__ float red[256 * 8];
  const int tpr = N >> 3;                 // threads per row (N % 8 == 0, N <= 640 -> tpr <= 80)
  const int rpp = 256 / tpr;              // rows per pass
  const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
  const int row0 = blockIdx.x * CS_ROWS, row1 = min(M, row0 + CS_ROWS);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float rs_acc = 0.0f;
  if (tr < rpp) {
    for (int m = row0 + tr; m < row1; m += rpp) {
      const float rsc = rowscale ? rowscale[m] : 1.0f;
      if (tc == 0) rs_acc += rsc;
      float v[8];
      if (Xf) {
        const float4 a0 = *reinterpret_cast<const float4*>(Xf + (long long)m * ld + tc * 8);
        const float4 a1 = *reinterpret_cast<const float4*>(Xf + (long long)m * ld + tc * 8 + 4);
        v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = 0.0f;
        for (int pl = 0; pl < n_planes; ++pl) {
          const uint4 t = *reinterpret_cast<const uint4*>(X.plane(pl) + (long long)m * X.ld + tc * 8);
          const uint32_t u[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            v[2 * k] += __uint_as_float(u[k] << 16);
            v[2 * k + 1] += __uint_as_float(u[k] & 0xFFFF0000u);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = fmaf(rsc, v[k], acc[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[threadIdx.x * 8 + k] = acc[k];
  __syncthreads();
  // thread t < N sums column t over the rpp row groups
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const int c = n >> 3, k = n & 7;
    float s = 0.0f;
    for (int g = 0; g < rpp; ++g) s += red[(g * tpr + c) * 8 + k];
    atomicAdd(&out[n], s);
  }
  if (out_rs && tc == 0 && tr < rpp) atomicAdd(out_rs, rs_acc);
}
int launch_colsum(Planes X, int n_planes, const float* Xf, int ld, int M, int N, const float* rowscale,
                  float* out, float* out_rowscale_sum, cudaStream_t s) {
  NRW_CHECK(N % 8 == 0 && N <= 640, NRW_ERR_ARG, "colsum: N=%d must be a multiple of 8 and <= 640", N);
  colsum_kernel<<<cdiv(M, CS_ROWS), 256, 0, s>>>(X, n_planes, Xf, ld, M, N, rowscale, out, out_rowscale_sum);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
