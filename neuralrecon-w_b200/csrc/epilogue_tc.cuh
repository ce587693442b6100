// Epilogue of the tensor-core GEMM kernels: one 32-row x 16-column chunk per call.
//
// The GEMM hands a warp its 32 x 16 accumulator chunk in the "line" layout: lane L owns columns 4*(L&3)..+3 of rows (L>>2) + 8*it,
// it = 0..3 (gemm_tc.cu reads it that way out of the shared-memory tile it stages the accumulator fragments in).  In that
// layout every auxiliary load and every store of the epilogue is a direct, sector-aligned global access (8 rows x 64 B per
// fp32 instruction, 8 rows x 32 B per bf16 instruction) and all arithmetic is elementwise, so nothing else goes through
// shared memory.
//
// This file is the line-layout I/O layer both chunk epilogues use (the generic epi_chunk16 below and the specialised kinds of
// epilogue_fast.cuh): the full-tile accessors, the line accessors with their ragged / unaligned fallbacks, bf16 packing and
// column sums.
#pragma once
#include "epilogue.cuh"

namespace nrw {

struct LineLayout {
  int sl;        // 16-byte column slot 0..3
  int r0;        // first row 0..7
  int rows_valid;
  bool full;     // all 32 rows and all 16 columns valid (warp-uniform)
};

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
__device__ __forceinline__ bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

// Side-stream loads.  Warps working on neighbouring column chunks of the same rows read NEIGHBOURING 64-byte (fp32) /
// 32-byte (bf16) pieces of the same rows, so the first of them asks L2 to fetch the whole aligned 256 bytes
// (ld.global.nc.L2::256B): the other three find their sectors in L2 instead of queueing a second HBM round trip.
__device__ __forceinline__ float4 ldg4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L2::256B.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ uint2 ldg2u(const bf16* p) {
  uint2 v;
  asm volatile("ld.global.nc.L2::256B.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}

// ---- full-tile accessors: all 32 rows and 16 columns valid, 16-byte aligned rows.  p = this lane's first element (row r0,
// column 4*sl of the tile); o[4*it + k] = p[it*8*ld + k]. ----
__device__ __forceinline__ void tile_load_f32(const float* p, long long ld, float (&o)[16]) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const float4 t = ldg4(p + it * 8 * ld);
    o[4 * it] = t.x; o[4 * it + 1] = t.y; o[4 * it + 2] = t.z; o[4 * it + 3] = t.w;
  }
}
// bf16 tiles can stay packed in registers (8 words for 16 values) until they are used: tile_load_bf16 = raw load + unpack
__device__ __forceinline__ void tile_load_bf16_raw(const bf16* p, long long ld, uint2 (&r)[4]) {
#pragma unroll
  for (int it = 0; it < 4; ++it) r[it] = ldg2u(p + it * 8 * ld);
}
__device__ __forceinline__ void unpack_bf16(const uint2 (&r)[4], float (&o)[16]) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const uint2 t = r[it];
    o[4 * it] = __uint_as_float(t.x << 16); o[4 * it + 1] = __uint_as_float(t.x & 0xFFFF0000u);
    o[4 * it + 2] = __uint_as_float(t.y << 16); o[4 * it + 3] = __uint_as_float(t.y & 0xFFFF0000u);
  }
}
__device__ __forceinline__ void tile_load_bf16(const bf16* p, long long ld, float (&o)[16]) {
  uint2 r[4];
  tile_load_bf16_raw(p, ld, r);
  unpack_bf16(r, o);
}
__device__ __forceinline__ void tile_store_f32(float* p, long long ld, const float (&o)[16]) {
#pragma unroll
  for (int it = 0; it < 4; ++it)
    *reinterpret_cast<float4*>(p + it * 8 * ld) = make_float4(o[4 * it], o[4 * it + 1], o[4 * it + 2], o[4 * it + 3]);
}
// pk[2*it], pk[2*it+1] = the 4 bf16 of row it*8+r0
__device__ __forceinline__ void tile_store_bf16(bf16* p, long long ld, const uint32_t (&pk)[8]) {
#pragma unroll
  for (int it = 0; it < 4; ++it) *reinterpret_cast<uint2*>(p + it * 8 * ld) = make_uint2(pk[2 * it], pk[2 * it + 1]);
}
// w rounded to bf16 pairs without keeping the residual (split_plane<16> keeps it)
__device__ __forceinline__ void pack_bf16(const float (&w)[16], uint32_t (&pk)[8]) {
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(w[2 * t], w[2 * t + 1]);
    pk[t] = *reinterpret_cast<const uint32_t*>(&h);
  }
}
// a side stream's full tile at this lane's first element (row, col)
__device__ __forceinline__ void tile_load(const SideStream& s, long long row, int col, float (&o)[16]) {
  if (s.is_bf16()) tile_load_bf16(s.h() + row * s.ld + col, s.ld, o);
  else tile_load_f32(s.f32() + row * s.ld + col, s.ld, o);
}
__device__ __forceinline__ void tile_store(const SideStream& s, long long row, int col, const float (&o)[16]) {
  if (s.is_bf16()) {
    uint32_t pk[8];
    pack_bf16(o, pk);
    tile_store_bf16(s.h() + row * s.ld + col, s.ld, pk);
  } else {
    tile_store_f32(s.f32() + row * s.ld + col, s.ld, o);
  }
}

// ---- line accessors of the generic epilogue: any chunk (rows < L.rows_valid, columns < ncols), any alignment; full aligned
// tiles take the full-tile accessors.  `src` / `dst` = tile origin &matrix[m0w][nc]. ----
__device__ __forceinline__ bool line_fast(const LineLayout& L, const void* p, long long ld, int ncols) {
  return L.full && ncols >= 16 && aligned16(p) && (ld & 3) == 0;
}
__device__ __forceinline__ void line_load_f32(const LineLayout& L, const float* __restrict__ src, long long ld, int ncols,
                                              float (&o)[16]) {
  if (line_fast(L, src, ld, ncols)) {
    tile_load_f32(src + L.r0 * ld + L.sl * 4, ld, o);
    return;
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + L.r0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = L.sl * 4 + k;
      o[4 * it + k] = (rr < L.rows_valid && c < ncols) ? src[(long long)rr * ld + c] : 0.0f;
    }
  }
}
__device__ __forceinline__ void line_store_f32(const LineLayout& L, float* __restrict__ dst, long long ld, int ncols,
                                               const float (&o)[16], bool atomic) {
  if (!atomic && line_fast(L, dst, ld, ncols)) {
    tile_store_f32(dst + L.r0 * ld + L.sl * 4, ld, o);
    return;
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + L.r0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = L.sl * 4 + k;
      if (rr < L.rows_valid && c < ncols) {
        if (atomic) atomicAdd(dst + (long long)rr * ld + c, o[4 * it + k]);
        else dst[(long long)rr * ld + c] = o[4 * it + k];
      }
    }
  }
}
__device__ __forceinline__ void line_store_bf16(const LineLayout& L, bf16* __restrict__ dst, long long ld, int ncols,
                                                const uint32_t (&pk)[8]) {
  if (L.full && ncols >= 16 && aligned8(dst) && (ld & 3) == 0) {
    tile_store_bf16(dst + L.r0 * ld + L.sl * 4, ld, pk);
    return;
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + L.r0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = L.sl * 4 + k;
      if (rr < L.rows_valid && c < ncols)
        dst[(long long)rr * ld + c] = __ushort_as_bfloat16((unsigned short)((pk[2 * it + (k >> 1)] >> ((k & 1) * 16)) & 0xFFFFu));
    }
  }
}
// o[4*it + k] = scale * sum over planes of P[row it*8+r0][col 4*sl+k]   (tile origin: row m0w, column nc of P)
__device__ __forceinline__ void line_load_planes(const LineLayout& L, const Planes& P, int n_planes, long long m0w, int nc, int ncols,
                                                 float scale, float (&o)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i] = 0.0f;
  for (int pl = 0; pl < n_planes; ++pl) {
    const bf16* src = P.plane(pl) + m0w * P.ld + nc;
    if (L.full && ncols >= 16 && aligned8(src) && (P.ld & 3) == 0) {
      float t[16];
      tile_load_bf16(src + L.r0 * P.ld + L.sl * 4, P.ld, t);
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] += t[i];
    } else {
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + L.r0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = L.sl * 4 + k;
          if (rr < L.rows_valid && c < ncols) o[4 * it + k] += __bfloat162float(src[(long long)rr * P.ld + c]);
        }
      }
    }
  }
  if (scale != 1.0f) {
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] *= scale;
  }
}
// per-column [N] vector: the 4 values of this lane's column slot
__device__ __forceinline__ void line_load_cols(const LineLayout& L, const float* __restrict__ vec, int ncols, float (&b)[4]) {
  const float* p = vec + L.sl * 4;
  if (ncols >= 16 && aligned16(vec)) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    b[0] = t.x; b[1] = t.y; b[2] = t.z; b[3] = t.w;
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) b[k] = (L.sl * 4 + k < ncols) ? p[k] : 0.0f;
  }
}
__device__ __forceinline__ void line_load(const LineLayout& L, const SideStream& s, long long m0w, int nc, int ncols, float (&o)[16]) {
  if (s.is_bf16()) line_load_planes(L, Planes{s.h(), 0, s.ld}, 1, m0w, nc, ncols, 1.0f, o);
  else line_load_f32(L, s.f32() + m0w * s.ld + nc, s.ld, ncols, o);
}
__device__ __forceinline__ void line_store(const LineLayout& L, const SideStream& s, long long m0w, int nc, int ncols,
                                           const float (&o)[16]) {
  if (s.is_bf16()) {
    uint32_t pk[8];
    pack_bf16(o, pk);
    line_store_bf16(L, s.h() + m0w * s.ld + nc, s.ld, ncols, pk);
  } else {
    line_store_f32(L, s.f32() + m0w * s.ld + nc, s.ld, ncols, o, false);
  }
}

// column sums of a 32 x 16 line-layout tile into this CTA's shared accumulator cs_tile[16]: rows first (registers), then a
// halving butterfly over the 8 lanes that share a column slot: 4 SHFL instead of 12
__device__ __forceinline__ void line_colsum_add(const float (&w)[16], int lane, float* cs_tile) {
  float c0 = (w[0] + w[4]) + (w[8] + w[12]), c1 = (w[1] + w[5]) + (w[9] + w[13]);
  float c2 = (w[2] + w[6]) + (w[10] + w[14]), c3 = (w[3] + w[7]) + (w[11] + w[15]);
  const bool hi16 = (lane & 16) != 0, hi8 = (lane & 8) != 0;
  // round 1 (xor 16): lanes with bit 4 clear keep columns 0,1; the others keep 2,3
  const float s0 = hi16 ? c0 : c2, s1 = hi16 ? c1 : c3;
  float k0 = hi16 ? c2 : c0, k1 = hi16 ? c3 : c1;
  k0 += __shfl_xor_sync(0xFFFFFFFFu, s0, 16);
  k1 += __shfl_xor_sync(0xFFFFFFFFu, s1, 16);
  // round 2 (xor 8): bit 3 clear keeps the first of the two, set keeps the second
  const float s = hi8 ? k0 : k1;
  float k = hi8 ? k1 : k0;
  k += __shfl_xor_sync(0xFFFFFFFFu, s, 8);
  // round 3 (xor 4): both partners hold the same column
  k += __shfl_xor_sync(0xFFFFFFFFu, k, 4);
  if ((lane & 4) == 0) atomicAdd(cs_tile + (lane & 3) * 4 + (hi16 ? 2 : 0) + (hi8 ? 1 : 0), k);   // shared-memory reduction
}

// softplus gates from the stored softplus OUTPUT, 3 instructions: e = 2^(-100 log2(e) u) = 1 - sigmoid(100 a); s1 = 1 - e.
// (No small-argument series and no threshold select as in softplus100_d12_from_u: the absolute error of s1 is <= 1 ulp of
//  1.0 = 6e-8 and s2 = 100 s1 e is 2e-7 instead of exactly 0 above the softplus threshold - both far below the
//  accumulation error of the GEMM that produced the value the gate multiplies.)  GATE_FWD's gate (the normal chain of a
// forward) is formed alike in epi_chunk16 and in the specialised kind (epilogue_fast.cuh fast_finish), so a point's
// normal does not depend on whether its 32-row group reaches past M and takes epi_chunk16.  The backward gates of
// epi_chunk16 (TANGENT's out2, REVERSE's aux_add) keep softplus100_d12_from_u.
#define NRW_GATE_K (-144.269504088896341f)   // -100 * log2(e)

// x_acc: the accumulator chunk (columns nc..nc+15 of rows m0w..m0w+31) in the line layout.
// cs_tile: this CTA's shared column-sum accumulator for columns nc..nc+15 (flushed by the kernel); non-null iff e.colsum is set
// and the epilogue is not atomic.
__device__ __forceinline__ void epi_chunk16(const Epi& e, const float (&x_acc)[16], int m0w, int nc, int M, int N, int lane,
                                            float* cs_tile) {
  LineLayout L;
  L.rows_valid = min(32, M - m0w);
  if (L.rows_valid <= 0) return;   // warp-uniform
  const int n_all = min(N - nc, 16);
  const int n_st = min(e.n_store - nc, n_all);
  L.sl = lane & 3;
  L.r0 = lane >> 2;
  L.full = L.rows_valid == 32;
  float x[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) x[i] = x_acc[i];
  // ---- v = acc + bias + rowvec * colvec ----
  if (e.bias) {
    float b[4];
    line_load_cols(L, e.bias + nc, n_all, b);
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] += b[i & 3];
  }
  if (e.rowvec) {
    float cv[4];
    line_load_cols(L, e.colvec + nc, n_all, cv);
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const float rv = e.rowvec[min(m0w + it * 8 + L.r0, M - 1)];
#pragma unroll
      for (int k = 0; k < 4; ++k) x[4 * it + k] = fmaf(rv, cv[k], x[4 * it + k]);
    }
  }
  if (e.out_pre) line_store(L, e.out_pre, m0w, nc, n_all, x);
  if (n_st <= 0) return;
  if (e.atomic) {
    if (e.scale != 1.0f) {
#pragma unroll
      for (int i = 0; i < 16; ++i) x[i] *= e.scale;
    }
    line_store_f32(L, e.out_f32 + (long long)m0w * e.ld_f32 + nc, e.ld_f32, n_st, x, true);
    return;
  }
  // ---- activation / gating (elementwise, see epilogue.cuh) ----
  float w[16];
  if (e.aux_u.p && !e.out2 && !e.aux_add) {
    // GATE_FWD's gate exactly as fast_finish forms it (u = the plain sum of the planes, the plane scale folded into the
    // exponent's constant): a row's normal-chain value does not depend on whether its 32-row group is full
    float u[16];
    line_load_planes(L, e.aux_u, e.aux_u_planes, m0w, nc, n_st, 1.0f, u);
    const float kk = NRW_GATE_K * e.aux_u_scale, sc = e.scale;
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = x[i] * fmaf(-sc, mufu_ex2(u[i] * kk), sc);
  } else if (e.aux_u.p) {
    float a[16];   // the gate from the stored softplus OUTPUT planes (no fp32 pre-activation in HBM)
    line_load_planes(L, e.aux_u, e.aux_u_planes, m0w, nc, n_st, e.aux_u_scale, a);
    if (e.out2) {
      float q[16];
      if (e.aux_q_bcast) {
        float qb[4];
        line_load_cols(L, e.aux_q.f32() + nc, n_st, qb);
#pragma unroll
        for (int i = 0; i < 16; ++i) q[i] = qb[i & 3];
      } else {
        line_load(L, e.aux_q, m0w, nc, n_st, q);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float s1, s2;
        softplus100_d12_from_u(a[i], s1, s2);
        w[i] = x[i] * s1 * e.scale;
        q[i] = e.scale * x[i] * q[i] * s2;
      }
      line_store(L, e.out2, m0w, nc, n_st, q);
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float s1, s2;
        softplus100_d12_from_u(a[i], s1, s2);
        w[i] = x[i] * s1 * e.scale;
      }
    }
  } else {
    switch (e.act) {
      case ACT_SOFTPLUS100:
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = softplus100(x[i]) * e.scale;
        break;
      case ACT_RELU:
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = fmaxf(x[i], 0.0f) * e.scale;
        break;
      case ACT_SIGMOID:
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = sigmoidf_(x[i]) * e.scale;
        break;
      default:
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = x[i] * e.scale;
    }
    if (e.aux_relu) {
      float f[16];   // forward activation: 0 outside the chunk
      line_load_planes(L, Planes{const_cast<bf16*>(e.aux_relu), 0, e.ld_relu}, 1, m0w, nc, n_st, 1.0f, f);
#pragma unroll
      for (int i = 0; i < 16; ++i)
        if (!(f[i] > 0.0f)) w[i] = 0.0f;
    }
  }
  if (e.aux_add) {
    float ad[16];
    line_load(L, e.aux_add, m0w, nc, n_st, ad);
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] += ad[i];
  }
  if (cs_tile) {
    // rows and columns outside the chunk add nothing: the accumulator's entries at or beyond the tile's column count stay zero
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if ((i >> 2) * 8 + L.r0 >= L.rows_valid || L.sl * 4 + (i & 3) >= n_st) w[i] = 0.0f;
    line_colsum_add(w, lane, cs_tile);
  }
  if (e.out_f32) line_store_f32(L, e.out_f32 + (long long)m0w * e.ld_f32 + nc, e.ld_f32, n_st, w, false);
  for (int pl = 0; pl < e.n_planes; ++pl) {
    uint32_t pk[8];
    split_plane<16>(w, pk);
    line_store_bf16(L, e.out_pl.plane(pl) + (long long)m0w * e.out_pl.ld + nc, e.out_pl.ld, n_st, pk);
  }
}

// Column-sum accumulator of one consumer warpgroup (the n_cols columns of its current n-tile; the chunk epilogues add only
// zeros to the entries beyond n_cols, so those stay zero).  All `n_threads` threads of the warpgroup call this together (named
// barrier `bar_id`): adds the tile's partial sums to global memory and clears the accumulator.
__device__ __forceinline__ void colsum_flush(float* cs, float* __restrict__ colsum, int n0, int n_cols, int tid, int n_threads,
                                             int bar_id) {
  asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(n_threads) : "memory");
  for (int i = tid; i < n_cols; i += n_threads) {
    const float s = cs[i];
    if (i < n_cols && s != 0.0f) atomicAdd(colsum + n0 + i, s);
    cs[i] = 0.0f;
  }
  asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(n_threads) : "memory");
}

}  // namespace nrw
