// Epilogue of the tensor-core GEMM kernels: one 32-row x 16-column chunk per call.
//
// The GEMM hands lane r of a warp ROW r of the accumulator chunk (gemm_tc.cu stages it through shared memory).  Doing the global I/O in
// that layout would touch 32 different cache lines per instruction, so the chunk is transposed ONCE
// through a per-warp 2 KB shared staging tile (XOR-swizzled 16-byte slots, conflict-free both ways) into
// the "line" layout: lane L owns columns 4*(L&3)..+3 of rows (L>>2) + 8*it, it = 0..3.  In that layout
// every auxiliary load and every store of the epilogue is a direct, sector-aligned global access (8 rows
// x 64 B per fp32 instruction, 8 rows x 32 B per bf16 instruction) and all arithmetic is elementwise, so
// nothing else goes through shared memory.
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

// tile origin `src` = &matrix[m0w][nc]
__device__ __forceinline__ void line_load_f32(const LineLayout& L, const float* __restrict__ src, long long ld, int ncols,
                                              float (&o)[16]) {
  if (L.full && ncols >= 16 && aligned16(src) && (ld & 3) == 0) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(src + (long long)(it * 8 + L.r0) * ld + L.sl * 4));
      o[4 * it] = t.x; o[4 * it + 1] = t.y; o[4 * it + 2] = t.z; o[4 * it + 3] = t.w;
    }
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
  if (!atomic && L.full && ncols >= 16 && aligned16(dst) && (ld & 3) == 0) {
#pragma unroll
    for (int it = 0; it < 4; ++it)
      *reinterpret_cast<float4*>(dst + (long long)(it * 8 + L.r0) * ld + L.sl * 4) =
          make_float4(o[4 * it], o[4 * it + 1], o[4 * it + 2], o[4 * it + 3]);
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
// pk[2*it], pk[2*it+1] = the 4 bf16 of row it*8+r0
__device__ __forceinline__ void line_store_bf16(const LineLayout& L, bf16* __restrict__ dst, long long ld, int ncols,
                                                const uint32_t (&pk)[8]) {
  if (L.full && ncols >= 16 && aligned8(dst) && (ld & 3) == 0) {
#pragma unroll
    for (int it = 0; it < 4; ++it)
      *reinterpret_cast<uint2*>(dst + (long long)(it * 8 + L.r0) * ld + L.sl * 4) = make_uint2(pk[2 * it], pk[2 * it + 1]);
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
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const uint2 t = __ldg(reinterpret_cast<const uint2*>(src + (long long)(it * 8 + L.r0) * P.ld + L.sl * 4));
        o[4 * it] += __uint_as_float(t.x << 16);
        o[4 * it + 1] += __uint_as_float(t.x & 0xFFFF0000u);
        o[4 * it + 2] += __uint_as_float(t.y << 16);
        o[4 * it + 3] += __uint_as_float(t.y & 0xFFFF0000u);
      }
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
// bit e (= 4*it + k) set <=> src[row it*8+r0][col 4*sl+k] > 0
__device__ __forceinline__ uint32_t line_load_posmask(const LineLayout& L, const bf16* __restrict__ src, long long ld, int ncols) {
  uint32_t pos = 0;
  if (L.full && ncols >= 16 && aligned8(src) && (ld & 3) == 0) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const uint2 t = __ldg(reinterpret_cast<const uint2*>(src + (long long)(it * 8 + L.r0) * ld + L.sl * 4));
      const uint32_t u[2] = {t.x, t.y};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t lo = u[h] & 0xFFFFu, hi = u[h] >> 16;
        if (lo != 0u && lo < 0x8000u) pos |= 1u << (4 * it + 2 * h);
        if (hi != 0u && hi < 0x8000u) pos |= 1u << (4 * it + 2 * h + 1);
      }
    }
    return pos;
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + L.r0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = L.sl * 4 + k;
      if (rr < L.rows_valid && c < ncols && __bfloat162float(src[(long long)rr * ld + c]) > 0.0f) pos |= 1u << (4 * it + k);
    }
  }
  return pos;
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

// v: row `lane` of the accumulator chunk (columns nc..nc+15 of rows m0w..m0w+31).  stg: this warp's 2 KB tile.
// cs_tile: this CTA's shared column-sum accumulator for columns nc..nc+15 (flushed by the kernel), or nullptr.
__device__ __forceinline__ void epi_chunk16(const Epi& e, float* stg, const float (&v)[16], int m0w, int nc, int M, int N, int lane,
                                            float* cs_tile) {
  LineLayout L;
  L.rows_valid = min(32, M - m0w);
  if (L.rows_valid <= 0) return;   // warp-uniform
  const int n_all = min(N - nc, 16);
  const int n_st = min(e.n_store - nc, n_all);
  L.sl = lane & 3;
  L.r0 = lane >> 2;
  L.full = L.rows_valid == 32;
  // ---- the one transpose: row layout -> line layout (64-byte rows, slot' = slot ^ ((row >> 1) & 3)) ----
#pragma unroll
  for (int s = 0; s < 4; ++s)
    *reinterpret_cast<float4*>(stg + lane * 16 + ((s ^ ((lane >> 1) & 3)) << 2)) = make_float4(v[4 * s], v[4 * s + 1], v[4 * s + 2], v[4 * s + 3]);
  __syncwarp();
  float x[16];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + L.r0;
    const float4 t = *reinterpret_cast<const float4*>(stg + rr * 16 + ((L.sl ^ ((rr >> 1) & 3)) << 2));
    x[4 * it] = t.x; x[4 * it + 1] = t.y; x[4 * it + 2] = t.z; x[4 * it + 3] = t.w;
  }
  __syncwarp();   // the tile may be overwritten by the next chunk from here on
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
  if (e.out_pre) line_store_f32(L, e.out_pre + (long long)m0w * e.ld_pre + nc, e.ld_pre, n_all, x, false);
  if (e.out_pre_h) {
    uint32_t pk[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(x[2 * t], x[2 * t + 1]);
      pk[t] = *reinterpret_cast<const uint32_t*>(&h);
    }
    line_store_bf16(L, e.out_pre_h + (long long)m0w * e.ld_pre + nc, e.ld_pre, n_all, pk);
  }
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
  if (e.aux_sig || e.aux_u.p) {
    float a[16];
    const bool from_u = e.aux_u.p != nullptr;     // gate from the stored softplus OUTPUT planes (no fp32 pre-activation in HBM)
    if (from_u) line_load_planes(L, e.aux_u, e.aux_u_planes, m0w, nc, n_st, e.aux_u_scale, a);
    else line_load_f32(L, e.aux_sig + (long long)m0w * e.ld_aux + nc, e.ld_aux, n_st, a);
    if (e.out2 || e.out2_h) {
      float q[16];
      if (e.aux_q_h) {
        line_load_planes(L, Planes{const_cast<bf16*>(e.aux_q_h), 0, e.ld_aux}, 1, m0w, nc, n_st, 1.0f, q);
      } else if (e.aux_q_bcast) {
        float qb[4];
        line_load_cols(L, e.aux_q + nc, n_st, qb);
#pragma unroll
        for (int i = 0; i < 16; ++i) q[i] = qb[i & 3];
      } else {
        line_load_f32(L, e.aux_q + (long long)m0w * e.ld_aux + nc, e.ld_aux, n_st, q);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float s1, s2;
        if (from_u) softplus100_d12_from_u(a[i], s1, s2);
        else softplus100_d12(a[i], s1, s2);
        w[i] = x[i] * s1 * e.scale;
        q[i] = e.scale * x[i] * q[i] * s2;
      }
      if (e.out2_h) {
        uint32_t pk[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const __nv_bfloat162 h = __floats2bfloat162_rn(q[2 * t], q[2 * t + 1]);
          pk[t] = *reinterpret_cast<const uint32_t*>(&h);
        }
        line_store_bf16(L, e.out2_h + (long long)m0w * e.ld_out2 + nc, e.ld_out2, n_st, pk);
      } else {
        line_store_f32(L, e.out2 + (long long)m0w * e.ld_out2 + nc, e.ld_out2, n_st, q, false);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float s1, s2;
        if (from_u) softplus100_d12_from_u(a[i], s1, s2);
        else softplus100_d12(a[i], s1, s2);
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
      const uint32_t pos = line_load_posmask(L, e.aux_relu + (long long)m0w * e.ld_relu + nc, e.ld_relu, n_st);
#pragma unroll
      for (int i = 0; i < 16; ++i)
        if (!((pos >> i) & 1u)) w[i] = 0.0f;
    }
  }
  if (e.aux_add || e.aux_add_h) {
    float ad[16];
    if (e.aux_add_h) line_load_planes(L, Planes{const_cast<bf16*>(e.aux_add_h), 0, e.ld_aux}, 1, m0w, nc, n_st, 1.0f, ad);
    else line_load_f32(L, e.aux_add + (long long)m0w * e.ld_aux + nc, e.ld_aux, n_st, ad);
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] += ad[i];
  }
  if (e.colsum) {
    // column sums over the 32 rows: 4 rows per lane, then the 8 lanes sharing a column slot
    float cs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      cs[k] = 0.0f;
#pragma unroll
      for (int it = 0; it < 4; ++it) cs[k] += (it * 8 + L.r0 < L.rows_valid) ? w[4 * it + k] : 0.0f;
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) cs[k] += __shfl_xor_sync(0xFFFFFFFFu, cs[k], o);
    }
    if (lane < 4) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (lane * 4 + k < n_st) {
          if (cs_tile) atomicAdd(cs_tile + lane * 4 + k, cs[k]);   // shared-memory reduction (same-address global atomics serialise)
          else atomicAdd(e.colsum + nc + lane * 4 + k, cs[k]);
        }
    }
  }
  if (e.out_f32) line_store_f32(L, e.out_f32 + (long long)m0w * e.ld_f32 + nc, e.ld_f32, n_st, w, false);
  for (int pl = 0; pl < e.n_planes; ++pl) {
    uint32_t pk[8];
    split_plane<16>(w, pk);
    line_store_bf16(L, e.out_pl.plane(pl) + (long long)m0w * e.out_pl.ld + nc, e.out_pl.ld, n_st, pk);
  }
}

// Column-sum accumulator of one consumer warpgroup (the n_cols columns of its current n-tile; the chunk epilogues never
// touch an entry beyond n_cols, so those stay zero).  All `n_threads` threads of the warpgroup call this together (named
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
