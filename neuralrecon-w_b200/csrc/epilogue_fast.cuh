// Compile-time specialised epilogues of the tensor-core GEMM for the eight layer kinds that make up > 95 % of a
// training step.  Same arithmetic, in the same order, as the runtime-parameterised epi_chunk16 (epilogue_tc.cuh) - the
// difference is what is NOT executed: ncu's source view of the generic epilogue showed ISETP + BRA + LOP3 + IMAD + LDC
// (flag tests, alignment checks, 64-bit address arithmetic, ReLU bit masks) at > 50 % of all issued instructions and
// the useful FADD / FMUL / F2FP at ~12 % with the backward layers of the
// `mixed` mode (one MMA product) bound by epilogue instruction issue, not by the tensor pipe or HBM.
//
// A kind is chosen on the host (pick_epi_kind) from the Epi descriptor; anything that does not match exactly, ragged
// edge tiles and the column boundary of the skip layer (n_store = 473) fall back to epi_chunk16, warp-uniformly.
#pragma once
#include "epilogue_tc.cuh"

namespace nrw {

enum EpiKind {
  EK_GENERIC = 0,
  EK_FWD_SOFTPLUS,   // x + bias -> softplus100 -> * scale -> planes                              (SDF forward layers)
  EK_FWD_RELU,       // x + bias -> relu -> planes                                                 (colour / NeRF forward)
  EK_FWD_NONE,       // x + bias -> planes                                                         (feature layers)
  EK_GATE_FWD,       // out_pre = x ; w = x * softplus'(a) * scale -> planes                       (gradient chain, forward)
  EK_TANGENT,        // w = x * s1 * scale ; out2 = scale * x * q * s2 ; w -> planes | out_f32     (tangent sweep)
  EK_REVERSE,        // [x += rv * cv] ; w = x * s1 * scale + aux_add -> planes (+ column sums)    (reverse sweep)
  EK_RELU_BWD,       // [x += rv * cv] ; w = relu'(fwd) ? x * scale : 0 -> planes (+ column sums)  (ReLU nets, backward)
  EK_FWD_HEAD,       // softplus(x + bias) . head_w row partials, NO activation store               (last SDF layer of a forward-only query)
  EK_COUNT
};

// host: which specialisation implements `e` exactly (pointers 16-byte aligned, leading dimensions % 4 == 0 assumed by the
// fast paths are verified here once per launch instead of once per chunk)
inline int pick_epi_kind(const Epi& e) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (e.head_w || e.head_partial)
    return (e.head_w && e.head_partial && e.bias && al16(e.bias) && al16(e.head_w) && e.act == ACT_SOFTPLUS100 && e.scale == 1.0f && e.n_planes == 0 &&
            !e.atomic && !e.aux_sig && !e.aux_u.p && !e.rowvec && !e.aux_relu && !e.out_pre && !e.out_pre_h && !e.out2 && !e.out2_h && !e.out_f32 &&
            !e.colsum && !e.aux_add && !e.aux_add_h && e.n_store >= (1 << 29)) ? EK_FWD_HEAD : -1;      // -1: unsupported combination
  if (e.atomic || e.aux_sig || e.n_planes > 3) return EK_GENERIC;
  if (e.n_planes > 0 && (!al16(e.out_pl.p) || (e.out_pl.ld & 3) || (e.out_pl.pstride & 7))) return EK_GENERIC;
  if (e.aux_u.p && (!al16(e.aux_u.p) || (e.aux_u.ld & 3) || (e.aux_u.pstride & 7))) return EK_GENERIC;
  const bool pre = e.out_pre || e.out_pre_h, o2 = e.out2 || e.out2_h, q = e.aux_q || e.aux_q_h, add = e.aux_add || e.aux_add_h;
  if ((e.out_pre && e.out_pre_h) || (e.out2 && e.out2_h) || (e.aux_q && e.aux_q_h) || (e.aux_add && e.aux_add_h)) return EK_GENERIC;
  if ((pre && (!al16(e.out_pre) || !al16(e.out_pre_h) || (e.ld_pre & 3))) || (e.out_f32 && (!al16(e.out_f32) || (e.ld_f32 & 3))) ||
      (o2 && (!al16(e.out2) || !al16(e.out2_h) || (e.ld_out2 & 3))) || ((add || (q && !e.aux_q_bcast)) && (e.ld_aux & 3)) ||
      !al16(e.aux_add) || !al16(e.aux_add_h) || !al16(e.aux_q) || !al16(e.aux_q_h) ||
      (e.aux_relu && (!al16(e.aux_relu) || (e.ld_relu & 3))) || (e.bias && !al16(e.bias)) || (e.colvec && !al16(e.colvec)))
    return EK_GENERIC;
  const bool gate = e.aux_u.p != nullptr;
  if (gate && pre && !o2 && !add && !e.colsum && !e.bias && !e.rowvec && !e.aux_relu && e.n_planes > 0 && !e.out_f32)
    return EK_GATE_FWD;
  if (gate && o2 && q && !pre && !e.bias && !e.rowvec && !add && !e.colsum && !e.aux_relu &&
      ((e.n_planes > 0) != (e.out_f32 != nullptr)))
    return EK_TANGENT;
  if (gate && add && !o2 && !pre && !e.bias && !e.aux_relu && e.n_planes > 0 && !e.out_f32) return EK_REVERSE;
  if (!gate && e.aux_relu && !pre && !o2 && !add && !e.bias && e.n_planes > 0 && !e.out_f32 && e.act == ACT_NONE)
    return EK_RELU_BWD;
  if (!gate && e.bias && !e.rowvec && !e.aux_relu && !add && !pre && !o2 && !e.out_f32 && !e.colsum && e.n_planes > 0) {
    if (e.act == ACT_SOFTPLUS100) return EK_FWD_SOFTPLUS;
    if (e.act == ACT_RELU) return EK_FWD_RELU;
    if (e.act == ACT_NONE) return EK_FWD_NONE;
  }
  return EK_GENERIC;
}

// Side-stream loads of the epilogue.  Warps working on neighbouring column chunks of the same rows read NEIGHBOURING 64-byte (fp32) /
// 32-byte (bf16) pieces of the same rows, so the first of them asks L2 to fetch the whole aligned 256 bytes
// (ld.global.nc.L2::256B): the other three find their sectors in L2 instead of queueing a second HBM round trip.
#ifndef NRW_EPI_L2_256B
#define NRW_EPI_L2_256B 1
#endif
__device__ __forceinline__ float4 ldg4(const float* p) {
#if NRW_EPI_L2_256B
  float4 v;
  asm volatile("ld.global.nc.L2::256B.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
#else
  return __ldg(reinterpret_cast<const float4*>(p));
#endif
}
__device__ __forceinline__ uint2 ldg2u(const bf16* p) {
#if NRW_EPI_L2_256B
  uint2 v;
  asm volatile("ld.global.nc.L2::256B.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
#else
  return __ldg(reinterpret_cast<const uint2*>(p));
#endif
}
__device__ __forceinline__ void unpack_bf16x4(const uint2 t, float (&o)[4]) {
  o[0] = __uint_as_float(t.x << 16); o[1] = __uint_as_float(t.x & 0xFFFF0000u);
  o[2] = __uint_as_float(t.y << 16); o[3] = __uint_as_float(t.y & 0xFFFF0000u);
}

// softplus gates from the stored softplus OUTPUT, 3 instructions: e = 2^(-100 log2(e) u) = 1 - sigmoid(100 a); s1 = 1 - e.
// (No small-argument series and no threshold select as in softplus100_d12_from_u: the absolute error of s1 is <= 1 ulp of
//  1.0 = 6e-8 and s2 = 100 s1 e is 2e-7 instead of exactly 0 above the softplus threshold - both far below the
//  accumulation error of the GEMM that produced the value the gate multiplies.)
#define NRW_GATE_K (-144.269504088896341f)   // -100 * log2(e)

// column sums of a 32 x 16 line-layout tile (w[4*it + k] = row it*8 + (lane>>2), column 4*(lane&3) + k) into cs[16]:
// rows first (registers), then a halving butterfly over the 8 lanes that share a column slot: 4 SHFL instead of 12
__device__ __forceinline__ void line_colsum_add(const float (&w)[16], int lane, float* cs_tile, float* cs_global) {
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
  if ((lane & 4) == 0) {
    const int colk = (lane & 3) * 4 + (hi16 ? 2 : 0) + (hi8 ? 1 : 0);
    if (cs_tile) atomicAdd(cs_tile + colk, k);
    else atomicAdd(cs_global + colk, k);
  }
}

// `sa` (optional): the chunk's side streams already staged in shared memory as [32 rows][16 columns] bf16 boxes.
__device__ __forceinline__ bool epi_fast_eligible(const Epi& e, int m0w, int nc, int M, int N) {
  return M - m0w >= 32 && N - nc >= 16 && e.n_store - nc >= 16;
}
// host: the (at most two) bf16 side streams of kind `ek` that fit the 2 KB staging slot of a chunk: pointer + leading dimension
// of stream 0 / stream 1; returns the stream mask (0 = this launch keeps the register loads)
inline int pick_aux_streams(const Epi& e, int ek, const bf16** p0, int* ld0, const bf16** p1, int* ld1) {
  *p0 = *p1 = nullptr; *ld0 = *ld1 = 0;
  switch (ek) {
    case EK_GATE_FWD:
      if (e.aux_u_planes < 1 || e.aux_u_planes > 2) return 0;
      *p0 = e.aux_u.p; *ld0 = e.aux_u.ld;
      if (e.aux_u_planes == 2) { *p1 = e.aux_u.p + e.aux_u.pstride; *ld1 = e.aux_u.ld; }
      return e.aux_u_planes == 2 ? 3 : 1;
    case EK_TANGENT:
      if (e.aux_u_planes != 1 || !(e.aux_q_h || e.aux_q_bcast)) return 0;
      *p0 = e.aux_u.p; *ld0 = e.aux_u.ld;
      if (e.aux_q_h) { *p1 = e.aux_q_h; *ld1 = e.ld_aux; }
      return e.aux_q_h ? 3 : 1;
    case EK_REVERSE:
      if (e.aux_u_planes != 1 || !e.aux_add_h) return 0;
      *p0 = e.aux_u.p; *ld0 = e.aux_u.ld; *p1 = e.aux_add_h; *ld1 = e.ld_aux;
      return 3;
    case EK_RELU_BWD:
      *p0 = e.aux_relu; *ld0 = e.ld_relu;
      return 1;
    default: return 0;
  }
}

template <int EK>
__device__ __forceinline__ void epi_fast16(const Epi& e, float* stg, const float (&v)[16], int m0w, int nc, int M, int N, int lane,
                                           float* cs_tile, const uint8_t* sa = nullptr, int aux_mask = 0, float* hacc = nullptr) {
  if constexpr (EK == EK_GENERIC) {
    epi_chunk16(e, stg, v, m0w, nc, M, N, lane, cs_tile);
    return;
  } else if constexpr (EK == EK_FWD_HEAD) {
    // every row of the 32-row group is processed (rows beyond M hold zero-filled operands and are never written); only
    // column-indexed vectors are read, so there is no ragged fallback.  hacc[it] accumulates this lane's rows over the
    // warp's chunks of the tile in a FIXED order (deterministic SDF values).
    const int sl = lane & 3;
    const int col = nc + sl * 4;
    const float4 b = ldg4(e.bias + col), hw = ldg4(e.head_w + col);
#pragma unroll
    for (int s = 0; s < 4; ++s)
      *reinterpret_cast<float4*>(stg + lane * 16 + ((s ^ ((lane >> 1) & 3)) << 2)) = make_float4(v[4 * s], v[4 * s + 1], v[4 * s + 2], v[4 * s + 3]);
    __syncwarp();
    const int r0 = lane >> 2;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = it * 8 + r0;
      const float4 t = *reinterpret_cast<const float4*>(stg + rr * 16 + ((sl ^ ((rr >> 1) & 3)) << 2));
      float p = softplus100(t.x + b.x) * hw.x;
      p = fmaf(softplus100(t.y + b.y), hw.y, p);
      p = fmaf(softplus100(t.z + b.z), hw.z, p);
      p = fmaf(softplus100(t.w + b.w), hw.w, p);
      p += __shfl_xor_sync(0xFFFFFFFFu, p, 1);
      p += __shfl_xor_sync(0xFFFFFFFFu, p, 2);
      hacc[it] += p;
    }
    __syncwarp();
    return;
  } else {
    // ragged edge tile / column boundary of the stored range: the generic path handles every case
    if (M - m0w < 32 || N - nc < 16 || e.n_store - nc < 16) {
      epi_chunk16(e, stg, v, m0w, nc, M, N, lane, cs_tile);
      return;
    }
    const int sl = lane & 3, r0 = lane >> 2;
    const int col = nc + sl * 4;                      // this lane's 4 columns
    const long long row = (long long)m0w + r0;        // this lane's first row; rows row + 8*it
    // ---- auxiliary streams first (raw registers): their latency overlaps the transpose below ----
    uint2 ru0[4];                     // first gate plane (further planes are loaded in place below, except GATE_FWD's second)
    float4 rf[4];                     // fp32 side stream (aux_q / aux_add), or its bf16 twin's raw bits in .x/.y;
                                      // GATE_FWD: raw bits of the SECOND gate plane in .x/.y (its own exposed round trip was
                                      // 15 % of the stall samples); FWD_*: the bias in rf[0]
    // `sa` != nullptr: the side streams of this chunk are in shared memory:
    // stream 0 at sa, stream 1 at sa + 1024, each a row-major [32 rows][16 columns] bf16 box (32 bytes per row)
    const bool staged = sa != nullptr;
    if (staged) {
#pragma unroll
      for (int it = 0; it < 4; ++it) ru0[it] = *reinterpret_cast<const uint2*>(sa + (it * 8 + r0) * 32 + sl * 8);
      if (aux_mask & 2) {
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const uint2 t = *reinterpret_cast<const uint2*>(sa + 1024 + (it * 8 + r0) * 32 + sl * 8);
          rf[it].x = __uint_as_float(t.x); rf[it].y = __uint_as_float(t.y);
        }
      }
    }
    if constexpr (EK == EK_GATE_FWD || EK == EK_TANGENT || EK == EK_REVERSE) {
      const bf16* up = e.aux_u.p + row * e.aux_u.ld + col;
      if (!staged) {
#pragma unroll
        for (int it = 0; it < 4; ++it) ru0[it] = ldg2u(up + (long long)it * 8 * e.aux_u.ld);
      }
      if constexpr (EK == EK_GATE_FWD) {
        if (e.aux_u_planes > 1 && !staged) {
          const bf16* up1 = up + e.aux_u.pstride;
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const uint2 t = ldg2u(up1 + (long long)it * 8 * e.aux_u.ld);
            rf[it].x = __uint_as_float(t.x); rf[it].y = __uint_as_float(t.y);
          }
        }
      }
    }
    if constexpr (EK == EK_FWD_SOFTPLUS || EK == EK_FWD_RELU || EK == EK_FWD_NONE) rf[0] = ldg4(e.bias + col);
    if constexpr (EK == EK_TANGENT) {
      if (staged && (aux_mask & 2)) {
        // aux_q_h arrived through the staging slot
      } else if (e.aux_q_h) {
        const bf16* qp = e.aux_q_h + row * e.ld_aux + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const uint2 t = ldg2u(qp + (long long)it * 8 * e.ld_aux);
          rf[it].x = __uint_as_float(t.x); rf[it].y = __uint_as_float(t.y);
        }
      } else if (!e.aux_q_bcast) {
        const float* qp = e.aux_q + row * e.ld_aux + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) rf[it] = ldg4(qp + (long long)it * 8 * e.ld_aux);
      } else {
        const float4 qb = ldg4(e.aux_q + col);
#pragma unroll
        for (int it = 0; it < 4; ++it) rf[it] = qb;
      }
    }
    if constexpr (EK == EK_REVERSE) {
      if (staged && (aux_mask & 2)) {
        // aux_add_h arrived through the staging slot
      } else if (e.aux_add_h) {
        const bf16* ap = e.aux_add_h + row * e.ld_aux + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const uint2 t = ldg2u(ap + (long long)it * 8 * e.ld_aux);
          rf[it].x = __uint_as_float(t.x); rf[it].y = __uint_as_float(t.y);
        }
      } else {
        const float* ap = e.aux_add + row * e.ld_aux + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) rf[it] = ldg4(ap + (long long)it * 8 * e.ld_aux);
      }
    }
    if constexpr (EK == EK_RELU_BWD) {
      if (!staged) {
        const bf16* rp = e.aux_relu + row * e.ld_relu + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) ru0[it] = ldg2u(rp + (long long)it * 8 * e.ld_relu);
      }
    }
    // ---- the one transpose: row layout -> line layout (identical to epi_chunk16) ----
#pragma unroll
    for (int s = 0; s < 4; ++s)
      *reinterpret_cast<float4*>(stg + lane * 16 + ((s ^ ((lane >> 1) & 3)) << 2)) = make_float4(v[4 * s], v[4 * s + 1], v[4 * s + 2], v[4 * s + 3]);
    __syncwarp();
    float x[16];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = it * 8 + r0;
      const float4 t = *reinterpret_cast<const float4*>(stg + rr * 16 + ((sl ^ ((rr >> 1) & 3)) << 2));
      x[4 * it] = t.x; x[4 * it + 1] = t.y; x[4 * it + 2] = t.z; x[4 * it + 3] = t.w;
    }
    __syncwarp();
    float w[16];

    if constexpr (EK == EK_FWD_SOFTPLUS || EK == EK_FWD_RELU || EK == EK_FWD_NONE) {
      const float bb[4] = {rf[0].x, rf[0].y, rf[0].z, rf[0].w};     // loaded before the transpose
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float t = x[i] + bb[i & 3];
        if constexpr (EK == EK_FWD_SOFTPLUS) w[i] = softplus100(t) * e.scale;
        else if constexpr (EK == EK_FWD_RELU) w[i] = fmaxf(t, 0.0f) * e.scale;
        else w[i] = t * e.scale;
      }
    }
    if constexpr (EK == EK_REVERSE || EK == EK_RELU_BWD) {
      if (e.rowvec) {
        const float4 c = ldg4(e.colvec + col);
        const float cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const float rv = __ldg(e.rowvec + row + it * 8);
#pragma unroll
          for (int k = 0; k < 4; ++k) x[4 * it + k] = fmaf(rv, cc[k], x[4 * it + k]);
        }
      }
    }
    if constexpr (EK == EK_GATE_FWD) {
      if (e.out_pre_h) {
        bf16* op = e.out_pre_h + row * e.ld_pre + col;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const __nv_bfloat162 a = __floats2bfloat162_rn(x[4 * it], x[4 * it + 1]), b = __floats2bfloat162_rn(x[4 * it + 2], x[4 * it + 3]);
          *reinterpret_cast<uint2*>(op + (long long)it * 8 * e.ld_pre) =
              make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
        }
      } else {
        float* op = e.out_pre + row * e.ld_pre + col;
#pragma unroll
        for (int it = 0; it < 4; ++it)
          *reinterpret_cast<float4*>(op + (long long)it * 8 * e.ld_pre) = make_float4(x[4 * it], x[4 * it + 1], x[4 * it + 2], x[4 * it + 3]);
      }
    }
    if constexpr (EK == EK_GATE_FWD || EK == EK_TANGENT || EK == EK_REVERSE) {
      // u = sum(planes of the softplus output); e = 2^(K u) with the plane scale folded into K
      float u[16];
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        float t4[4];
        unpack_bf16x4(ru0[it], t4);
#pragma unroll
        for (int k = 0; k < 4; ++k) u[4 * it + k] = t4[k];
      }
      for (int pl = 1; pl < e.aux_u_planes; ++pl) {         // further planes: hoisted (GATE_FWD, plane 1) or loaded in place
        const bf16* up = e.aux_u.plane(pl) + row * e.aux_u.ld + col;
        const bool hoisted = EK == EK_GATE_FWD && pl == 1;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          float t4[4];
          unpack_bf16x4(hoisted ? make_uint2(__float_as_uint(rf[it].x), __float_as_uint(rf[it].y)) : ldg2u(up + (long long)it * 8 * e.aux_u.ld), t4);
#pragma unroll
          for (int k = 0; k < 4; ++k) u[4 * it + k] += t4[k];
        }
      }
      const float kk = NRW_GATE_K * e.aux_u_scale, sc = e.scale;
      if constexpr (EK == EK_TANGENT) {
        float q[16];
        if (e.aux_q_h) {
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            float t4[4];
            unpack_bf16x4(make_uint2(__float_as_uint(rf[it].x), __float_as_uint(rf[it].y)), t4);
            q[4 * it] = t4[0]; q[4 * it + 1] = t4[1]; q[4 * it + 2] = t4[2]; q[4 * it + 3] = t4[3];
          }
        } else {
#pragma unroll
          for (int it = 0; it < 4; ++it) { q[4 * it] = rf[it].x; q[4 * it + 1] = rf[it].y; q[4 * it + 2] = rf[it].z; q[4 * it + 3] = rf[it].w; }
        }
        const float sc100 = 100.0f * sc;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float ee = mufu_ex2(u[i] * kk);
          const float s1 = 1.0f - ee;
          const float xs = x[i] * s1;
          w[i] = xs * sc;                                  // x * softplus'(a) * scale
          q[i] = (xs * q[i]) * (ee * sc100);               // scale * x * q * softplus''(a),  softplus'' = 100 s1 e
        }
        if (e.out2_h) {
          bf16* o2 = e.out2_h + row * e.ld_out2 + col;
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const __nv_bfloat162 a = __floats2bfloat162_rn(q[4 * it], q[4 * it + 1]), b = __floats2bfloat162_rn(q[4 * it + 2], q[4 * it + 3]);
            *reinterpret_cast<uint2*>(o2 + (long long)it * 8 * e.ld_out2) =
                make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
          }
        } else {
          float* o2 = e.out2 + row * e.ld_out2 + col;
#pragma unroll
          for (int it = 0; it < 4; ++it)
            *reinterpret_cast<float4*>(o2 + (long long)it * 8 * e.ld_out2) = make_float4(q[4 * it], q[4 * it + 1], q[4 * it + 2], q[4 * it + 3]);
        }
      } else if constexpr (EK == EK_REVERSE) {
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          float ad[4] = {rf[it].x, rf[it].y, rf[it].z, rf[it].w};
          if (e.aux_add_h) unpack_bf16x4(make_uint2(__float_as_uint(rf[it].x), __float_as_uint(rf[it].y)), ad);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int i = 4 * it + k;
            const float ee = mufu_ex2(u[i] * kk);
            w[i] = fmaf(x[i], fmaf(-sc, ee, sc), ad[k]);  // x * (1 - e) * scale + aux_add
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float ee = mufu_ex2(u[i] * kk);
          w[i] = x[i] * fmaf(-sc, ee, sc);
        }
      }
    }
    if constexpr (EK == EK_RELU_BWD) {
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        float f[4];
        unpack_bf16x4(ru0[it], f);
#pragma unroll
        for (int k = 0; k < 4; ++k) w[4 * it + k] = f[k] > 0.0f ? x[4 * it + k] * e.scale : 0.0f;
      }
    }
    if constexpr (EK == EK_REVERSE || EK == EK_RELU_BWD) {
      if (e.colsum) line_colsum_add(w, lane, cs_tile, e.colsum + nc);
    }
    if constexpr (EK == EK_TANGENT) {
      if (e.out_f32) {
        float* of = e.out_f32 + row * e.ld_f32 + col;
#pragma unroll
        for (int it = 0; it < 4; ++it)
          *reinterpret_cast<float4*>(of + (long long)it * 8 * e.ld_f32) = make_float4(w[4 * it], w[4 * it + 1], w[4 * it + 2], w[4 * it + 3]);
      }
    }
    for (int pl = 0; pl < e.n_planes; ++pl) {
      uint32_t pk[8];
      if (pl + 1 < e.n_planes) {
        split_plane<16>(w, pk);                            // rounded plane, residual stays in w
      } else {
#pragma unroll
        for (int t = 0; t < 8; ++t) {                      // last plane: no residual needed
          const __nv_bfloat162 h = __floats2bfloat162_rn(w[2 * t], w[2 * t + 1]);
          pk[t] = *reinterpret_cast<const uint32_t*>(&h);
        }
      }
      bf16* dp = e.out_pl.plane(pl) + row * e.out_pl.ld + col;
#pragma unroll
      for (int it = 0; it < 4; ++it) *reinterpret_cast<uint2*>(dp + (long long)it * 8 * e.out_pl.ld) = make_uint2(pk[2 * it], pk[2 * it + 1]);
    }
  }
}

}  // namespace nrw
