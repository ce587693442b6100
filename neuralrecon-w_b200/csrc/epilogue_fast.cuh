// Compile-time specialised epilogues of the tensor-core GEMM for the eight layer kinds that make up > 95 % of a
// training step.  Same arithmetic, in the same order, as the runtime-parameterised epi_chunk16 (epilogue_tc.cuh), except
// for the softplus gates of TANGENT and REVERSE, which epi_chunk16 forms with softplus100_d12_from_u (GATE_FWD's gate is
// the same in both, NRW_GATE_K) - the difference is what is NOT executed: ncu's source view of the generic epilogue showed ISETP + BRA + LOP3 + IMAD + LDC
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
  auto rows16 = [&](const void* p, int ld) { return !p || (al16(p) && (ld & 3) == 0); };   // absent, or aligned rows
  if (e.head_w || e.head_partial)
    return (e.head_w && e.head_partial && e.bias && al16(e.bias) && al16(e.head_w) && e.act == ACT_SOFTPLUS100 && e.scale == 1.0f && e.n_planes == 0 &&
            !e.atomic && !e.aux_u.p && !e.rowvec && !e.aux_relu && !e.out_pre && !e.out2 && !e.out_f32 &&
            !e.colsum && !e.aux_add && e.n_store >= (1 << 29)) ? EK_FWD_HEAD : -1;      // -1: unsupported combination
  if (e.atomic || e.n_planes > 3) return EK_GENERIC;
  if (e.n_planes > 0 && (!al16(e.out_pl.p) || (e.out_pl.ld & 3) || (e.out_pl.pstride & 7))) return EK_GENERIC;
  if (e.aux_u.p && (!al16(e.aux_u.p) || (e.aux_u.ld & 3) || (e.aux_u.pstride & 7))) return EK_GENERIC;
  if (!rows16(e.out_pre.p, e.out_pre.ld) || !rows16(e.out2.p, e.out2.ld) || !rows16(e.aux_add.p, e.aux_add.ld) ||
      !rows16(e.aux_q.p, e.aux_q_bcast ? 0 : e.aux_q.ld) || !rows16(e.out_f32, e.ld_f32) || !rows16(e.aux_relu, e.ld_relu) ||
      !al16(e.bias) || !al16(e.colvec))
    return EK_GENERIC;
  const bool gate = e.aux_u.p != nullptr;
  if (gate && e.out_pre && !e.out2 && !e.aux_add && !e.colsum && !e.bias && !e.rowvec && !e.aux_relu && e.n_planes > 0 && !e.out_f32)
    return EK_GATE_FWD;
  if (gate && e.out2 && e.aux_q && !e.out_pre && !e.bias && !e.rowvec && !e.aux_add && !e.colsum && !e.aux_relu &&
      ((e.n_planes > 0) != (e.out_f32 != nullptr)))
    return EK_TANGENT;
  if (gate && e.aux_add && !e.out2 && !e.out_pre && !e.bias && !e.aux_relu && e.n_planes > 0 && !e.out_f32) return EK_REVERSE;
  if (!gate && e.aux_relu && !e.out_pre && !e.out2 && !e.aux_add && !e.bias && e.n_planes > 0 && !e.out_f32 && e.act == ACT_NONE)
    return EK_RELU_BWD;
  if (!gate && e.bias && !e.rowvec && !e.aux_relu && !e.aux_add && !e.out_pre && !e.out2 && !e.out_f32 && !e.colsum && e.n_planes > 0) {
    if (e.act == ACT_SOFTPLUS100) return EK_FWD_SOFTPLUS;
    if (e.act == ACT_RELU) return EK_FWD_RELU;
    if (e.act == ACT_NONE) return EK_FWD_NONE;
  }
  return EK_GENERIC;
}

// Side streams of one specialised chunk in the line layout.  For a chunk pair they are loaded before the kernel's staging
// barrier, so their latency overlaps that barrier and the other chunk's arithmetic.
// The bf16 planes stay packed until they are used (8 registers per 16 values): with a chunk pair's side streams and 96
// accumulators live, that is what keeps the gate kinds within the consumer register budget.
struct FastSide {
  uint2 u[4];    // first gate plane (further planes are loaded in fast_finish, except GATE_FWD's second); RELU_BWD: forward activation
  uint2 u2[4];   // GATE_FWD: the SECOND gate plane (its own exposed round trip was 15 % of the stall samples)
  float s[16];   // TANGENT: aux_q; REVERSE: aux_add
  float4 b;      // FWD_*: bias
};

// row = this lane's first row, col = its first column (line layout of a full chunk)
template <int EK>
__device__ __forceinline__ void fast_side_load(const Epi& e, long long row, int col, FastSide& f) {
  if constexpr (EK == EK_GATE_FWD || EK == EK_TANGENT || EK == EK_REVERSE) {
    tile_load_bf16_raw(e.aux_u.p + row * e.aux_u.ld + col, e.aux_u.ld, f.u);
    if constexpr (EK == EK_GATE_FWD) {
      if (e.aux_u_planes > 1) tile_load_bf16_raw(e.aux_u.plane(1) + row * e.aux_u.ld + col, e.aux_u.ld, f.u2);
    }
  }
  if constexpr (EK == EK_FWD_SOFTPLUS || EK == EK_FWD_RELU || EK == EK_FWD_NONE) f.b = ldg4(e.bias + col);
  if constexpr (EK == EK_TANGENT) {
    if (e.aux_q_bcast) {
      const float4 qb = ldg4(e.aux_q.f32() + col);
#pragma unroll
      for (int it = 0; it < 4; ++it) { f.s[4 * it] = qb.x; f.s[4 * it + 1] = qb.y; f.s[4 * it + 2] = qb.z; f.s[4 * it + 3] = qb.w; }
    } else {
      tile_load(e.aux_q, row, col, f.s);
    }
  }
  if constexpr (EK == EK_REVERSE) tile_load(e.aux_add, row, col, f.s);
  if constexpr (EK == EK_RELU_BWD) tile_load_bf16_raw(e.aux_relu + row * e.ld_relu + col, e.ld_relu, f.u);
}

// arithmetic and stores of one full chunk (x_acc: its accumulators in the line layout) whose side streams are in f
template <int EK>
__device__ __forceinline__ void fast_finish(const Epi& e, const float (&x_acc)[16], long long row, int col, int lane, float* cs_tile,
                                            const FastSide& f) {
  float x[16], w[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) x[i] = x_acc[i];
  if constexpr (EK == EK_FWD_SOFTPLUS || EK == EK_FWD_RELU || EK == EK_FWD_NONE) {
    const float bb[4] = {f.b.x, f.b.y, f.b.z, f.b.w};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float t = x[i] + bb[i & 3];
      if constexpr (EK == EK_FWD_SOFTPLUS) w[i] = softplus100(t) * e.scale;
      else if constexpr (EK == EK_FWD_RELU) w[i] = fmaxf(t, 0.0f) * e.scale;
      else w[i] = t * e.scale;
    }
  }
  if constexpr (EK == EK_REVERSE || EK == EK_RELU_BWD) {
    if (e.rowvec) {   // (one launch per step: loaded here, not with the side streams, to keep registers for those)
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
  if constexpr (EK == EK_GATE_FWD) tile_store(e.out_pre, row, col, x);
  if constexpr (EK == EK_GATE_FWD || EK == EK_TANGENT || EK == EK_REVERSE) {
    // u = sum(planes of the softplus output); e = 2^(K u) with the plane scale folded into K
    float u[16], s[16];
    unpack_bf16(f.u, u);
    if constexpr (EK == EK_GATE_FWD) {
      if (e.aux_u_planes > 1) {
        float u2[16];
        unpack_bf16(f.u2, u2);
#pragma unroll
        for (int i = 0; i < 16; ++i) u[i] += u2[i];
      }
    }
    for (int pl = EK == EK_GATE_FWD ? 2 : 1; pl < e.aux_u_planes; ++pl) {
      float t[16];
      tile_load_bf16(e.aux_u.plane(pl) + row * e.aux_u.ld + col, e.aux_u.ld, t);
#pragma unroll
      for (int i = 0; i < 16; ++i) u[i] += t[i];
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) s[i] = f.s[i];
    const float kk = NRW_GATE_K * e.aux_u_scale, sc = e.scale;
    if constexpr (EK == EK_TANGENT) {
      const float sc100 = 100.0f * sc;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float ee = mufu_ex2(u[i] * kk);
        const float s1 = 1.0f - ee;
        const float xs = x[i] * s1;
        w[i] = xs * sc;                                  // x * softplus'(a) * scale
        s[i] = (xs * s[i]) * (ee * sc100);               // scale * x * q * softplus''(a),  softplus'' = 100 s1 e
      }
      tile_store(e.out2, row, col, s);
    } else if constexpr (EK == EK_REVERSE) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float ee = mufu_ex2(u[i] * kk);
        w[i] = fmaf(x[i], fmaf(-sc, ee, sc), s[i]);      // x * (1 - e) * scale + aux_add
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
    float fw[16];
    unpack_bf16(f.u, fw);
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = fw[i] > 0.0f ? x[i] * e.scale : 0.0f;
  }
  if constexpr (EK == EK_REVERSE || EK == EK_RELU_BWD) {
    if (cs_tile) line_colsum_add(w, lane, cs_tile);
  }
  if constexpr (EK == EK_TANGENT) {
    if (e.out_f32) tile_store_f32(e.out_f32 + row * e.ld_f32 + col, e.ld_f32, w);
  }
  for (int pl = 0; pl < e.n_planes; ++pl) {
    uint32_t pk[8];
    if (pl + 1 < e.n_planes) split_plane<16>(w, pk);   // rounded plane, residual stays in w
    else pack_bf16(w, pk);                             // last plane: no residual needed
    tile_store_bf16(e.out_pl.plane(pl) + row * e.out_pl.ld + col, e.out_pl.ld, pk);
  }
}

// One 32-row x 16-column chunk on its own: x = the accumulators of columns nc..nc+15 of rows m0w..m0w+31 in the line layout.
template <int EK>
__device__ __forceinline__ void epi_fast16(const Epi& e, const float (&x)[16], int m0w, int nc, int M, int N, int lane, float* cs_tile,
                                           float* hacc) {
  if constexpr (EK == EK_GENERIC) {
    epi_chunk16(e, x, m0w, nc, M, N, lane, cs_tile);
  } else if constexpr (EK == EK_FWD_HEAD) {
    // every row of the 32-row group is processed (rows beyond M hold zero-filled operands and are never written); only
    // column-indexed vectors are read, so there is no ragged fallback.  hacc[it] accumulates this lane's rows over the
    // warp's chunks of the tile in a FIXED order (deterministic SDF values).
    const int col = nc + (lane & 3) * 4;
    const float4 b = ldg4(e.bias + col), hw = ldg4(e.head_w + col);
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      float p = softplus100(x[4 * it] + b.x) * hw.x;
      p = fmaf(softplus100(x[4 * it + 1] + b.y), hw.y, p);
      p = fmaf(softplus100(x[4 * it + 2] + b.z), hw.z, p);
      p = fmaf(softplus100(x[4 * it + 3] + b.w), hw.w, p);
      p += __shfl_xor_sync(0xFFFFFFFFu, p, 1);
      p += __shfl_xor_sync(0xFFFFFFFFu, p, 2);
      hacc[it] += p;
    }
  } else {
    // ragged edge tile / column boundary of the stored range: the generic path handles every case
    if (M - m0w < 32 || N - nc < 16 || e.n_store - nc < 16) {
      epi_chunk16(e, x, m0w, nc, M, N, lane, cs_tile);
      return;
    }
    const int col = nc + (lane & 3) * 4;                  // this lane's 4 columns
    const long long row = (long long)m0w + (lane >> 2);   // this lane's first row; rows row + 8*it
    FastSide f;
    fast_side_load<EK>(e, row, col, f);
    fast_finish<EK>(e, x, row, col, lane, cs_tile, f);
  }
}

// ---- the chunk pair of one epilogue round: chunk 0 = columns nc..nc+15, chunk 1 = columns nc+32..nc+47 of the same 32 rows ----
// If pair_full is true (a kind with side streams, and both chunks full: rows, columns and the stored range - the test on
// chunk 1 covers chunk 0's columns too), the kernel calls pair_load once it has staged the round's accumulators: every
// side-stream load of both chunks at once, so their latency overlaps the staging barrier, and epi_pair_chunk finishes
// each chunk from them.  Otherwise epi_pair_chunk runs the per-chunk path: per element exactly what epi_fast16 computes.
// Kinds whose pair fits the consumer register budget (232) without spilling.  GATE_FWD, TANGENT and REVERSE do not (fp32 side
// streams of two chunks next to 96 live accumulators): they load one chunk's side streams at a time.
template <int EK>
constexpr bool pair_kind() {
  return EK == EK_FWD_SOFTPLUS || EK == EK_FWD_RELU || EK == EK_FWD_NONE || EK == EK_RELU_BWD;
}
template <int EK>
__device__ __forceinline__ bool pair_full(const Epi& e, int m0w, int nc, int M, int N) {
  if constexpr (!pair_kind<EK>()) return false;
  else return M - m0w >= 32 && N - (nc + 32) >= 16 && e.n_store - (nc + 32) >= 16;
}
template <int EK>
__device__ __forceinline__ void pair_load(const Epi& e, int m0w, int nc, int lane, FastSide& f0, FastSide& f1) {
  const int col = nc + (lane & 3) * 4;
  const long long row = (long long)m0w + (lane >> 2);
  fast_side_load<EK>(e, row, col, f0);
  fast_side_load<EK>(e, row, col + 32, f1);
}
// chunk at column nc of the pair (nc < N, m0w < M); f: its side streams if `full`
template <int EK>
__device__ __forceinline__ void epi_pair_chunk(const Epi& e, const float (&x)[16], bool full, const FastSide& f, int m0w, int nc, int M,
                                               int N, int lane, float* cs_tile, float* hacc) {
  if constexpr (pair_kind<EK>()) {
    if (full) {   // warp-uniform
      fast_finish<EK>(e, x, (long long)m0w + (lane >> 2), nc + (lane & 3) * 4, lane, cs_tile, f);
      return;
    }
  }
  epi_fast16<EK>(e, x, m0w, nc, M, N, lane, cs_tile, hacc);
}

}  // namespace nrw
