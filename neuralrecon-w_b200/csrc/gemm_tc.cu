// wgmma / TMA GEMM for sm_90a (Hopper) with split-bf16 operand planes and a fused epilogue.
//
//   D[M,N] (fp32, registers) = sum_{(pa,pb) in products(n_planes)}  A_pa[M,K] * B_pb[N,K]^T
//
// * operands are bf16 planes (hi / lo / lo2) of fp32 tensors; n_planes=1 is plain bf16,
//   n_planes=2 issues hi*hi + hi*lo + lo*hi (~16 mantissa bits), n_planes=3 all six
//   products whose weight is >= 2^-16 (~fp32).  All products accumulate into the same fp32
//   register accumulator, so precision is a loop bound, not a different kernel.
// * persistent CTAs (one per SM), warp-specialised ping-pong: warps 0-7 = two consumer warpgroups, warps 8-11 =
//   producer warpgroup (one thread issues the TMA).  A CTA's work items (128 x BN tiles, or tile x K-slice)
//   alternate between the consumer warpgroups: warpgroup wg takes items blockIdx.x + (2 i + wg) gridDim.x and
//   runs the whole tile (two wgmma.m64nBNk16 per k16 step, one per 64-row half: 2 x BN/2 fp32 accumulators).
//   An ordered math barrier hands the tensor cores from one warpgroup's main loop to the other's, so the
//   epilogue of item i runs while the other warpgroup's MMAs of item i+1 do.  setmaxnreg moves registers from
//   the producer warpgroup (40) to the consumers (232).
// * one smem ring of TMA stages (128B swizzle), filled in item order, so the loads of the next k-blocks (and of
//   the next items) overlap the MMAs and the epilogues.  A stage has a single consuming warpgroup.
// * the epilogue stages a warpgroup's accumulators (64 columns of one 64-row half per round) through shared memory into the
//   line layout the chunk epilogues take (epilogue_tc.cuh / epilogue_fast.cuh: two 32-row x 16-column chunks per warp and round).
// * Each instantiation runs one schedule (Sched): K-major ping-pong (data GEMMs), MN-major ping-pong, cooperative weight
//   gradients, or paired launches.  All four share one producer loop and one consumer loop over the CTA's item list (tc_item);
//   a schedule only changes compile-time properties of them (operand layout, item kinds, which warpgroup owns an item).
// * MN-major operands (Sched::MNMAJOR) are consumed "transposed" straight from their natural row-major
//   [rows=K][cols=M|N] layout (MN-major wgmma descriptors) - used for weight gradients
//   dW = dY^T X with split-K over the sample dimension and fp32 atomics in the epilogue.
// * Sched::COOP (one-plane weight gradients with M >= 256, gemm_tc_dw_coop): a work item is a 256 x 128 tile x K-slice that
//   both consumer warpgroups run at the same time, warpgroup wg on rows 128 wg .. +127 (two m64n128 halves), both reading
//   the stage's one B tile.  Per 64-row k-block that moves 48 KB for 4.2 MFLOP instead of 32 KB for 2.1 MFLOP.  No turn
//   barrier: each stage's empty barrier counts all 8 consumer warps.  The epilogue is one fp32 vector reduction
//   (red.global.add.v2.f32) per accumulator pair straight from the fragment: no staging tile and no named barriers, while
//   the producer already loads the next item's k-blocks.
// * Sched::PAIR (gemm_tc_pair): one launch runs a backward layer's data GEMM and its weight gradient together.  Work items are
//   the 128 x 128 tiles of the one-plane K-major data GEMM (epilogue kind EK) and 128 x 128 x K-slice items of the one-plane
//   MN-major dW.  Both fill the same 32 KB stage, so ring, stage count and barriers are those of the ping-pong schedule; the
//   item kind (warp-uniform) selects the tensor maps, the descriptors and the epilogue: data tiles take the staged epilogue,
//   dW items the fragment red.add of Sched::COOP.  The combined list is laid out in rounds of gridDim.x items (round j = the
//   j-th item of every CTA, so warpgroup j & 1 runs it): data and dW rounds alternate while both remain, then the rest follow.
//   So one warpgroup runs a data tile's epilogue while the other runs a dW item's main loop on the tensor cores.  A dW
//   round numbers its items tile-minor over consecutive K-slices: the CTAs of a round share each slice's operand slabs in L2.
//   K-slice rule (host, gemm_tc_pair_k_slices): 128 k-blocks of 64 samples per dW item.  At the tensor-core peak a k-block
//   is about 512 cycles, so 40 k-blocks would match a data tile's epilogue (22-25 k cycles at N = 512) minus its main loop.
//   But both kinds stream 32 KB per k-block from L2 into shared memory, and that stream, not the tensor pipe, bounds a
//   paired launch: longer items mean fewer items, fewer fragment reductions and fewer turn hand-overs.  Measured per C2
//   step: 24, 40, 64 and 128 k-blocks in that order ran faster (DESIGN.md 5.1).
#include <stdlib.h>

#include <mutex>
#include <unordered_map>
#include <vector>
#include <algorithm>
#include <type_traits>
#include <stdio.h>

#include "gemm.h"
#include "epilogue_fast.cuh"

namespace nrw {

static constexpr int BM = 128;
static constexpr int BK = 64;                          // 64 bf16 = 128 B = one swizzle row
static constexpr int RING_BYTES = 192 * 1024;          // TMA stages
static constexpr int MAX_STAGES = 8;
static constexpr int N_CONSUMER_WARPS = 8;             // two ping-pong warpgroups, each owning whole 128-row tiles
static constexpr int N_THREADS = 32 * N_CONSUMER_WARPS + 128;   // + the producer warpgroup
static constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // setmaxnreg split: 128 x 40 + 256 x 232 <= 65536
static constexpr int EPI_COLS = 64;                    // columns per epilogue round; staging rows are unpadded (16-byte slots XOR-swizzled)
static constexpr int EPI_WG_BYTES = 64 * EPI_COLS * 4; // one warpgroup's staging tile [64 rows][64 columns]
static constexpr int CS_BYTES = 1024;                  // column-sum accumulators: 128 columns of the current n-tile per warpgroup
static constexpr int BAR_TURN = 4;                     // named barriers 4 + wg: warpgroup wg's turn at the tensor cores
static_assert(PRODUCER_REGS * 128 + CONSUMER_REGS * 32 * N_CONSUMER_WARPS <= 65536, "register file");
static constexpr int BAR_BYTES = 256;                  // 2 x MAX_STAGES mbarriers
static constexpr int SMEM_BYTES = 1024 + RING_BYTES + BAR_BYTES + 2 * EPI_WG_BYTES + CS_BYTES;
static_assert(SMEM_BYTES <= 232448, "dynamic shared memory limit of sm_90");

// Staging tile: 16-byte slot s of row r is stored at slot s ^ epi_swz(r) of the row.  The XOR permutes the 8 bank groups of a
// 128-byte wavefront: a half-warp's fragment stores (4 consecutive rows 4k..4k+3 x slots 2j, 2j+1: epi_swz / 2 takes 4
// different values) and a quarter-warp's line-layout reads (rows 2k, 2k+1 x slots 4c..4c+3: epi_swz differs in bit 2) hit 8
// different bank groups, so both directions are conflict-free without padding.
__device__ __forceinline__ int epi_swz(int r) { return ((r & 1) << 2) | (r & 2) | ((r >> 2) & 1); }

struct TcParams {
  CUtensorMap tmA[3];
  CUtensorMap tmB[3];
  int M, N, K;
  int n_planes;
  int k_slices;
  int m_tiles, n_tiles;
  Epi epi;
  // Sched::PAIR: the weight gradient, out_f32[dw_M, dw_N] += dw_scale * A2^T B2 (one plane, MN-major, split into dw_k_slices)
  CUtensorMap tmA2, tmB2;
  int dw_M, dw_N, dw_K, dw_k_slices, dw_m_tiles, dw_n_tiles;
  float* dw_out;
  int dw_ld;
  float dw_scale;
  // optional cycle attribution (debug): per CTA 16 counters
  //  [0] producer: waiting for a free stage   [5] kernel cycles
  //  first warp of consumer warpgroup wg, o = 8 wg: [1 + o] waiting for TMA data   [3 + o] waiting for its turn at the
  //  tensor cores   [4 + o] epilogue   [6 + o] tiles (Sched::COOP: both warpgroups count every non-empty item; Sched::PAIR:
  //  data tiles)   [7 + o] Sched::PAIR: dW items
  unsigned long long* prof;
};
#define NRW_PROF_T0(cond) const long long _t0 = (cond) ? clock64() : 0
#define NRW_PROF_ADD(cond, slot) \
  if (cond) atomicAdd(&p.prof[blockIdx.x * 16 + (slot)], (unsigned long long)(clock64() - _t0))

// ---------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// Programmatic dependent launch: a GEMM launched with the stream-serialisation attribute may have its CTAs scheduled while the
// previous kernel of the stream drains, so barrier init and descriptor prefetch overlap the predecessor's tail.  pdl_wait()
// returns once the predecessor has completed and its writes are visible: nothing before it may touch global memory.  Both are
// no-ops in a normally launched kernel.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// named barrier over `n` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// arrive without waiting: the barrier completes once the waiting side's bar.sync threads join
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// per-thread register budget of the executing warpgroup (all its threads execute it)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// generic-proxy shared-memory stores -> visible to the tensor core's (async proxy) reads
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// out[0], out[1] += a, b: one sm_90 vector fp32 reduction (out 8-byte aligned)
__device__ __forceinline__ void red_add_v2(float* out, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(out), "f"(a), "f"(b) : "memory");
}

// wgmma matrix descriptor (sm_90), 128B swizzle:
//   bits [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout = 1 (128B swizzle)
// K-major: SBO = 8 rows * 128 B (LBO unused).  MN-major: LBO = stride between 64-wide MN slabs, SBO = 8 k-rows * 128 B.
__device__ __forceinline__ uint64_t make_gdesc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {   // keeps the accumulator registers in place across the async MMAs
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x BN] (+)= A[64 x 16] * B[BN x 16]^T, bf16 in, fp32 accumulate; TA / TB = 1: MN-major operand
template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate);

template <>
__device__ __forceinline__ void wgmma_bf16<64, 0, 0>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_bf16<64, 1, 1>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
#define NRW_WGMMA_N128(TA, TB)                                                                                                          \
  template <>                                                                                                                           \
  __device__ __forceinline__ void wgmma_bf16<128, TA, TB>(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {              \
    asm volatile(                                                                                                                       \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                                    \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "                                                                        \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "    \
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, " \
        "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, " #TA ", " #TB ";\n}\n"                   \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),     \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),        \
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),        \
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),        \
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])         \
        : "l"(da), "l"(db), "r"(accumulate));                                                                                           \
  }
NRW_WGMMA_N128(0, 0)
NRW_WGMMA_N128(1, 1)
#undef NRW_WGMMA_N128

// out[row][c] += scale * acc for the 128 rows m0 .. m0 + 127 (two m64 halves) of one warpgroup's MN-major weight-gradient
// fragment: one red.global.add.v2.f32 per accumulator pair, masked at the M / N edges.  Fragment of warp wi in half h:
// acc[h][4j + {0,1}] = row 64 h + 16 wi + lane / 4, columns 8 j + 2 (lane % 4) + {0,1}; acc[h][4j + {2,3}] = the same
// columns of row + 8.
template <int BN>
__device__ __forceinline__ void dw_reduce(const float (&acc)[2][BN / 2], float* out, int ld, float scale, int m0, int n0,
                                          int M, int n_lim, int wi, int lane) {
  const int c0 = n0 + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      const int row = m0 + 64 * h + 16 * wi + (lane >> 2) + 8 * r8;
      if (row >= M) continue;
      float* dst = out + (long long)row * ld;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = c0 + 8 * j;
        const float x0 = acc[h][4 * j + 2 * r8] * scale, x1 = acc[h][4 * j + 2 * r8 + 1] * scale;
        if (c + 1 < n_lim) red_add_v2(dst + c, x0, x1);
        else if (c < n_lim) atomicAdd(dst + c, x0);
      }
    }
}

// Schedule of one gemm_tc_kernel instantiation (header comment): K-major or MN-major ping-pong, cooperative weight gradients,
// or a paired data GEMM + weight-gradient launch.  The kernel reads it only through the properties below.
enum class Sched { KMAJOR, MNMAJOR, COOP, PAIR };
// tmA / tmB hold MN-major planes; otherwise K-major ones
constexpr bool mn_operands(Sched s) { return s == Sched::MNMAJOR || s == Sched::COOP; }
// both consumer warpgroups run every item, warpgroup wg on its rows 128 wg .. +127: no turn barrier, and a stage's empty
// barrier counts all 8 consumer warps
constexpr bool shared_items(Sched s) { return s == Sched::COOP; }
constexpr int item_rows(Sched s) { return shared_items(s) ? 2 * BM : BM; }
// item kinds: data tiles (staged epilogue) and weight-gradient items (one MN-major plane, fragment red.add epilogue)
constexpr bool data_items(Sched s) { return s != Sched::COOP; }
constexpr bool dw_items(Sched s) { return s == Sched::COOP || s == Sched::PAIR; }
// both kinds in one launch: the weight gradient's operands are tmA2 / tmB2, its output the dw_* fields
constexpr bool paired(Sched s) { return data_items(s) && dw_items(s); }

// operand layout of an item's k-blocks: K-major planes, MN-major planes, or one MN-major weight-gradient plane
enum class Ops { K, MN, DW };

// One work item of a CTA: output tile origin, k-block range [kb0, kb1) (empty: kb1 <= kb0), and its kind.
struct TcItem { int m0, n0, kb0, kb1; bool dw; };

// item j of this CTA.  Plain launches: item blockIdx.x + j gridDim.x of the slice-minor list.  Paired launches: round j
// (see the header comment); positions past the end of a kind's last round are empty items.
template <int BN, Sched S>
__device__ __forceinline__ TcItem tc_item(const TcParams& p, int j, int kb_total, int kb_per) {
  TcItem it;
  it.dw = !data_items(S);
  if constexpr (paired(S)) {
    const int G = gridDim.x;
    const int n_data = p.m_tiles * p.n_tiles, dw_tiles = p.dw_m_tiles * p.dw_n_tiles, n_dw = dw_tiles * p.dw_k_slices;
    const int rd = (n_data + G - 1) / G, rw = (n_dw + G - 1) / G, ri = min(rd, rw);
    int r;
    if (j < 2 * ri) { it.dw = (j & 1) != 0; r = j >> 1; }
    else { it.dw = rd <= ri; r = j - ri; }
    const int i = r * G + blockIdx.x;
    if (!it.dw) {
      it.n0 = (i % p.n_tiles) * BN; it.m0 = (i / p.n_tiles) * BM;
      it.kb0 = 0; it.kb1 = i < n_data ? kb_total : 0;
    } else {
      const int t = i % dw_tiles, ks = i / dw_tiles;
      const int dw_kb_total = (p.dw_K + BK - 1) / BK, dw_kb_per = (dw_kb_total + p.dw_k_slices - 1) / p.dw_k_slices;
      it.n0 = (t % p.dw_n_tiles) * BN; it.m0 = (t / p.dw_n_tiles) * BM;
      it.kb0 = ks * dw_kb_per; it.kb1 = i < n_dw ? min(dw_kb_total, it.kb0 + dw_kb_per) : 0;
    }
    return it;
  }
  const int item = blockIdx.x + j * gridDim.x;
  const int ks = item % p.k_slices;
  const int t = item / p.k_slices;
  it.n0 = (t % p.n_tiles) * BN; it.m0 = (t / p.n_tiles) * item_rows(S);
  it.kb0 = ks * kb_per; it.kb1 = min(kb_total, it.kb0 + kb_per);
  return it;
}

// product p of the plane expansion -> (a_plane, b_plane); ordered small-to-large magnitude last
//   n_planes==1: (0,0); ==2: (0,1),(1,0),(0,0); ==3: (0,2),(2,0),(1,1),(0,1),(1,0),(0,0)
// With q = n_products-1-p (q=0 is (hi,hi)): a_plane = nibble q of 0x021010, b_plane = nibble q of 0x201100.

// EK: compile-time epilogue kind of the data tiles (epilogue_fast.cuh); MN-major launches use EK_GENERIC.  S: the schedule.
template <int BN, Sched S, int EK>
__global__ void __launch_bounds__(N_THREADS, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
  static_assert(BN == 64 || BN == 128, "wgmma tile width");
  static_assert(data_items(S) || (BN == 128 && EK == EK_GENERIC), "the cooperative schedule is the 256 x 128 weight-gradient tile");
  static_assert(!paired(S) || BN == 128, "paired launches run 128 x 128 items of both kinds");
  constexpr int TM = item_rows(S);              // rows of a work item
  constexpr int A_TILE = TM * BK * 2;
  constexpr int B_TILE = BN * BK * 2;
  constexpr int WG_A = 64 * BK * 2;           // one 64-row half of the A tile (K-major: 64 rows; MN-major: one 64-wide slab)
  extern __shared__ uint8_t smem_raw[];
  // align inside the shared window by OFFSET (an integer round trip of the pointer would turn every staging access
  // into a generic LD/ST instead of LDS/STS)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int P = p.n_planes;
  const int stage_bytes = P * (A_TILE + B_TILE);
  int stages = RING_BYTES / stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RING_BYTES);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + MAX_STAGES);
  float* epi_buf = reinterpret_cast<float*>(smem + RING_BYTES + BAR_BYTES);
  float* cs_buf = reinterpret_cast<float*>(smem + RING_BYTES + BAR_BYTES + 2 * EPI_WG_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long t_kernel0 = clock64();

  if (warp == N_CONSUMER_WARPS && lane == 0) {
    for (int i = 0; i < P; ++i) {
      tma_prefetch_desc(&p.tmA[i]);
      tma_prefetch_desc(&p.tmB[i]);
    }
    if (paired(S)) {
      tma_prefetch_desc(&p.tmA2);
      tma_prefetch_desc(&p.tmB2);
    }
    for (int i = 0; i < MAX_STAGES; ++i) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, shared_items(S) ? 8 : 4);   // the four warps of the stage's consuming warpgroup (or both)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < 256) cs_buf[threadIdx.x] = 0.0f;
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  const int kb_total = (p.K + BK - 1) / BK;
  const int kb_per = (kb_total + p.k_slices - 1) / p.k_slices;
  const int n_items = p.m_tiles * p.n_tiles * p.k_slices;
  const int n_prod = (P == 1) ? 1 : (P == 2 ? 3 : 6);
  int n_j;   // items of this CTA (paired: rounds, empty items included)
  if constexpr (paired(S)) {
    const int G = gridDim.x, n_dw = p.dw_m_tiles * p.dw_n_tiles * p.dw_k_slices;
    n_j = (n_items + G - 1) / G + (n_dw + G - 1) / G;
  } else {
    n_j = (n_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  }

  if (warp >= N_CONSUMER_WARPS) {
    // ===================== TMA producer: every item's k-blocks in item order =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == N_CONSUMER_WARPS && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_j; ++j) {
        const TcItem it = tc_item<BN, S>(p, j, kb_total, kb_per);
        const int n0 = it.n0, m0 = it.m0;
        for (int kb = it.kb0; kb < it.kb1; ++kb) {
          {
            NRW_PROF_T0(p.prof != nullptr);
            mbar_wait(bar_empty + 8 * s, ph ^ 1);
            NRW_PROF_ADD(p.prof != nullptr, 0);
          }
          mbar_arrive_expect_tx(bar_full + 8 * s, stage_bytes);
          const uint32_t sa = smem_u32(smem + s * stage_bytes);
          const uint32_t sb = sa + P * A_TILE;
          if (paired(S) && it.dw) {                    // MN-major weight-gradient k-block: two 64-wide slabs of each operand
#pragma unroll
            for (int sl = 0; sl < 2; ++sl) {
              tma_load_2d(sa + sl * (64 * BK * 2), &p.tmA2, bar_full + 8 * s, m0 + 64 * sl, kb * BK);
              tma_load_2d(sb + sl * (64 * BK * 2), &p.tmB2, bar_full + 8 * s, n0 + 64 * sl, kb * BK);
            }
          } else for (int pl = 0; pl < P; ++pl) {
            if (!mn_operands(S)) {
              tma_load_2d(sa + pl * A_TILE, &p.tmA[pl], bar_full + 8 * s, kb * BK, m0);
              tma_load_2d(sb + pl * B_TILE, &p.tmB[pl], bar_full + 8 * s, kb * BK, n0);
            } else {
#pragma unroll
              for (int sl = 0; sl < TM / 64; ++sl)
                tma_load_2d(sa + pl * A_TILE + sl * (64 * BK * 2), &p.tmA[pl], bar_full + 8 * s,
                            m0 + 64 * sl, kb * BK);
#pragma unroll
              for (int sl = 0; sl < BN / 64; ++sl)
                tma_load_2d(sb + pl * B_TILE + sl * (64 * BK * 2), &p.tmB[pl], bar_full + 8 * s,
                            n0 + 64 * sl, kb * BK);
            }
          }
          if (++s == stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: each warpgroup runs the MMAs and then the epilogue of the items it owns =====================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = warp >> 2, wi = warp & 3;
    const uint32_t smem0 = smem_u32(smem);
    float* stage_tile = epi_buf + wg * (EPI_WG_BYTES / 4);
    const bool use_cs = data_items(S) && p.epi.colsum != nullptr && !p.epi.atomic;
    float* cs_wg = cs_buf + 128 * wg;                        // this warpgroup's column-sum accumulator
    const int ctid = threadIdx.x & 127;
    const bool prof = p.prof != nullptr && wi == 0 && lane == 0;
    const int po = 8 * wg;                                   // this warpgroup's prof slots
    int cs_n0 = -1;   // n-tile the column-sum accumulator currently holds
    int s = 0;        // ring position (stage, phase) of the next k-block, over every item of the CTA
    uint32_t ph = 0;
    // item j of the CTA: every item is walked, owned or not, so that the ring position stays in step with the producer
    for (int j = 0; j < n_j; ++j) {
      const TcItem it = tc_item<BN, S>(p, j, kb_total, kb_per);
      const int n0 = it.n0, m0 = it.m0, kb0 = it.kb0, kb1 = it.kb1;
      const bool dw = it.dw;                                 // warp-uniform; compile-time unless paired
      if (!shared_items(S) && (j & 1) != wg) {               // the other warpgroup's item: skip its stages
        for (int kb = kb0; kb < kb1; ++kb)
          if (++s == stages) { s = 0; ph ^= 1; }
        continue;
      }
      if (use_cs && !dw && n0 != cs_n0) {
        if (cs_n0 >= 0) colsum_flush(cs_wg, p.epi.colsum, cs_n0, min(min(p.N, p.epi.n_store) - cs_n0, BN), ctid, 128, 2 + wg);
        cs_n0 = n0;
      }
      float acc[2][BN / 2];                                  // rows 0-63 and 64-127 of the warpgroup's 128
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.0f;
      // Wait for this warpgroup's turn: the other one has issued every MMA of item j-1.  Besides keeping the tensor cores
      // with one warpgroup at a time, this is what makes the parity waits on the shared ring safe: every full-barrier
      // phase before this item's k-blocks has completed, so a stage cannot be seen one phase early.
      if (!shared_items(S) && j > 0) {
        NRW_PROF_T0(prof);
        named_bar_sync(BAR_TURN + wg, 256);
        NRW_PROF_ADD(prof, 3 + po);
      }
      // One item's k-blocks, from the first wgmma fence to the release of the last stage, for operand layout L: K-major
      // planes, MN-major planes, or one MN-major weight-gradient plane (Ops::DW, whose A slabs start at a_off).  Each item
      // kind's wgmma sequence lies on one path, its own instantiation of this lambda: wgmma variants that share
      // accumulators under a per-k-block branch would make ptxas serialise every wgmma of the kernel.
      auto mma_item = [&](auto layout, uint32_t a_off) {
        constexpr Ops L = decltype(layout)::value;
        constexpr int TR = L == Ops::K ? 0 : 1;                // transpose flag of both wgmma operands
        constexpr uint32_t KSTEP = TR ? (16 * 128) : 32;      // bytes per wgmma K=16
        // K-major: SBO = 8 rows * 128 B; MN-major: LBO = stride between 64-wide MN slabs, SBO = 8 k-rows
        const uint64_t desc_hi = make_gdesc(0, TR ? (64 * BK * 2) : 16, 1024);   // everything but the start address
        int prev_s = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
          {
            NRW_PROF_T0(prof);
            mbar_wait(bar_full + 8 * s, ph);
            NRW_PROF_ADD(prof, 1 + po);
          }
          const uint32_t sa = smem0 + s * stage_bytes;
          const uint32_t sb = smem0 + s * stage_bytes + P * A_TILE;
          wgmma_fence();
          for (int pr = 0; pr < (L == Ops::DW ? 1 : n_prod); ++pr) {
            const int q = 4 * (n_prod - 1 - pr);             // product order of product_planes(), packed lookup
            const uint32_t pa = L == Ops::DW ? 0 : (0x021010u >> q) & 0xFu, pb = L == Ops::DW ? 0 : (0x201100u >> q) & 0xFu;
            const uint64_t da = desc_hi | (uint64_t)(((sa + pa * A_TILE + a_off) & 0x3FFFFu) >> 4);
            const uint64_t db = desc_hi | (uint64_t)(((sb + pb * B_TILE) & 0x3FFFFu) >> 4);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k)
#pragma unroll
              for (int h = 0; h < 2; ++h)                    // 64-row half h: K-major rows at +8 KB, or the next MN-major slab
                wgmma_bf16<BN, TR, TR>(acc[h], da + ((h * WG_A + k * KSTEP) >> 4), db + ((k * KSTEP) >> 4), 1u);
          }
          wgmma_commit();
          acc_fence(acc[0]);
          acc_fence(acc[1]);
          if (prev_s >= 0) {                                  // the previous stage's MMAs have completed: hand it back
            wgmma_wait<1>();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            if (lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
          }
          prev_s = s;
          if (++s == stages) { s = 0; ph ^= 1; }
        }
        // every MMA of this item is issued: the other warpgroup's main loop may start (if the CTA has an item j+1)
        if (!shared_items(S) && j + 1 < n_j) named_bar_arrive(BAR_TURN + (wg ^ 1), 256);
        wgmma_wait<0>();
        acc_fence(acc[0]);
        acc_fence(acc[1]);
        if (prev_s >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
      };
      if (dw) mma_item(std::integral_constant<Ops, Ops::DW>{}, shared_items(S) ? 2 * wg * WG_A : 0);   // shared: A slabs 2 wg, 2 wg + 1
      else mma_item(std::integral_constant<Ops, mn_operands(S) ? Ops::MN : Ops::K>{}, 0);
      // (an empty k-slice accumulates nothing and stores nothing)
      if (kb1 <= kb0) continue;
      NRW_PROF_T0(prof);
      if (prof) atomicAdd(&p.prof[blockIdx.x * 16 + (paired(S) && dw ? 7 : 6) + po], 1ull);
      if (dw) {
        if (paired(S)) dw_reduce<BN>(acc, p.dw_out, p.dw_ld, p.dw_scale, m0, n0, p.dw_M, p.dw_N, wi, lane);
        else dw_reduce<BN>(acc, p.epi.out_f32, p.epi.ld_f32, p.epi.scale, m0 + 128 * wg, n0, p.M, min(p.N, p.epi.n_store), wi, lane);
        NRW_PROF_ADD(prof, 4 + po);
        continue;
      }
      // ---- epilogue, per 64-row half h: 64 columns per round through the warpgroup's staging tile.  Fragment of warp wi:
      // acc[h][4j + {0,1}] = row 64 h + 16 wi + lane / 4, columns 8 j + 2 (lane % 4) + {0,1}; acc[h][4j + {2,3}] = the same columns
      // of row + 8.  After the barrier warp wi reads rows 64 h + 32 (wi & 1) .. +31 and columns 16 (wi >> 1) .. +15 (chunk 0) and
      // 32 + 16 (wi >> 1) .. +15 (chunk 1) of the round's 64 straight in the line layout of the chunk epilogues (lane L: rows
      // L / 4 + 8 it, columns 4 (L % 4) .. +3). ----
      const int r0 = 16 * wi + (lane >> 2), c0 = 2 * (lane & 3);
      const int qq = wi & 1, cc = wi >> 1;
      const int n_rounds = (min(BN, p.N - n0) + EPI_COLS - 1) / EPI_COLS;
      float* st_w = stage_tile + r0 * EPI_COLS + (c0 & 3);          // fragment stores: row r0 (r0 + 8 has the same swizzle)
      const int st_x = (c0 >> 2) ^ epi_swz(r0);                      // slot 2 jj + (c0 >> 2) -> 2 jj ^ st_x
      const float* st_l = stage_tile + (32 * qq + (lane >> 2)) * EPI_COLS;   // line reads: rows + 8 it share the swizzle
      const int ln_x = (lane & 3) ^ epi_swz(lane >> 2);              // slot 4 c + (lane & 3) -> 4 c ^ ln_x
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m0w = m0 + 64 * h + 32 * qq;
        float hacc[4] = {0.0f, 0.0f, 0.0f, 0.0f};   // FWD_HEAD: this lane's rows of the fused SDF-head dot product
#pragma unroll
        for (int rd = 0; rd < BN / EPI_COLS; ++rd) {
          if (rd >= n_rounds) break;                 // warpgroup-uniform
          const int nc = n0 + EPI_COLS * rd + 16 * cc;
          const bool act = nc < p.N && m0w < p.M;    // warp-uniform
          const bool full = act && pair_full<EK>(p.epi, m0w, nc, p.M, p.N);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int jf = 8 * rd + jj;
            float* d = st_w + (((2 * jj) ^ st_x) << 2);
            *reinterpret_cast<float2*>(d) = make_float2(acc[h][4 * jf], acc[h][4 * jf + 1]);
            *reinterpret_cast<float2*>(d + 8 * EPI_COLS) = make_float2(acc[h][4 * jf + 2], acc[h][4 * jf + 3]);
          }
          FastSide f0, f1;                           // issued before the barrier: their latency overlaps its wait
          if (full) pair_load<EK>(p.epi, m0w, nc, lane, f0, f1);
          named_bar_sync(2 + wg, 128);
          if (act) {
            float* cs = use_cs ? cs_wg + EPI_COLS * rd + 16 * cc : nullptr;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              if (c == 1 && nc + 32 >= p.N) break;   // warp-uniform
              float x[16];
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const float4 t = *reinterpret_cast<const float4*>(st_l + it * 8 * EPI_COLS + (((4 * cc + 8 * c) ^ ln_x) << 2));
                x[4 * it] = t.x; x[4 * it + 1] = t.y; x[4 * it + 2] = t.z; x[4 * it + 3] = t.w;
              }
              epi_pair_chunk<EK>(p.epi, x, full, c ? f1 : f0, m0w, nc + 32 * c, p.M, p.N, lane, cs ? cs + 32 * c : nullptr, hacc);
            }
          }
          named_bar_sync(2 + wg, 128);               // every warp has read the staging tile: the next round may overwrite it
        }
        if (EK == EK_FWD_HEAD && (lane & 3) == 0) { // partial[row][slot], slot = n-tile * 2 + column class: plain stores
          const int slot = (n0 / BN) * 2 + cc;
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int row = m0w + it * 8 + (lane >> 2);
            if (row < p.M) p.epi.head_partial[(long long)row * 8 + slot] = hacc[it];
          }
        }
      }
      NRW_PROF_ADD(prof, 4 + po);
    }
    if (use_cs && cs_n0 >= 0) colsum_flush(cs_wg, p.epi.colsum, cs_n0, min(min(p.N, p.epi.n_store) - cs_n0, BN), ctid, 128, 2 + wg);
  }
  __syncthreads();
  if (p.prof && threadIdx.x == 0) atomicAdd(&p.prof[blockIdx.x * 16 + 5], (unsigned long long)(clock64() - t_kernel0));
}

// ---------------------------------------------------------------------------------------
// host side: tensor maps (driver entry point fetched at run time: no link-time libcuda)
// ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  });
  return fn;
}

struct MapKey {
  const void* ptr; long long inner, outer, ld; int box_inner, box_outer;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && ld == o.ld &&
           box_inner == o.box_inner && box_outer == o.box_outer;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h = h * 1000003u ^ (size_t)k.inner; h = h * 1000003u ^ (size_t)k.outer;
    h = h * 1000003u ^ (size_t)k.ld; h = h * 1000003u ^ (size_t)(k.box_inner * 1024 + k.box_outer);
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
static std::mutex g_map_mutex;

// 2-D bf16 tensor map: inner (contiguous) x outer rows, row pitch ld elements, 128B swizzle.
static int make_map(CUtensorMap* out, const bf16* ptr, long long inner, long long outer, long long ld,
                    int box_inner, int box_outer, bool swizzle = true) {
  MapKey key{ptr, inner, outer, ld, swizzle ? box_inner : -box_inner, box_outer};
  {
    std::lock_guard<std::mutex> lk(g_map_mutex);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { *out = it->second; return NRW_OK; }
  }
  EncodeTiledFn enc = get_encode();
  NRW_CHECK(enc != nullptr, NRW_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  NRW_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (ld % 8) == 0, NRW_ERR_ARG,
            "TMA operand must be 16B aligned with ld %% 8 == 0 (ptr=%p ld=%lld)", (const void*)ptr, ld);
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  NRW_CHECK(r == CUDA_SUCCESS, NRW_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%lld outer=%lld ld=%lld",
            (int)r, inner, outer, ld);
  std::lock_guard<std::mutex> lk(g_map_mutex);
  if (g_map_cache.size() > 65536) g_map_cache.clear();
  g_map_cache.emplace(key, *out);
  return NRW_OK;
}

static unsigned long long* g_prof_ptr = nullptr;
void gemm_tc_set_profile_buffer(unsigned long long* p) { g_prof_ptr = p; }
static long long g_tc_launches = 0;
long long gemm_tc_launch_count() { return g_tc_launches; }

// per-device state (cudaFuncSetAttribute and the SM count are per device; a process may touch several GPUs)
static constexpr int MAX_DEV = 64;
static int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < MAX_DEV) ? dev : 0;
}

// Every tensor-core kernel goes through here: grid = min(items, SMs) persistent CTAs, launched with programmatic dependent
// launch (see pdl_wait), so consecutive GEMMs of a layer chain overlap their prologues with the predecessor's tail.  Other
// kernels of the stream are launched normally and serialise as usual.
template <auto Kernel, typename Params>
static int launch_tc(const Params& p, int items, int threads, int smem_bytes, cudaStream_t stream) {
  static bool attr_set[MAX_DEV] = {false};
  static int n_sm[MAX_DEV] = {0};
  const int dev = current_device();
  if (!attr_set[dev]) {
    NRW_CUDA_OK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    attr_set[dev] = true;
  }
  if (!n_sm[dev]) NRW_CUDA_OK(cudaDeviceGetAttribute(&n_sm[dev], cudaDevAttrMultiProcessorCount, dev));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(std::min(items, n_sm[dev]), 1, 1);
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  NRW_CUDA_OK(cudaLaunchKernelEx(&cfg, Kernel, p));
  NRW_LAUNCH_OK();
  ++g_tc_launches;
  return NRW_OK;
}

template <int BN, Sched S, int EK>
static int launch(const TcParams& p, cudaStream_t stream) {
  const int items = p.m_tiles * p.n_tiles * p.k_slices + (paired(S) ? p.dw_m_tiles * p.dw_n_tiles * p.dw_k_slices : 0);
  return launch_tc<gemm_tc_kernel<BN, S, EK>>(p, items, N_THREADS, SMEM_BYTES, stream);
}

static int gemm_tc_impl(const GemmDesc& g, cudaStream_t stream);

// ---- live kernel timing (bench.py roofline): CUDA events around every launch on the launching stream ----
// (a paired launch records its data GEMM's shape and epilogue in M .. epi and its weight gradient's in M2, N2, K2, ks2; flops,
// mma_flops and bytes are the sums of both)
struct TimedLaunch {
  cudaEvent_t e0, e1; double flops; double mma_flops; int M, N, K, P, mn, ks; unsigned epi; double bytes;
  int M2 = 0, N2 = 0, K2 = 0, ks2 = 0;
};
static constexpr int TIMED_MN_PAIR = 3;   // TimedLaunch::mn (the dump's mn_major column) of a paired launch
static std::vector<TimedLaunch> g_timed;
static std::vector<cudaEvent_t> g_event_pool;
static bool g_timing_on = false;
void gemm_tc_timing_enable(bool on) { g_timing_on = on; }
static cudaEvent_t get_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
// sums (and clears) the recorded launches: total kernel ms, algorithmic FLOP (2MNK), MMA FLOP (x products), count
int gemm_tc_timing_read(double* ms, double* flops, double* mma_flops, long long* launches, double* bytes) {
  double t = 0, f = 0, mf = 0, by = 0;
  // tuning: NRW_GEMM_TIMING_DUMP=<path> appends one CSV row per launch: M,N,K,planes,mn_major,k_slices,epilogue bits,
  // algorithmic bytes,ms   (bits: 1 out_pre 2 out_f32 4 out2 8 planes 16 gate (aux_u) 32 aux_q 64 aux_add 128 aux_relu 256 atomic 512 colsum)
  // A paired launch (mn_major 3) appends its weight gradient's M,N,K,k_slices; bytes and ms cover both GEMMs.
  FILE* dump = getenv("NRW_GEMM_TIMING_DUMP") ? fopen(getenv("NRW_GEMM_TIMING_DUMP"), "a") : nullptr;
  for (auto& L : g_timed) {
    NRW_CUDA_OK(cudaEventSynchronize(L.e1));
    float dt = 0;
    NRW_CUDA_OK(cudaEventElapsedTime(&dt, L.e0, L.e1));
    t += dt; f += L.flops; mf += L.mma_flops; by += L.bytes;
    g_event_pool.push_back(L.e0); g_event_pool.push_back(L.e1);
    if (dump && L.mn == TIMED_MN_PAIR)
      fprintf(dump, "%d,%d,%d,%d,%d,%d,%u,%.0f,%.4f,%d,%d,%d,%d\n", L.M, L.N, L.K, L.P, L.mn, L.ks, L.epi, L.bytes, dt, L.M2, L.N2,
              L.K2, L.ks2);
    else if (dump) fprintf(dump, "%d,%d,%d,%d,%d,%d,%u,%.0f,%.4f\n", L.M, L.N, L.K, L.P, L.mn, L.ks, L.epi, L.bytes, dt);
  }
  if (dump) fclose(dump);
  *ms = t; *flops = f; *mma_flops = mf; *launches = (long long)g_timed.size();
  if (bytes) *bytes = by;
  g_timed.clear();
  return NRW_OK;
}

// Runs launch(); with timing on, between two events on `stream`, recorded with the TimedLaunch that describe() returns.
template <typename Describe, typename Launch>
static int timed(cudaStream_t stream, Describe describe, Launch launch) {
  if (!g_timing_on) return launch();
  TimedLaunch L = describe();
  L.e0 = get_event(); L.e1 = get_event();
  NRW_CUDA_OK(cudaEventRecord(L.e0, stream));
  const int rc = launch();
  NRW_CUDA_OK(cudaEventRecord(L.e1, stream));
  g_timed.push_back(L);
  return rc;
}

// adds g's algorithmic FLOP, MMA FLOP and bytes to L
static void account(const GemmDesc& g, TimedLaunch& L) {
  L.flops += 2.0 * g.M * g.N * g.K;
  L.mma_flops += 2.0 * g.M * g.N * g.K * n_products(g.n_planes);
  const Epi& e = g.epi;
  const int q_bytes = e.aux_q_bcast ? 0 : e.aux_q.elem_bytes();   // a broadcast row vector is no stream
  const double mn = (double)g.M * (double)std::min(g.N, e.n_store);
  L.bytes += 2.0 * g.n_planes * ((double)g.M * g.K + (double)g.N * g.K) + (double)e.out_pre.elem_bytes() * g.M * g.N +
             mn * (4.0 * (e.out_f32 ? 1 : 0) + e.out2.elem_bytes() + q_bytes + e.aux_add.elem_bytes() + 2.0 * e.n_planes +
                   (e.aux_relu ? 2.0 : 0.0) + (e.aux_u.p ? 2.0 * e.aux_u_planes : 0.0));
}
static TimedLaunch describe(const GemmDesc& g) {
  TimedLaunch L;
  L.flops = L.mma_flops = L.bytes = 0.0;
  account(g, L);
  L.M = g.M; L.N = g.N; L.K = g.K; L.P = g.n_planes; L.mn = g.mn_major; L.ks = g.k_slices;
  const Epi& e = g.epi;
  const int q_bytes = e.aux_q_bcast ? 0 : e.aux_q.elem_bytes();
  L.epi = (e.out_pre ? 1u : 0u) | (e.out_f32 ? 2u : 0u) | (e.out2 ? 4u : 0u) | (e.n_planes ? 8u : 0u) | (e.aux_u.p ? 16u : 0u) |
          (q_bytes ? 32u : 0u) | (e.aux_add ? 64u : 0u) | (e.aux_relu ? 128u : 0u) | (e.atomic ? 256u : 0u) | (e.colsum ? 512u : 0u);
  return L;
}

int gemm_tc(const GemmDesc& g, cudaStream_t stream) {
  return timed(stream, [&] { return describe(g); }, [&] { return gemm_tc_impl(g, stream); });
}

// tensor maps of operand plane pl of g for tiles bn columns wide: K-major rows in boxes of BK x rows, or MN-major 64-wide
// slabs of BK k-rows
static int operand_maps(const GemmDesc& g, int pl, int bn, CUtensorMap* a, CUtensorMap* b) {
  if (!g.mn_major) {
    NRW_CHECK(g.K % BK == 0, NRW_ERR_ARG, "gemm_tc: K=%d must be a multiple of %d (pad the operand)", g.K, BK);
    NRW_TRY(make_map(a, g.A.plane(pl), g.K, g.M, g.A.ld, BK, BM));
    return make_map(b, g.B.plane(pl), g.K, g.N, g.B.ld, BK, bn);
  }
  NRW_TRY(make_map(a, g.A.plane(pl), g.M, g.K, g.A.ld, 64, BK));
  return make_map(b, g.B.plane(pl), g.N, g.K, g.B.ld, 64, BK);
}

// launch parameters of g on items of item_rows x bn
static int tc_params(const GemmDesc& g, int item_rows, int bn, TcParams& p) {
  memset(&p, 0, sizeof(p));
  p.M = g.M; p.N = g.N; p.K = g.K; p.n_planes = g.n_planes; p.k_slices = g.k_slices;
  p.m_tiles = cdiv(g.M, item_rows); p.n_tiles = cdiv(g.N, bn);
  p.epi = g.epi;
  p.prof = g_prof_ptr;
  for (int pl = 0; pl < g.n_planes; ++pl) NRW_TRY(operand_maps(g, pl, bn, &p.tmA[pl], &p.tmB[pl]));
  return NRW_OK;
}

bool gemm_tc_pair_ok(const GemmPair& pr) {
  const GemmDesc &d = pr.data, &w = pr.dw;
  const int ek = d.mn_major ? -1 : pick_epi_kind(d.epi);
  return d.n_planes == 1 && w.n_planes == 1 && d.k_slices == 1 && !d.epi.atomic && gemm_tc_tile_n(d.N) == 128 &&
         (ek == EK_GENERIC || ek == EK_TANGENT || ek == EK_REVERSE || ek == EK_RELU_BWD) && w.N >= 128 && gemm_tc_dw_only(w);
}

static int gemm_tc_pair_impl(const GemmPair& pr, cudaStream_t stream) {
  const GemmDesc &d = pr.data, &w = pr.dw;
  NRW_CHECK(d.M > 0 && d.N > 0 && d.K > 0 && w.M > 0 && w.N > 0 && w.K > 0 && w.k_slices >= 1, NRW_ERR_ARG,
            "gemm_tc_pair: empty problem %d %d %d / %d %d %d", d.M, d.N, d.K, w.M, w.N, w.K);
  NRW_CHECK(gemm_tc_pair_ok(pr), NRW_ERR_ARG, "gemm_tc_pair: the two GEMMs cannot share a launch");
  TcParams p;
  NRW_TRY(tc_params(d, BM, 128, p));
  NRW_TRY(operand_maps(w, 0, 128, &p.tmA2, &p.tmB2));
  p.dw_M = w.M; p.dw_N = std::min(w.N, w.epi.n_store); p.dw_K = w.K; p.dw_k_slices = w.k_slices;
  p.dw_m_tiles = cdiv(w.M, BM); p.dw_n_tiles = cdiv(w.N, 128);
  p.dw_out = w.epi.out_f32; p.dw_ld = w.epi.ld_f32; p.dw_scale = w.epi.scale;
  switch (pick_epi_kind(d.epi)) {
    case EK_TANGENT: return launch<128, Sched::PAIR, EK_TANGENT>(p, stream);
    case EK_REVERSE: return launch<128, Sched::PAIR, EK_REVERSE>(p, stream);
    case EK_RELU_BWD: return launch<128, Sched::PAIR, EK_RELU_BWD>(p, stream);
    default: return launch<128, Sched::PAIR, EK_GENERIC>(p, stream);
  }
}

int gemm_tc_pair(const GemmPair& pr, cudaStream_t stream) {
  return timed(
      stream,
      [&] {
        TimedLaunch L = describe(pr.data);
        account(pr.dw, L);
        L.mn = TIMED_MN_PAIR;
        L.M2 = pr.dw.M; L.N2 = pr.dw.N; L.K2 = pr.dw.K; L.ks2 = pr.dw.k_slices;
        return L;
      },
      [&] { return gemm_tc_pair_impl(pr, stream); });
}

static int gemm_tc_impl(const GemmDesc& g, cudaStream_t stream) {
  NRW_CHECK(g.M > 0 && g.N > 0 && g.K > 0, NRW_ERR_ARG, "gemm_tc: empty problem %d %d %d", g.M, g.N, g.K);
  NRW_CHECK(g.n_planes >= 1 && g.n_planes <= 3, NRW_ERR_ARG, "gemm_tc: n_planes=%d", g.n_planes);
  NRW_CHECK(g.k_slices == 1 || g.epi.atomic, NRW_ERR_ARG, "gemm_tc: split-K needs an atomic epilogue");
  // 128 x 128 tiles (one warpgroup, two m64n128 halves): with two operand planes that is 64 KB per k-block and 3 TMA stages
  const int BN = gemm_tc_tile_n(g.N);
  TcParams p;
  NRW_TRY(tc_params(g, gemm_tc_tile_m(g), BN, p));
  const int ek = g.mn_major ? EK_GENERIC : pick_epi_kind(g.epi);
  NRW_CHECK(ek >= 0 && (ek != EK_FWD_HEAD || g.N == 512), NRW_ERR_ARG,
            "gemm_tc: the fused SDF-head epilogue needs N = 512, bias + softplus and no other output");
  if (gemm_tc_dw_coop(g)) return launch<128, Sched::COOP, EK_GENERIC>(p, stream);
  if (g.mn_major)
    return BN == 64 ? launch<64, Sched::MNMAJOR, EK_GENERIC>(p, stream) : launch<128, Sched::MNMAJOR, EK_GENERIC>(p, stream);
  if (BN == 64) return launch<64, Sched::KMAJOR, EK_GENERIC>(p, stream);
  switch (ek) {
    case EK_FWD_SOFTPLUS: return launch<128, Sched::KMAJOR, EK_FWD_SOFTPLUS>(p, stream);
    case EK_FWD_RELU: return launch<128, Sched::KMAJOR, EK_FWD_RELU>(p, stream);
    case EK_FWD_NONE: return launch<128, Sched::KMAJOR, EK_FWD_NONE>(p, stream);
    case EK_FWD_HEAD: return launch<128, Sched::KMAJOR, EK_FWD_HEAD>(p, stream);
    case EK_GATE_FWD: return launch<128, Sched::KMAJOR, EK_GATE_FWD>(p, stream);
    case EK_TANGENT: return launch<128, Sched::KMAJOR, EK_TANGENT>(p, stream);
    case EK_REVERSE: return launch<128, Sched::KMAJOR, EK_REVERSE>(p, stream);
    case EK_RELU_BWD: return launch<128, Sched::KMAJOR, EK_RELU_BWD>(p, stream);
    default: return launch<128, Sched::KMAJOR, EK_GENERIC>(p, stream);
  }
}


// =======================================================================================
// Fused forward-only SDF chain (sampler queries, NeuconWRenderer.sdf, the 512^3 grid of config 5):
//   positional encoding -> 8 x (512-wide layer, bias, softplus, [skip concat]) -> sdf head, ONE persistent kernel.
//   models/neuconw.py:263-279 (SDFNetwork.forward) + :281-282 (sdf): the reference runs 9 Linear + 8 Softplus + cat per chunk.
//
//   A CTA owns 64 sample rows.  The two bf16 planes of the 64 x 512 activation tile live in shared memory (128 KB) in exactly
//   the K-major 128B-swizzled layout the next layer's wgmma reads.  Four consumer warpgroups each compute 128 of the 512 output
//   columns (two m64n64 register accumulators) over all k-blocks, and streams its own weights from L2 through a private 3-stage
//   TMA ring (one stage = one 64-wide k-block of 64 weight rows, one plane: 8 KB): one thread of the warpgroup refills a stage
//   as soon as the warpgroup's MMAs on it have completed, two stages ahead, across layer and tile boundaries.  Private rings keep
//   every stage with a single consumer (no empty barriers, no producer warp: 512 threads leave 128 registers per thread).  Per k-block and 64-column half
//   the lo-plane weights come first - product (hi, lo) - then the hi plane - (lo, hi), (hi, hi): the product order of the
//   per-layer kernels.  Once every warpgroup has finished a layer's MMAs (named barrier) the epilogues overwrite the input
//   activations IN PLACE with the new ones.  HBM sees 12 bytes per sample in and 4 bytes out.  Results agree with the
//   per-layer chain to fp32 accumulation order and are run-to-run bit-identical (fixed-order head reduction).
// =======================================================================================
static constexpr int FZ_ROWS = 64;                         // rows per CTA
static constexpr int FZ_APLANE = FZ_ROWS * 512 * 2;        // one bf16 plane of the activation tile: 8 k-blocks of [64 x 64]
static constexpr int FZ_A = 2 * FZ_APLANE;
static constexpr int FZ_WG = 4;                            // consumer warpgroups, 128 output columns each
static constexpr int FZ_WSTAGE = 64 * BK * 2;              // 64 weight rows of one k-block, one plane
static constexpr int FZ_NST = 3;                           // stages per warpgroup ring
static constexpr int FZ_BAR = FZ_A + FZ_WG * FZ_NST * FZ_WSTAGE;
static constexpr int FZ_SMEM = 1024 + FZ_BAR + 256;
static constexpr int FZ_THREADS = 128 * FZ_WG;
static constexpr int FZ_POS_PER_TILE = 4 * (1 + 7 * 8);    // ring positions of one tile: 4 stages per k-block, 1 + 7 x 8 k-blocks
static_assert(FZ_SMEM <= 232448, "dynamic shared memory limit of sm_90");

struct SdfFusedParams {
  CUtensorMap tmW[8][2];     // layer l, plane p: [512 n-rows] x [Kp] bf16, box {64 k, 64 n}, 128B swizzle
  const float* bias[8];
  const float* head_w;       // lin8 row 0 (512)
  const float* head_b;       // its bias
  const float* pts;          // [M, 3]
  float* sdf;                // [M]
  int M, n_tiles;            // n_tiles counts 64-row tiles
};

// feature f (0..38) of the 6-frequency positional encoding of x[3]: [x, sin(2^k x), cos(2^k x)]_k, as csrc/embed.cu lays it out
__device__ __forceinline__ float pe6_feature(const float (&x)[3], int f) {
  if (f < 3) return x[f];
  const int k = (f - 3) / 6, wi = (f - 3) % 6, c = wi % 3;
  float sn, cs;
  sincosf(x[c] * (float)(1 << k), &sn, &cs);
  return wi < 3 ? sn : cs;
}

__global__ void __launch_bounds__(FZ_THREADS, 1) sdf_fused_kernel(const __grid_constant__ SdfFusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FZ_BAR);
  const uint32_t w_full = smem_u32(bars);        // w_full[g * FZ_NST + s]: stage s of warpgroup g's ring
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem0 = smem_u32(smem);
  const int g = warp >> 2, wi = warp & 3, et = threadIdx.x;
  const bool loader = wi == 0 && lane == 0;      // issues this warpgroup's weight loads

  if (et == 0) {
    for (int l = 0; l < 8; ++l) { tma_prefetch_desc(&p.tmW[l][0]); tma_prefetch_desc(&p.tmW[l][1]); }
    for (int i = 0; i < FZ_WG * FZ_NST; ++i) mbar_init(w_full + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  // ring position pos of this warpgroup (tile, layer, k-block kb, u = 2 h + (hi-plane weights)) -> TMA load into stage pos % FZ_NST
  auto load = [&](int pos) {
    const int tile = blockIdx.x + (pos / FZ_POS_PER_TILE) * gridDim.x;
    if (tile >= p.n_tiles) return;
    const int q = pos % FZ_POS_PER_TILE;
    const int l = q < 4 ? 0 : 1 + (q - 4) / 32, r = q < 4 ? q : (q - 4) % 32;
    const int kb = r >> 2, u = r & 3;
    const uint32_t st = g * FZ_NST + pos % FZ_NST;
    mbar_arrive_expect_tx(w_full + 8 * st, FZ_WSTAGE);
    tma_load_2d(smem0 + FZ_A + st * FZ_WSTAGE, &p.tmW[l][(u & 1) ? 0 : 1], w_full + 8 * st, kb * BK, 128 * g + 64 * (u >> 1));
  };
  if (loader)
    for (int i = 0; i < FZ_NST; ++i) load(i);

  {
    // ===================== warpgroup g: output columns 128 g .. 128 g + 127 of every layer =====================
    const int r0 = 16 * wi + (lane >> 2), c0 = 2 * (lane & 3);   // fragment rows r0, r0 + 8; columns 8 j + c0 + {0, 1}
    const uint64_t desc_hi = make_gdesc(0, 16, 1024);
    float* part = reinterpret_cast<float*>(smem);                 // head partials [64 rows][4], over k-block 0 once layer 7 has read it
    int pos = 0;                                                  // ring position consumed next
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
      const int m0 = tile * FZ_ROWS;
      // ---- layer-0 input: positional encoding of this CTA's 64 points, written as the k-block-0 tiles of both planes ----
      *reinterpret_cast<uint4*>(smem + et * 16) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(smem + FZ_APLANE + et * 16) = make_uint4(0, 0, 0, 0);
      named_bar_sync(1, 128 * FZ_WG);
      if (et < 3 * FZ_ROWS) {
        const int r = et / 3, c = et % 3, m = m0 + r;
        const float x = m < p.M ? __ldg(p.pts + (long long)m * 3 + c) : 0.0f;
        auto put = [&](int j, float v) {
          const bf16 hi = __float2bfloat16_rn(v), lo = __float2bfloat16_rn(v - __bfloat162float(hi));
          const int off = r * 128 + (((j >> 3) ^ (r & 7)) << 4) + (j & 7) * 2;
          *reinterpret_cast<bf16*>(smem + off) = hi;
          *reinterpret_cast<bf16*>(smem + FZ_APLANE + off) = lo;
        };
        put(c, x);
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          float sn, cs;
          sincosf(x * (float)(1 << k), &sn, &cs);
          put(3 + 6 * k + c, sn);
          put(3 + 6 * k + 3 + c, cs);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128 * FZ_WG);
      float hsum[2] = {0.0f, 0.0f};
      for (int l = 0; l < 8; ++l) {
        const int nkb = l == 0 ? 1 : 8;
        float acc0[32], acc1[32];                 // columns 128 g + [0, 64) and 128 g + [64, 128)
#pragma unroll
        for (int i = 0; i < 32; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
        // one ring stage: u = 2 h + (hi-plane weights); lo-plane weights carry product (hi, lo), hi-plane ones (lo, hi), (hi, hi)
        auto stage = [&](float (&ah)[32], const uint32_t sa, const int u) {
          const uint32_t st = g * FZ_NST + pos % FZ_NST;
          mbar_wait(w_full + 8 * st, (pos / FZ_NST) & 1);
          const uint64_t db = desc_hi | (uint64_t)(((smem0 + FZ_A + st * FZ_WSTAGE) & 0x3FFFFu) >> 4);
          wgmma_fence();
          if ((u & 1) == 0) {
            const uint64_t da = desc_hi | (uint64_t)((sa & 0x3FFFFu) >> 4);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_bf16<64, 0, 0>(ah, da + 2 * k, db + 2 * k, 1u);
          } else {
#pragma unroll
            for (int pa = 1; pa >= 0; --pa) {
              const uint64_t da = desc_hi | (uint64_t)(((sa + pa * FZ_APLANE) & 0x3FFFFu) >> 4);
#pragma unroll
              for (int k = 0; k < BK / 16; ++k) wgmma_bf16<64, 0, 0>(ah, da + 2 * k, db + 2 * k, 1u);
            }
          }
          wgmma_commit();
          acc_fence(acc0);
          acc_fence(acc1);
          if (pos > 0) {                          // the previous stage's MMAs have completed: refill it, two positions ahead
            wgmma_wait<1>();
            acc_fence(acc0);
            acc_fence(acc1);
            if (loader) load(pos + FZ_NST - 1);
          }
          ++pos;
        };
        for (int kb = 0; kb < nkb; ++kb) {
          const uint32_t sa = smem0 + kb * (FZ_ROWS * BK * 2);
          stage(acc0, sa, 0);
          stage(acc0, sa, 1);
          stage(acc1, sa, 2);
          stage(acc1, sa, 3);
        }
        wgmma_wait<0>();
        acc_fence(acc0);
        acc_fence(acc1);
        named_bar_sync(1, 128 * FZ_WG);           // every warpgroup has read this layer's input: it may be overwritten
        const float* bias = p.bias[l];
        if (l == 7) {                             // sdf head: fixed-order partial dot product with lin8's row 0
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int n = 128 * g + 8 * j + c0;
            const float2 b = __ldg(reinterpret_cast<const float2*>(bias + n));
            const float2 hw = __ldg(reinterpret_cast<const float2*>(p.head_w + n));
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const float* a = j < 8 ? acc0 + 4 * j : acc1 + 4 * (j - 8);
              hsum[rr] = fmaf(softplus100(a[2 * rr] + b.x), hw.x, hsum[rr]);
              hsum[rr] = fmaf(softplus100(a[2 * rr + 1] + b.y), hw.y, hsum[rr]);
            }
          }
          break;
        }
        const float scale = l == 3 ? 0.70710678118654752440f : 1.0f;
        float x[2][3];                            // skip connection: columns 473-511 of layer 4's input = PE(x) / sqrt(2)
        if (l == 3 && g == 3) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int m = m0 + r0 + 8 * rr;
#pragma unroll
            for (int i = 0; i < 3; ++i) x[rr][i] = m < p.M ? __ldg(p.pts + (long long)m * 3 + i) : 0.0f;
          }
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int n = 128 * g + 8 * j + c0;
          const float2 b = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int row = r0 + 8 * rr;
            const float* a = j < 8 ? acc0 + 4 * j : acc1 + 4 * (j - 8);
            float w0 = softplus100(a[2 * rr] + b.x) * scale, w1 = softplus100(a[2 * rr + 1] + b.y) * scale;
            if (l == 3 && n + 1 >= 473) {
              if (n >= 473) w0 = pe6_feature(x[rr], n - 473) * 0.70710678118654752440f;
              w1 = pe6_feature(x[rr], n + 1 - 473) * 0.70710678118654752440f;
            }
            const __nv_bfloat162 hh = __floats2bfloat162_rn(w0, w1);
            const float2 hf = __bfloat1622float2(hh);
            const __nv_bfloat162 ll = __floats2bfloat162_rn(w0 - hf.x, w1 - hf.y);
            const int off = (n >> 6) * (FZ_ROWS * BK * 2) + row * 128 + ((((n & 63) >> 3) ^ (row & 7)) << 4) + (n & 7) * 2;
            *reinterpret_cast<__nv_bfloat162*>(smem + off) = hh;
            *reinterpret_cast<__nv_bfloat162*>(smem + FZ_APLANE + off) = ll;
          }
        }
        fence_proxy_async_smem();                 // generic-proxy stores -> visible to the next layer's wgmma
        named_bar_sync(1, 128 * FZ_WG);
      }
      // ---- sdf = the four warpgroups' partials in a fixed order + bias ----
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        hsum[rr] += __shfl_xor_sync(0xFFFFFFFFu, hsum[rr], 1);
        hsum[rr] += __shfl_xor_sync(0xFFFFFFFFu, hsum[rr], 2);
        if ((lane & 3) == 0) part[(r0 + 8 * rr) * 4 + g] = hsum[rr];
      }
      named_bar_sync(1, 128 * FZ_WG);
      if (et < FZ_ROWS) {
        const float4 a = *reinterpret_cast<const float4*>(part + et * 4);
        const int m = m0 + et;
        if (m < p.M) p.sdf[m] = ((a.x + a.y) + (a.z + a.w)) + __ldg(p.head_b);
      }
      named_bar_sync(1, 128 * FZ_WG);             // the partials are read before the next tile's encoding overwrites them
    }
  }
}

int sdf_fused_forward(const SdfFusedDesc& d, cudaStream_t stream) {
  NRW_CHECK(d.M > 0 && d.pts && d.sdf && d.head_w && d.head_b, NRW_ERR_ARG, "sdf_fused_forward: bad arguments (M=%d)", d.M);
  SdfFusedParams p;
  memset(&p, 0, sizeof(p));
  for (int l = 0; l < 8; ++l) {
    const int K = l == 0 ? 64 : 512;
    NRW_CHECK(d.W[l].p && d.W[l].ld == K && d.bias[l], NRW_ERR_ARG, "sdf_fused_forward: layer %d needs packed [512 x %d] weights (ld=%d)", l, K, d.W[l].ld);
    for (int pl = 0; pl < 2; ++pl) NRW_TRY(make_map(&p.tmW[l][pl], d.W[l].plane(pl), K, 512, d.W[l].ld, BK, 64));
    p.bias[l] = d.bias[l];
  }
  p.head_w = d.head_w; p.head_b = d.head_b; p.pts = d.pts; p.sdf = d.sdf; p.M = d.M;
  p.n_tiles = cdiv(d.M, FZ_ROWS);
  auto describe_fused = [&] {   // bench.py roofline: this launch replaces the 8 per-layer GEMMs of a forward-only chunk
    TimedLaunch L;
    L.flops = 2.0 * d.M * 512.0 * (64.0 + 7.0 * 512.0);
    L.mma_flops = 3.0 * L.flops;
    L.M = d.M; L.N = 512; L.K = 64 + 7 * 512; L.P = 2; L.mn = 0; L.ks = 1; L.epi = 4096u;
    L.bytes = 16.0 * d.M;
    return L;
  };
  return timed(stream, describe_fused, [&] { return launch_tc<sdf_fused_kernel>(p, p.n_tiles, FZ_THREADS, FZ_SMEM, stream); });
}

}  // namespace nrw
