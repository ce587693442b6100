// Parameter table (flat fp32 layout) and packed GEMM-layer descriptors for the fixed
// NeuralRecon-W architecture (SURVEY.md 9.1/9.4; models/neuconw.py:183-259, models/nerf.py:86-154).
#pragma once
#include <vector>

#include "common.cuh"

namespace nrw {

// ---- indices into the parameter table ----------------------------------------------------
enum {
  PI_EMB = 0,
  PI_SDF_BASE = 1,       // v(l)=1+3l, g(l)=2+3l, b(l)=3+3l, l=0..8
  PI_DEAD_XF_W = 28, PI_DEAD_XF_B = 29, PI_VARIANCE = 30,
  PI_COL_BASE = 31,      // v(l)=31+3l, g=32+3l, b=33+3l, l=0..4
  PI_CS0_W = 46, PI_CS0_B = 47, PI_CS1_W = 48, PI_CS1_B = 49, PI_CX_W = 50, PI_CX_B = 51,
  PI_NPTS_BASE = 52,     // w(i)=52+2i, b(i)=53+2i, i=0..7
  PI_NAPP_BASE = 68,     // w(s)=68+2s, b(s)=69+2s, s=0..3
  PI_NVIEWS_W = 76, PI_NVIEWS_B = 77, PI_NF_W = 78, PI_NF_B = 79, PI_NA_W = 80, PI_NA_B = 81,
  PI_NR_W = 82, PI_NR_B = 83,
  PI_COUNT = 84
};
inline int pi_sdf_v(int l) { return PI_SDF_BASE + 3 * l; }
inline int pi_sdf_g(int l) { return PI_SDF_BASE + 3 * l + 1; }
inline int pi_sdf_b(int l) { return PI_SDF_BASE + 3 * l + 2; }
inline int pi_col_v(int l) { return PI_COL_BASE + 3 * l; }
inline int pi_col_g(int l) { return PI_COL_BASE + 3 * l + 1; }
inline int pi_col_b(int l) { return PI_COL_BASE + 3 * l + 2; }

struct ParamInfo {
  std::string name;
  int rows, cols;
  long long offset, numel;
};
std::vector<ParamInfo> build_param_table(int n_vocab, int n_a);

// ---- packed GEMM layers ---------------------------------------------------------------------
enum {
  L_SDF0 = 0,  // .. L_SDF7 = 7
  L_SDF8F = 8,
  L_CX = 9, L_CS0 = 10, L_CS1 = 11,
  L_CL0 = 12,  // .. L_CL3 = 15
  L_N0 = 16,   // .. L_N7 = 23
  L_NF = 24,
  L_NS0 = 25,  // .. L_NS3 = 28
  L_COUNT = 29
};

static constexpr int MAX_KP = 640;
static constexpr int MAX_SRC_COLS = 640;

// One packed layer: effective weight rows [row_off, row_off+n_rows) of the source tensor,
// columns permuted/padded through colmap, stored as bf16 planes W[P][Np][Kp] (K contiguous),
// WT[P][Kp][Np] and fp32 bias[Np].  (POD: a copy lives in device memory for pack/unpack.)
struct PackedLayer {
  long long w_off, g_off, b_off;  // float offsets in the flat param buffer (g_off = -1: no weight norm)
  int src_rows, src_cols;
  int row_off, n_rows;
  int Np, Kp;
  long long W_off, WT_off;        // bf16 element offsets in the packed buffer (plane 0)
  long long bias_off;             // float offset in the packed fp32 area
  long long rnorm_off;            // float offset: 1/||v_row|| per packed row (weight-normed layers)
  long long dW_off, db_off;       // float offsets in the gradient scratch (dWp [Np][Kp], dbp [Np])
  short colmap[MAX_KP];           // packed col -> source col (-1 = zero pad)
  short colinv[MAX_SRC_COLS];     // source col -> packed col
};

// small fp32 heads kept outside the GEMM path
struct Heads {
  long long sdf_w0, sdf_b0;     // [512], [1]    row 0 of sdf lin8 (effective)
  long long cl4_w, cl4_b;       // [3,256], [3]  colour lin4 (effective, weight-normed)
  long long na_w, na_b;         // [256], [1]    nerf alpha_linear
  long long nr_w, nr_b;         // [3,128], [3]  nerf rgb_linear
  long long sdf_rn0, cl4_rn;    // rnorm of the weight-normed head rows: [1], [3]
  // gradient scratch offsets (same shapes)
  long long d_sdf_w0, d_sdf_b0, d_cl4_w, d_cl4_b, d_na_w, d_na_b, d_nr_w, d_nr_b;
};

struct PackedModel {
  PackedLayer layers[L_COUNT];
  Heads heads;
  long long table_bytes;      // device copy of `layers` at the start of the packed buffer
  long long bf16_off_bytes;   // start of the bf16 area (bytes from packed base)
  long long f32_off_bytes;    // start of the fp32 area
  long long total_bytes;
  long long plane_stride[L_COUNT];   // bf16 elements between planes of W (== Np*Kp), same for WT
  long long grad_floats;      // size of the gradient scratch (dWp/dbp/head grads), floats
};
// nerf_app = 0: the background NeRF without appearance codes (nerf.py encode_appearance=False) - L_NS0 packs
// views_linears.0 and L_NS1..L_NS3 hold no rows (same sizes, so the packed layout does not depend on the flag)
PackedModel build_packed_model(const std::vector<ParamInfo>& tab, int n_planes, bool nerf_app);

int pack_weights(const PackedModel& pm, const std::vector<ParamInfo>& tab, int n_planes, const float* params,
                 void* packed_base, cudaStream_t s);
int unpack_grads(const PackedModel& pm, const std::vector<ParamInfo>& tab, const float* params,
                 const void* packed_base, const float* grad_scratch, float* grad_params, cudaStream_t s);
const char* last_error_cstr();

}  // namespace nrw
