// The per-pixel camera ray of the Phototourism pipeline (datasets/ray_utils.py::get_ray_directions + get_rays), shared by
// the ray-cache pass (raygen.cu) and the ROI view selection (viewsel.cu) so that both follow one fp32 rule:
//   i = (float)c, j = (float)r exactly; dx = (i - cx) / fx, ndy = -((j - cy) / fy);
//   d_k = (dx*M[k][0] + ndy*M[k][1]) + (-M[k][2]) with M = c2w[:, :3] (fp32, row-major); origin o_k = c2w[k][3];
//   |d| = sqrt((d_0*d_0 + d_1*d_1) + d_2*d_2), then d_k / |d|.
// Every step is one fp32 _rn operation, no contraction.
#pragma once
#include "../../include/nrw_math.h"
#include "common.cuh"

namespace nrw {

// ray of pixel (r, c): writes the origin o and the unit direction d, returns |d| before the normalisation
__device__ __forceinline__ float pixel_ray(const float* c2w, float fx, float fy, float cx, float cy, int r, int c, float o[3],
                                           float d[3]) {
  const float dx = NRW_DIV(NRW_SUB((float)c, cx), fx);
  const float ndy = -NRW_DIV(NRW_SUB((float)r, cy), fy);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    d[k] = NRW_ADD(NRW_ADD(NRW_MUL(dx, c2w[4 * k]), NRW_MUL(ndy, c2w[4 * k + 1])), -c2w[4 * k + 2]);
    o[k] = c2w[4 * k + 3];
  }
  const float nrm = NRW_SQRT(NRW_ADD(NRW_ADD(NRW_MUL(d[0], d[0]), NRW_MUL(d[1], d[1])), NRW_MUL(d[2], d[2])));
#pragma unroll
  for (int k = 0; k < 3; ++k) d[k] = NRW_DIV(d[k], nrm);
  return nrm;
}

}  // namespace nrw
