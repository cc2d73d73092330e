// The LO-RANSAC pieces shared by the relative pose (lo_pose_api.cu, header steps L3 and L7), the homography
// (lo_homography_api.cu, LH3 and LH7) and the fundamental matrix (lo_fundamental_api.cu, LF3 and LF7), all compiled
// with -fmad=false: the packed MSAC score term and the fixed-order sums of the Levenberg-Marquardt terms.
#pragma once
#include <cuda_runtime.h>

#include "geo_common.cuh"

namespace {

constexpr unsigned long long LO_COUNT_ONE = 1ull << 40;  // a score sum's count field (header GEO_LO_MAX_MATCHES)
constexpr unsigned long long LO_SCORE_MASK = LO_COUNT_ONE - 1;

// L3's per-point term of one fp32 error, with the count in bit 40.  A non-finite error is an outlier.  An inlier's
// product is clamped to GEO_LO_QSCALE, so a subnormal thr2 (w = +inf) stays defined, and e == 0 scores 0 (0 * inf).
__device__ __forceinline__ unsigned long long lo_term(float e, float thr2, float w) {
  if (!(e < thr2)) return GEO_LO_QSCALE;
  return LO_COUNT_ONE + (e == 0.f ? 0u : (unsigned)fminf(e * w, (float)GEO_LO_QSCALE));
}

// The fixed-order sums (header step 2) of T terms at once, through red [T][RED]; every thread of the CTA calls it
template <int T>
__device__ void lo_tree_sums(const double* acc, double (*red)[RED], double* out, int tid) {
  for (int i = 0; i < T; ++i) red[i][tid] = acc[i];
  __syncthreads();
  for (int h = RED / 2; h > 0; h >>= 1) {
    if (tid < h)
      for (int i = 0; i < T; ++i) red[i][tid] = red[i][tid] + red[i][tid + h];
    __syncthreads();
  }
  if (tid < T) out[tid] = red[tid][0];
  __syncthreads();
}

}  // namespace
