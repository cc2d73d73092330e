// Helpers shared by every geometry estimator (geo_api.cu, pose_api.cu, lo_pose_api.cu, lo_hf_api.cu, pnp_api.cu), all
// compiled with -fmad=false.  include/geometry_b200.h states each step; oracle/geometry_oracle.py and
// oracle/pose_oracle.py restate them in numpy.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

#include "../../include/geometry_b200.h"
#include "lg_internal.h"

namespace {

constexpr int RED = 256;  // partial sums of the fixed summation order (header step 2)

// Score CTAs per pair of every estimator's score kernel: enough to cover the SMs twice, with at least 128 points each
int geo_score_splits(int B, int M) {
  const int want = (2 * lg_num_sms() + B - 1) / B;
  int splits = (M + 127) / 128;
  if (splits > want) splits = want;
  if (splits < 1) splits = 1;
  return splits;
}

// A keypoint with a non-finite coordinate makes its match invalid at compaction (header steps 1, P1 and A1)
__device__ __forceinline__ bool finite2(float2 p) { return isfinite(p.x) && isfinite(p.y); }

__device__ __forceinline__ unsigned geo_mix(unsigned x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// Up to s distinct indices of hypothesis h of a pair with n points (header step 3); returns how many were drawn.
// geo_hypothesis keeps its own copy of this loop: calling this one there changes its register allocation.
__device__ __forceinline__ int geo_sample(unsigned seed, unsigned h, int n, int s, int* id) {
  int k = 0;
  const unsigned x = geo_mix(geo_mix(seed ^ 0x9e3779b9u) ^ h);
  for (unsigned t = 0; t < GEO_MAX_DRAWS && k < s; ++t) {
    const int j = (int)(((unsigned long long)geo_mix(x + t) * (unsigned)n) >> 32);
    bool dup = false;
    for (int q = 0; q < k; ++q) dup = dup || id[q] == j;
    if (!dup) id[k++] = j;
  }
  return k;
}

// The fixed-order sum of the block's RED partials (threads tid < RED hold one each).  Every thread of the block calls
// it; every thread gets the sum.
__device__ double tree_sum(double p, double* red, int tid) {
  if (tid < RED) red[tid] = p;
  __syncthreads();
  for (int h = RED / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] = red[tid] + red[tid + h];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ double sgn1(double z) { return z >= 0.0 ? 1.0 : -1.0; }

// GEO_SVD_SWEEPS sweeps of one-sided Jacobi on the columns of a row-major 3x3 A, accumulating the rotations in V
// (header step 4)
__device__ __forceinline__ void jacobi_columns3(double* A, double* V) {
  const int PQ[3][2] = {{0, 1}, {0, 2}, {1, 2}};
  for (int sweep = 0; sweep < GEO_SVD_SWEEPS; ++sweep)
    for (int r = 0; r < 3; ++r) {
      const int p = PQ[r][0], q = PQ[r][1];
      double al = 0.0, be = 0.0, ga = 0.0;
      for (int i = 0; i < 3; ++i) {
        al = al + A[i * 3 + p] * A[i * 3 + p];
        be = be + A[i * 3 + q] * A[i * 3 + q];
        ga = ga + A[i * 3 + p] * A[i * 3 + q];
      }
      if (fabs(ga) <= 1e-15 * sqrt(al * be)) continue;
      const double z = (be - al) / (2.0 * ga);
      const double t = sgn1(z) / (fabs(z) + sqrt(1.0 + z * z));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
      for (int i = 0; i < 3; ++i) {
        const double ap = A[i * 3 + p], aq = A[i * 3 + q];
        A[i * 3 + p] = c * ap - s * aq;
        A[i * 3 + q] = s * ap + c * aq;
        const double vp = V[i * 3 + p], vq = V[i * 3 + q];
        V[i * 3 + p] = c * vp - s * vq;
        V[i * 3 + q] = s * vp + c * vq;
      }
    }
}

// OpenCV's RANSACUpdateNumIters, with pow(1 - ep, s) as repeated products (header step 6)
__device__ int update_num_iters(double p, double ep, int s, int max_iters) {
  if (p >= 1.0) return max_iters;
  p = fmin(fmax(p, 0.0), 1.0);
  ep = fmin(fmax(ep, 0.0), 1.0);
  double num = fmax(1.0 - p, DBL_MIN);
  const double q = 1.0 - ep;
  double pw = q;
  for (int i = 1; i < s; ++i) pw = pw * q;
  double denom = 1.0 - pw;
  if (denom < DBL_MIN) return 0;
  num = log(num);
  denom = log(denom);
  return (denom >= 0.0 || -num >= max_iters * (-denom)) ? max_iters : __double2int_rn(num / denom);
}

// Smallest-eigenvalue eigenvector of a symmetric NxN by cyclic Jacobi (header step 7)
template <int N>
__device__ void smallest_eigvec(double (*A)[N], double* out) {
  double V[N][N];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < GEO_EIG_SWEEPS; ++sweep)
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double z = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = sgn1(z) / (fabs(z) + sqrt(z * z + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  int m = 0;
  for (int k = 1; k < N; ++k)
    if (A[k][k] < A[m][m]) m = k;
  for (int k = 0; k < N; ++k) out[k] = V[k][m];
}

}  // namespace
