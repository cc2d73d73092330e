// The LO-RANSAC pieces shared by the relative pose (lo_pose_api.cu, header steps L3 and L7), the homography and the
// fundamental matrix (lo_hf_api.cu, LH3 and LH7, LF3 and LF7) and the absolute pose (lo_pnp_api.cu, LA3 and LA7), all
// compiled with -fmad=false: the packed MSAC score term, the fixed-order sums of the Levenberg-Marquardt terms, and one
// LM loop and re-score over a model policy.
#pragma once
#include <cuda_runtime.h>

#include "geo_common.cuh"
#include "geo_lm.cuh"

namespace {

constexpr unsigned long long LO_COUNT_ONE = 1ull << 40;  // a score sum's count field (header GEO_LO_MAX_MATCHES)
constexpr unsigned long long LO_SCORE_MASK = LO_COUNT_ONE - 1;

// L3's per-point term of one fp32 error, with the count in bit 40.  A non-finite error is an outlier.  An inlier's
// product is clamped to GEO_LO_QSCALE, so a subnormal thr2 (w = +inf) stays defined, and e == 0 scores 0 (0 * inf).
__device__ __forceinline__ unsigned long long lo_term(float e, float thr2, float w) {
  if (!(e < thr2)) return GEO_LO_QSCALE;
  return LO_COUNT_ONE + (e == 0.f ? 0u : (unsigned)fminf(e * w, (float)GEO_LO_QSCALE));
}

// The fixed-order sums (header step 2) of T terms, G at a time through red [G][RED]; every thread of the CTA calls it
template <int T, int G>
__device__ void lo_tree_sums(const double* acc, double (*red)[RED], double* out, int tid) {
#pragma unroll
  for (int g = 0; g < T; g += G) {
    for (int i = 0; i < G; ++i) red[i][tid] = acc[g + i];
    __syncthreads();
    for (int h = RED / 2; h > 0; h >>= 1) {
      if (tid < h)
        for (int i = 0; i < G; ++i) red[i][tid] = red[i][tid] + red[i][tid + h];
      __syncthreads();
    }
    if (tid < G) out[g + tid] = red[tid][0];
    __syncthreads();
  }
}

// Shared state of one pair's CTA in an LO or final kernel.  Model is the policy of one estimator:
//   DOF, TERMS (J^T J upper triangle, J^T r, truncated cost: DOF (DOF + 1) / 2 + DOF + 1), GROUP (the terms per pass of
//   lo_tree_sums, which keeps red within static shared memory), NP (the length of the parameter vector x) and NF (the
//   length of the pixel model that is scored);
//   Scratch, the model's own shared state;
//   terms(s, P, x, pts, n, thr2, out, tid), the TERMS sums at x (every thread);
//   update(s, x, d, out), x moved by the LM step d (thread 0);
//   pixels(s, P, x, out), x as the scaled pixel model that is rounded to float and scored (thread 0);
//   err(h, pts[k]), the fp32 error of point k against a float model.
// P, the pair's constants, and pts, its points (a pointer, or any type whose pts[k] is one point), pass through the
// LM loop and the re-score to the model unread.
template <class Model>
struct LoShared {
  double red[Model::GROUP][RED];
  double x[Model::NP], cand[Model::NP];  // the model being refined and the LM step's candidate
  double sums[Model::TERMS], csum[Model::TERMS];
  typename Model::Scratch m;
  double px[Model::NF];                  // the scaled pixel model of the last re-scored x
  float fm[Model::NF];                   // a model rounded to float
  unsigned long long key, score;
  int take, step_ok;
};

// steps LM steps from s.x, in place (header steps L7, LH7, LF7, LA7); every thread of the CTA calls it
template <class Model, class Pair, class Points>
__device__ void lo_refine(LoShared<Model>& s, const Pair& P, Points pts, int n, double thr2, int steps, int tid) {
  constexpr int NH = Model::DOF * (Model::DOF + 1) / 2;
  Model::terms(s, P, s.x, pts, n, thr2, s.sums, tid);
  double lam = GEO_LO_LAMBDA0;  // every thread keeps the same schedule
  for (int it = 0; it < steps; ++it) {
    if (tid == 0) {
      double d[Model::DOF];
      s.step_ok = lm_solve<Model::DOF>(s.sums, s.sums + NH, lam, d);
      if (s.step_ok) Model::update(s, s.x, d, s.cand);
    }
    __syncthreads();
    if (!s.step_ok) {
      lam = lam * 10.0;
      __syncthreads();
      continue;
    }
    Model::terms(s, P, s.cand, pts, n, thr2, s.csum, tid);
    const bool better = s.csum[Model::TERMS - 1] < s.sums[Model::TERMS - 1];
    __syncthreads();
    if (better) {
      if (tid < Model::NP) s.x[tid] = s.cand[tid];
      if (tid < Model::TERMS) s.sums[tid] = s.csum[tid];
      lam = lam / 10.0;
    } else {
      lam = lam * 10.0;
    }
    __syncthreads();
  }
}

// L3 / LH3 / LF3 / LA3 score and count of s.x in pixels (s.px), rounded to float (s.fm)
template <class Model, class Pair, class Points>
__device__ void lo_rescore(LoShared<Model>& s, const Pair& P, Points pts, int n, float thr2, int tid) {
  if (tid == 0) {
    Model::pixels(s, P, s.x, s.px);
    for (int i = 0; i < Model::NF; ++i) s.fm[i] = (float)s.px[i];
    s.score = 0;
  }
  __syncthreads();
  const float w = (float)GEO_LO_QSCALE / thr2;
  unsigned long long acc = 0;
  for (int k = tid; k < n; k += RED) acc += lo_term(Model::err(s.fm, pts[k]), thr2, w);
  if (acc) atomicAdd(&s.score, acc);
  __syncthreads();
}

}  // namespace
