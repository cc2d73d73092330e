// The LO-RANSAC pieces shared by the relative pose (lo_pose_api.cu, header steps L1-L8), the homography and the
// fundamental matrix (lo_hf_api.cu, LH1-LH8 and LF1-LF8) and the absolute pose (lo_pnp_api.cu, LA1-LA8), all compiled
// with -fmad=false: the packed score term of the MSAC and MAGSAC++ losses, the fixed-order sums of the
// Levenberg-Marquardt terms, one LM loop and re-score over a model policy, and the schedule of L4-L6 and L8 that every
// LO estimator runs on it (the MAGSAC++ homography and fundamental matrix, MH1-MH8 and MF1-MF8, included).
#pragma once
#include <cuda_runtime.h>

#include "geo_common.cuh"
#include "geo_lm.cuh"
#include "magsac_table.h"
#include "ws_bump.h"

namespace {

constexpr unsigned long long LO_COUNT_ONE = 1ull << 40;  // a score sum's count field (header GEO_LO_MAX_MATCHES)
constexpr unsigned long long LO_SCORE_MASK = LO_COUNT_ONE - 1;

// L3's per-point term of one fp32 error, with the count in bit 40.  A non-finite error is an outlier.  An inlier's
// product is clamped to GEO_LO_QSCALE, so a subnormal thr2 (w = +inf) stays defined, and e == 0 scores 0 (0 * inf).
__device__ __forceinline__ unsigned long long lo_term(float e, float thr2, float w) {
  if (!(e < thr2)) return GEO_LO_QSCALE;
  return LO_COUNT_ONE + (e == 0.f ? 0u : (unsigned)fminf(e * w, (float)GEO_LO_QSCALE));
}

// The loss of an LO estimator: the score term of its fp32 errors (L3) and the per-point cost and weight of its LM
// (L7).  A loss object carries the call's thresholds; term() gives the score term's functor, lm() the scale the LM
// loop passes to the model's terms(), whose per-point sums read point(scale, err, cost, wt) and weigh(wt, x):
//   Msac, the truncated squared error of L3 and L7 at the user's thr2 (every estimator but MH / MF);
//   Magsac, MAGSAC++'s sigma-marginalised loss at the scale T^2 = mt2 (header steps MH3 and MH7), with the count bit
//   still at the user's thr2.
struct Msac {
  float thr2;
  struct Term {
    float thr2, w;
    __device__ __forceinline__ unsigned long long operator()(float e) const { return lo_term(e, thr2, w); }
  };
  __device__ __forceinline__ Term term() const { return {thr2, (float)GEO_LO_QSCALE / thr2}; }
  __device__ __forceinline__ double lm() const { return (double)thr2; }
  // An inlier (err < thr2) adds err and its unweighted terms; any other point adds thr2
  static __device__ __forceinline__ bool point(double thr2, double err, double& cost, double&) {
    const bool in = err < thr2;
    cost = in ? err : thr2;
    return in;
  }
  static __device__ __forceinline__ double weigh(double, double x) { return x; }
};

struct Magsac {
  float thr2, mt2;  // the user's squared threshold (the count) and T^2 (the loss)
  // MH3: u = e * (KNOTS / mt2) in fp32; for u < KNOTS, i = (int)u, f = u - i and rho = R_i + f * (R_(i+1) - R_i)
  // with R the table rounded to float, q = (uint32)fminf(rho * QSCALE, QSCALE); else (NaN included) q = QSCALE
  struct Term {
    float thr2, ks;
    __device__ __forceinline__ unsigned long long operator()(float e) const {
      const unsigned long long c = e < thr2 ? LO_COUNT_ONE : 0ull;
      const float u = e * ks;
      if (!(u < (float)GEO_MAGSAC_KNOTS)) return c + GEO_LO_QSCALE;
      const int i = (int)u;
      const float f = u - (float)i, r0 = (float)MAGSAC_RHO[i], r1 = (float)MAGSAC_RHO[i + 1];
      return c + (unsigned)fminf((r0 + f * (r1 - r0)) * (float)GEO_LO_QSCALE, (float)GEO_LO_QSCALE);
    }
  };
  __device__ __forceinline__ Term term() const { return {thr2, (float)GEO_MAGSAC_KNOTS / mt2}; }
  __device__ __forceinline__ double lm() const { return (double)mt2; }
  // MH7: u = err * ((double)KNOTS / T^2); for u < KNOTS, i = (int)u, f = u - i, cost = R_i + f * (R_(i+1) - R_i) and
  // wt = W_i + f * (W_(i+1) - W_i) in double; else the point costs 1 and adds no terms
  static __device__ __forceinline__ bool point(double mt2, double err, double& cost, double& wt) {
    const double u = err * ((double)GEO_MAGSAC_KNOTS / mt2);
    if (!(u < (double)GEO_MAGSAC_KNOTS)) {
      cost = 1.0;
      return false;
    }
    const int i = (int)u;
    const double f = u - (double)i;
    cost = MAGSAC_RHO[i] + f * (MAGSAC_RHO[i + 1] - MAGSAC_RHO[i]);
    wt = MAGSAC_W[i] + f * (MAGSAC_W[i + 1] - MAGSAC_W[i]);
    return true;
  }
  static __device__ __forceinline__ double weigh(double wt, double x) { return wt * x; }
};

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
//   terms(s, P, x, pts, n, scale, out, tid), the TERMS sums at x (every thread), scale the loss's lm();
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

// steps LM steps from s.x at damping lam0, in place (header steps L7, LH7, LF7, LA7, A7 and AF6); every thread of the
// CTA calls it
template <class Model, class Pair, class Points>
__device__ void lo_refine(LoShared<Model>& s, const Pair& P, Points pts, int n, double thr2, int steps, double lam0,
                          int tid) {
  constexpr int NH = Model::DOF * (Model::DOF + 1) / 2;
  Model::terms(s, P, s.x, pts, n, thr2, s.sums, tid);
  double lam = lam0;  // every thread keeps the same schedule
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

// L3 / LH3 / LF3 / LA3 / MH3 / MF3 score and count of s.x in pixels (s.px), rounded to float (s.fm)
template <class Model, class Pair, class Points, class Loss>
__device__ void lo_rescore(LoShared<Model>& s, const Pair& P, Points pts, int n, Loss loss, int tid) {
  if (tid == 0) {
    Model::pixels(s, P, s.x, s.px);
    for (int i = 0; i < Model::NF; ++i) s.fm[i] = (float)s.px[i];
    s.score = 0;
  }
  __syncthreads();
  const auto term = loss.term();
  unsigned long long acc = 0;
  for (int k = tid; k < n; k += RED) acc += term(Model::err(s.fm, pts[k]));
  if (acc) atomicAdd(&s.score, acc);
  __syncthreads();
}

// ---- the LO schedule (header steps L4-L6 and L8; LH, LF and LA likewise) ----

struct LoPair {
  double model[12];          // the pair's model: R | t (relative and absolute pose), the scaled pixel model (H, F)
  unsigned long long score;  // its score
  int count;                 // its inliers
  int hr;                    // h * 16 + r of the solution that seeded it; -1: none yet
  int nlo;                   // local optimisations adopted
};

struct LoWs {
  LoPair* pair;             // [B]
  unsigned long long* acc;  // [B, GEO_CHUNK, SOLS] count << 40 | score of the current chunk's solutions
};

// The kernels' arguments: Base is the estimator's RANSAC arguments (GeoArgs, PoseArgs or PnpArgs)
template <class Base>
struct LoArgs {
  Base p;
  LoWs l;
  int32_t* num_lo;
  int64_t* cost;
};

// The estimator's workspace, then the LO one
template <class Est>
size_t lo_carve(char* base, int B, int M, LoArgs<typename Est::Base>* a) {
  WsBump b{base, carve(base, B, M, &a->p.w)};
  a->l.pair = b.take<LoPair>(B);
  a->l.acc = b.take<unsigned long long>((size_t)B * GEO_CHUNK * Est::SOLS);
  return b.bytes();
}

template <class Est>
size_t lo_workspace_bytes(int B, int M) {
  if (B < 0 || M < 0) return 0;
  LoArgs<typename Est::Base> a;
  return lo_carve<Est>(nullptr, B, M, &a) + 256;
}

// Pair b's LO state before its first chunk
__device__ __forceinline__ void lo_reset(const LoWs& l, int b, int c) {
  if (c == 0 && threadIdx.x == 0) {
    LoPair& L = l.pair[b];
    L.score = 0;
    L.count = 0;
    L.hr = -1;
    L.nlo = 0;
  }
}

// geo_hyp_kernel's LO-RANSAC schedule (geo_common.cuh): lo_reset on entry, and the MSAC sums zeroed
template <class Solver, class Base>
__device__ __forceinline__ const Base& geo_enter(const LoArgs<Base>& a, int b, int c) {
  lo_reset(a.l, b, c);
  return a.p;
}

template <class Base>
__device__ __forceinline__ unsigned long long* geo_sums(const LoArgs<Base>& a) { return a.l.acc; }

// The schedule runs over Est, the estimator's model policy (LoShared above) with:
//   Base, its RANSAC arguments (a.p.w.pair[b] the pair, a.p.out the outputs); Solver, its geo_hyp_kernel solver;
//   Score, its geo_score_kernel policy; S, the points per sample; SOLS, the solutions per sample;
//   points(a, b), consts(a, b) and loss(a, b), pair b's points, constants and loss (Msac or Magsac above) as the LM
//   loop and the re-score read them;
//   seed(s, a, b, hr, m, L, t), the LM start s.x of solution hr (index m of acc) and L.model of it (every thread; a
//   barrier follows);
//   store(s, L), the re-scored model of s into L.model (thread 0);
//   load(s, a, b, L, t), the LM start of L.model (every thread; a barrier follows);
//   restore(s, a, b, L, t), L's model, score and count as the re-scored model of s (every thread; ends on a barrier);
//   fail(a, b, t), the model fields of a pair without a model, o.inliers already cleared (every thread);
//   write(s, a, b, t), the masks and model fields of the re-scored model of s (every thread).

// L4 and L5 after chunk c: the chunk's lowest (score, h, r); when it beats the pair's model, LM from it and a re-score,
// adopted at a strictly lower score; then the adaptive stop.  A stopped pair's CTA returns at once.
template <class Est>
__global__ void __launch_bounds__(RED, 1) lo_chunk_kernel(LoArgs<typename Est::Base> a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  auto& P = a.p.w.pair[b];
  if (P.stop) return;
  LoPair& L = a.l.pair[b];
  __shared__ LoShared<Est> s;
  if (t == 0) s.key = ~0ull;
  __syncthreads();
  if (t < GEO_CHUNK) {
    const long slot = (long)b * GEO_CHUNK + t;
    const int ns = geo_models(a.p.w, slot);
    const unsigned h = c * GEO_CHUNK + t;
    for (int r = 0; r < ns; ++r)
      atomicMin(&s.key, (a.l.acc[slot * Est::SOLS + r] & LO_SCORE_MASK) << 28 | (h * 16u + (unsigned)r));
  }
  __syncthreads();
  const unsigned long long key = s.key;
  if (t == 0) s.take = key != ~0ull && (L.hr < 0 || (key >> 28) < L.score);
  __syncthreads();
  if (s.take) {
    const unsigned hr = (unsigned)(key & 0xfffffffu);
    const long m = ((long)b * GEO_CHUNK + (hr >> 4) - c * GEO_CHUNK) * Est::SOLS + (hr & 15);
    Est::seed(s, a, b, hr, m, L, t);
    if (t == 0) {
      L.score = key >> 28;
      L.count = (int)(a.l.acc[m] >> 40);
      L.hr = (int)hr;
    }
    __syncthreads();
    const auto pts = Est::points(a, b);
    const auto loss = Est::loss(a, b);
    lo_refine(s, Est::consts(a, b), pts, P.n, loss.lm(), GEO_LO_STEPS, GEO_LO_LAMBDA0, t);
    lo_rescore(s, Est::consts(a, b), pts, P.n, loss, t);
    if (t == 0 && (s.score & LO_SCORE_MASK) < L.score) {
      Est::store(s, L);
      L.score = s.score & LO_SCORE_MASK;
      L.count = (int)(s.score >> 40);
      L.nlo = L.nlo + 1;
    }
  }
  if (t == 0) {
    const int drawn = min((c + 1) * GEO_CHUNK, a.p.max_iters);
    const int cnt = L.hr >= 0 ? L.count : 0;
    P.drawn = drawn;
    P.stop = drawn >= a.p.max_iters ||
             drawn >= update_num_iters(a.p.confidence, 1.0 - (double)cnt / P.n, Est::S, a.p.max_iters);
  }
}

// L6 and L8: the final refinement, kept unless its score rises, and the outputs
template <class Est>
__global__ void __launch_bounds__(RED, 1) lo_final_kernel(LoArgs<typename Est::Base> a) {
  const int b = blockIdx.x, t = threadIdx.x;
  const auto& P = a.p.w.pair[b];
  const LoPair& L = a.l.pair[b];
  const auto& o = a.p.out;
  if (!P.ok || L.hr < 0) {
    for (int i = t; i < a.p.M; i += RED) o.inliers[(long)b * a.p.M + i] = 0;
    Est::fail(a, b, t);
    if (t == 0) {
      o.num_inliers[b] = 0;
      o.success[b] = 0;
      o.best_hypothesis[b] = -1;
      if constexpr (Est::SOLS > 1) o.best_solution[b] = -1;  // only an estimator with several solutions reports one
      o.num_hypotheses[b] = P.drawn;
      a.num_lo[b] = 0;
      a.cost[b] = 0;
    }
    return;
  }
  __shared__ LoShared<Est> s;
  const auto pts = Est::points(a, b);
  const auto loss = Est::loss(a, b);
  Est::load(s, a, b, L, t);
  __syncthreads();
  lo_refine(s, Est::consts(a, b), pts, P.n, loss.lm(), GEO_LO_FINAL_STEPS, GEO_LO_LAMBDA0, t);
  lo_rescore(s, Est::consts(a, b), pts, P.n, loss, t);
  if (t == 0) s.take = (s.score & LO_SCORE_MASK) > L.score;
  __syncthreads();
  if (s.take) Est::restore(s, a, b, L, t);
  Est::write(s, a, b, t);
  if (t == 0) {
    o.num_inliers[b] = (int)(s.score >> 40);
    o.success[b] = 1;
    o.best_hypothesis[b] = L.hr >> 4;
    if constexpr (Est::SOLS > 1) o.best_solution[b] = L.hr & 15;
    o.num_hypotheses[b] = P.drawn;
    a.num_lo[b] = L.nlo;
    a.cost[b] = (int64_t)(s.score & LO_SCORE_MASK);
  }
}

// Every LO estimator's launches, all fixed by (B, M, max_iters): prepare, the estimator's compaction kernel; per chunk
// of GEO_CHUNK samples, geo_hyp_kernel (one CTA per pair, one thread per sample: the minimal solutions, fp32),
// geo_score_kernel (count << 40 | score of every solution) and lo_chunk_kernel (one CTA per pair); then
// lo_final_kernel.
template <class Est, class Base>
int lo_launch(const Base& p, int32_t* num_lo, int64_t* cost, void* workspace, void (*prepare)(Base), void* stream_) {
  LoArgs<Base> a{p, {}, num_lo, cost};
  lo_carve<Est>(geo_workspace_base(workspace), p.B, p.M, &a);
  const int splits = geo_score_splits(p.B, p.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  prepare<<<p.B, 1024, 0, stream>>>(a.p);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < p.chunks; ++c) {
    geo_hyp_kernel<typename Est::Solver, LoArgs<Base>><<<p.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<typename Est::Score><<<dim3(p.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
    lo_chunk_kernel<Est><<<p.B, RED, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
  }
  lo_final_kernel<Est><<<p.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}

}  // namespace
