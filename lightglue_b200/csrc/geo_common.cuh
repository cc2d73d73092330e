// Helpers shared by every geometry estimator (geo_api.cu, pose_api.cu, lo_pose_api.cu, lo_hf_api.cu, pnp_api.cu,
// lo_pnp_api.cu), all compiled with -fmad=false.  include/geometry_b200.h states each step; oracle/geometry_oracle.py and
// oracle/pose_oracle.py restate them in numpy.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <initializer_list>

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

// The valid models of chunk slot `slot` of a workspace that counts them in nsol (pose, PnP); geo_hf.cuh overloads it
// for the H/F workspace, whose one model is valid when its count is >= 0
template <class Ws>
__device__ __forceinline__ int geo_models(const Ws& w, long slot) { return w.nsol[slot]; }

// Records that chunk slot `slot` holds ns models, as geo_models reads it back
template <class Ws>
__device__ __forceinline__ void geo_set_models(const Ws& w, long slot, int ns) { w.nsol[slot] = ns; }

// Folds chunk c's counts (SOLS per sample) into the pair's best and decides whether the pair stops after s-point
// samples.  The best is packed (count + 1) << 32 | ~(h * 16 + r) and kept by atomic max, so ties go to the smallest
// hypothesis h, then solution r.  Called by every thread of a GEO_CHUNK-thread CTA; thread t owns sample
// c * GEO_CHUNK + t.
template <int SOLS, class Args>
__device__ void geo_fold(const Args& a, int s, int b, int c) {
  __shared__ unsigned long long best;
  auto* P = a.w.pair + b;
  const int t = threadIdx.x;
  const bool live = P->stop == 0;
  if (t == 0) best = P->best;
  __syncthreads();
  const long slot = (long)b * GEO_CHUNK + t;
  const int ns = geo_models(a.w, slot);
  const unsigned h = c * GEO_CHUNK + t;
  for (int r = 0; live && r < ns; ++r) {
    const int k = a.w.count[slot * SOLS + r];
    atomicMax(&best, ((unsigned long long)(k + 1) << 32) | (unsigned)~(h * 16u + (unsigned)r));
  }
  __syncthreads();
  if (t == 0 && live) {
    const int drawn = min((c + 1) * GEO_CHUNK, a.max_iters);
    const int cnt = best ? (int)(best >> 32) - 1 : 0;
    P->best = best;
    P->drawn = drawn;
    P->stop = drawn >= a.max_iters || drawn >= update_num_iters(a.confidence, 1.0 - (double)cnt / P->n, s, a.max_iters);
  }
  __syncthreads();
}

// The score launch of a chunk, (B, splits) CTAs of GEO_CHUNK threads: each CTA streams a slice of its pair's points
// through shared memory, one thread per sample sums Q's per-point term over its valid models, and adds each nonzero
// sum with one atomic.  Q is the estimator's score policy:
//   Args, the kernel's argument struct, and ws(a), its workspace (pair, hyp, count; nsol where SOLS > 1);
//   SOLS models of NF floats per sample, at hyp[(slot * SOLS + r) * NF];
//   K float4 arrays per point (src[0..K-1]), staged TILE points at a time;
//   Q(a, P, b), the call's constants and point arrays of pair b; term(g, p), the term of point p for model g, of type
//   Acc; sums, the [B, GEO_CHUNK, SOLS] array the sums are added into.
template <class Q>
__global__ void __launch_bounds__(GEO_CHUNK) geo_score_kernel(typename Q::Args a) {
  const int b = blockIdx.x, split = blockIdx.y, t = threadIdx.x;
  const auto& w = Q::ws(a);
  const auto& P = w.pair[b];
  if (P.stop) return;
  const int lo = (int)((long)P.n * split / gridDim.y), hi = (int)((long)P.n * (split + 1) / gridDim.y);
  const long slot = (long)b * GEO_CHUNK + t;
  const int ns = geo_models(w, slot);
  const Q q(a, P, b);
  float g[Q::SOLS][Q::NF];
  typename Q::Acc k[Q::SOLS];
#pragma unroll
  for (int r = 0; r < Q::SOLS; ++r) {
    k[r] = 0;
#pragma unroll
    for (int i = 0; i < Q::NF; ++i) g[r][i] = r < ns ? w.hyp[(slot * Q::SOLS + r) * Q::NF + i] : 0.f;
  }
  __shared__ float4 tile[Q::K][Q::TILE];
  for (int base = lo; base < hi; base += Q::TILE) {
    const int m = min(Q::TILE, hi - base);
    __syncthreads();
    for (int i = t; i < m; i += GEO_CHUNK)
#pragma unroll
      for (int j = 0; j < Q::K; ++j) tile[j][i] = q.src[j][base + i];
    __syncthreads();
    if (Q::SOLS > 1 || ns > 0)  // a one-model sample tests its validity once per tile, not once per point
      for (int i = 0; i < m; ++i) {
        float4 p[Q::K];
#pragma unroll
        for (int j = 0; j < Q::K; ++j) p[j] = tile[j][i];
#pragma unroll
        for (int r = 0; r < Q::SOLS; ++r)
          if (r < ns) k[r] += q.term(g[r], p);
      }
  }
#pragma unroll
  for (int r = 0; r < Q::SOLS; ++r)
    if (r < ns && k[r]) atomicAdd(q.sums + slot * Q::SOLS + r, k[r]);
}

// The hyp launch of a chunk runs on a Solver, the estimator's minimal solve:
//   SOLS, NX and NF: up to SOLS solutions of NX doubles per sample, each scored as a pixel model of NF floats;
//   s(a), the points per sample;
//   solve(a, b, h, x), sample h of pair b solved into x[0..ns-1], returning ns (0 for a degenerate sample);
//   pixels(a, b, x, px), a solution's pixel model.
// The schedule is picked by the argument type: plain RANSAC (Base) folds the previous chunk on entry and zeroes the
// inlier counts; LO-RANSAC (LoArgs<Base>, lo_common.cuh) resets the pair's LO state and zeroes the MSAC sums.
template <class Solver, class Base>
__device__ __forceinline__ const Base& geo_enter(const Base& a, int b, int c) {
  if (c > 0) geo_fold<Solver::SOLS>(a, Solver::s(a), b, c - 1);
  return a;
}

template <class Base>
__device__ __forceinline__ int* geo_sums(const Base& a) { return a.w.count; }

// Chunk c's hypotheses, one CTA per pair, one thread per sample: solved in double, rounded into w.hyp
template <class Solver, class Args>
__global__ void __launch_bounds__(GEO_CHUNK, 1) geo_hyp_kernel(Args a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  const auto& p = geo_enter<Solver>(a, b, c);
  const auto& P = p.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  const long slot = (long)b * GEO_CHUNK + t;
  int ns = 0;
  if (P.stop == 0 && h < p.max_iters) {
    double x[Solver::SOLS][Solver::NX];
    ns = Solver::solve(p, b, h, x);
    float* hm = p.w.hyp + slot * Solver::SOLS * Solver::NF;
    for (int r = 0; r < ns; ++r) {
      double px[Solver::NF];
      Solver::pixels(p, b, x[r], px);
      for (int i = 0; i < Solver::NF; ++i) hm[r * Solver::NF + i] = (float)px[i];
      geo_sums(a)[slot * Solver::SOLS + r] = 0;
    }
  }
  // On the plain H/F workspace the one count is also the slot's model record, so a valid slot gets the same 0 again
  geo_set_models(p.w, slot, ns);
}

// The upper triangle of A^T A (45 sums, row-major) over the points k < n with inlier(k), each adding the rows that
// rows(k, ra, rb) fills (it returns 1 or 2), in step 2's fixed order.  One pass over the points per row i keeps 9
// accumulators in registers.  Every thread of a RED-thread CTA calls it; ata is valid on thread 0.
template <class Inlier, class Rows>
__device__ void geo_ata(int n, Inlier inlier, Rows rows, double* red, double* ata, int t) {
  for (int i = 0, e0 = 0; i < 9; e0 += 9 - i, ++i) {
    double acc[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) acc[j] = 0.0;
    for (int k = t; k < n; k += RED) {
      if (!inlier(k)) continue;
      double ra[9], rb[9];
      const int nr = rows(k, ra, rb);
#pragma unroll
      for (int j = 0; j < 9; ++j)
        if (j >= i) acc[j] = acc[j] + (nr == 2 ? ra[i] * ra[j] + rb[i] * rb[j] : ra[i] * ra[j]);
    }
#pragma unroll
    for (int j = 0; j < 9; ++j)
      if (j >= i) {
        const double s = tree_sum(acc[j], red, t);
        if (t == 0) ata[e0 + j - i] = s;
      }
  }
}

// The smallest-eigenvalue eigenvector of the symmetric 9x9 whose upper triangle is ata (geo_ata's layout)
__device__ __forceinline__ void ata_null_vector(const double* ata, double* v) {
  double A[9][9];
  for (int i = 0, e = 0; i < 9; ++i)
    for (int j = i; j < 9; ++j, ++e) A[i][j] = A[j][i] = ata[e];
  smallest_eigvec<9>(A, v);
}

// The final kernel's shared state: the best hypothesis re-solved (0) and its refit (1)
template <class Est>
struct GeoFinal {
  double x[2][Est::NX];   // the solutions
  double px[2][Est::NF];  // their pixel models
  float fm[2][Est::NF];   // rounded to float
  int count[2];           // their inliers; count[1] == -1: no refit
  typename Est::Scratch m;
};

// The final launch of plain RANSAC, one RED-thread CTA per pair: folds the last chunk, solves the best hypothesis again
// in double, refits it on its inliers, keeps the refit unless it has fewer inliers, and writes the outputs.  Est is the
// Solver with:
//   Base, the kernel's arguments; Score, its geo_score_kernel policy; Scratch, its shared state in GeoFinal;
//   clear(a, b, t), the masks set to 0 before anything else (every thread);
//   fail(a, b, t), the model fields of a pair without a model (every thread);
//   refits(a, hcount), whether a best hypothesis with hcount inliers is refitted;
//   refit(s, a, b, t), s.x[1] from s.x[0] on the inliers of s.fm[0] (every thread, ends with s.x[1] on thread 0);
//   inlier(a, b, g, k), the fp32 test of compacted point k against the float model g;
//   write(s, a, b, u, t), the masks and model fields of solution u of s (every thread).
template <class Est>
__global__ void __launch_bounds__(RED, 1) geo_final_kernel(typename Est::Base a) {
  const int b = blockIdx.x, t = threadIdx.x;
  geo_fold<Est::SOLS>(a, Est::s(a), b, a.chunks - 1);
  const auto& P = a.w.pair[b];
  const auto& o = a.out;
  __shared__ GeoFinal<Est> s;
  Est::clear(a, b, t);
  const unsigned long long key = P.best;
  if (!P.ok || key == 0) {
    Est::fail(a, b, t);
    if (t == 0) {
      o.num_inliers[b] = 0;
      o.success[b] = 0;
      o.best_hypothesis[b] = -1;
      if constexpr (Est::SOLS > 1) o.best_solution[b] = -1;  // only an estimator with several solutions reports one
      o.num_hypotheses[b] = P.drawn;
    }
    return;
  }
  const unsigned hr = ~(unsigned)(key & 0xffffffffu);
  const int hcount = (int)(key >> 32) - 1;
  if (t == 0) {
    double x[Est::SOLS][Est::NX];
    Est::solve(a, b, hr >> 4, x);
    for (int i = 0; i < Est::NX; ++i) s.x[0][i] = x[hr & 15][i];
    Est::pixels(a, b, s.x[0], s.px[0]);
    for (int i = 0; i < Est::NF; ++i) s.fm[0][i] = (float)s.px[0][i];
    s.count[0] = hcount;
    s.count[1] = -1;
  }
  __syncthreads();
  if (Est::refits(a, hcount)) {
    Est::refit(s, a, b, t);
    if (t == 0) {
      Est::pixels(a, b, s.x[1], s.px[1]);
      for (int i = 0; i < Est::NF; ++i) s.fm[1][i] = (float)s.px[1][i];
      s.count[1] = 0;
    }
    __syncthreads();
    int k1 = 0;
    for (int k = t; k < P.n; k += RED) k1 += Est::inlier(a, b, s.fm[1], k);
    if (k1) atomicAdd(&s.count[1], k1);
    __syncthreads();
  }
  const int u = s.count[1] >= s.count[0] ? 1 : 0;
  Est::write(s, a, b, u, t);
  if (t == 0) {
    o.num_inliers[b] = s.count[u];
    o.success[b] = 1;
    o.best_hypothesis[b] = (int)(hr >> 4);
    if constexpr (Est::SOLS > 1) o.best_solution[b] = (int)(hr & 15);
    o.num_hypotheses[b] = P.drawn;
  }
}

// The mask of the inliers of float model g, by row of matches0 through w.idx (every thread; clear(a, b, t) zeroed it)
template <class Est>
__device__ void geo_write_mask(const typename Est::Base& a, int b, const float* g, int t) {
  const int* idx = a.w.idx + (long)b * a.M;
  uint8_t* inl = a.out.inliers + (long)b * a.M;
  for (int k = t; k < a.w.pair[b].n; k += RED)
    if (Est::inlier(a, b, g, k)) inl[idx[k]] = 1;
}

// Every plain estimator's launches, all fixed by (B, M, max_iters): prepare, the estimator's compaction kernel; per
// chunk of GEO_CHUNK samples, geo_hyp_kernel and geo_score_kernel (the inlier counts of every solution); then
// geo_final_kernel.  The caller launches the estimator's tail after it.  Returns 0 or the launch error.
template <class Est, class Base>
int geo_launch(const Base& a, void (*prepare)(Base), cudaStream_t stream) {
  const int splits = geo_score_splits(a.B, a.M);
  prepare<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    geo_hyp_kernel<Est, Base><<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<typename Est::Score><<<dim3(a.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  geo_final_kernel<Est><<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}

// ---- host side of the entry points ----

constexpr int GEO_RUN = -1;  // geo_check_config, geo_check_buffers: the arguments pass, the call goes on

int geo_error(const char* entry, const char* what) {
  char msg[96];
  snprintf(msg, sizeof(msg), "%s: %s", entry, what);
  return lg_set_error(msg);
}

const char* geo_no_check() { return nullptr; }

// The configuration and size checks of every entry point, in order, reported as "<entry>: <what>": null arguments, ABI
// version, model(), max_iters, threshold, confidence, distance(), negative sizes, M above max_m.  model and distance
// are the entry point's own checks at their place, each an error or nullptr.  Returns 0 when B == 0 (nothing to do),
// GEO_RUN, or the error code.
template <class Cfg, class In, class Model, class Distance>
int geo_check_config(const char* entry, const Cfg* cfg, const In* in, const void* out, int max_m, Model model,
                     Distance distance) {
  if (!cfg || !in || !out) return geo_error(entry, "null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return geo_error(entry, "ABI version mismatch");
  if (const char* what = model()) return geo_error(entry, what);
  if (cfg->max_iters < 1 || cfg->max_iters > GEO_MAX_ITERS) return geo_error(entry, "max_iters outside [1, 2^24]");
  if (!(cfg->threshold > 0.0) || !isfinite(cfg->threshold)) return geo_error(entry, "threshold must be positive");
  if (!(cfg->confidence >= 0.0 && cfg->confidence <= 1.0)) return geo_error(entry, "confidence outside [0, 1]");
  if (const char* what = distance()) return geo_error(entry, what);
  if (in->B < 0 || in->M < 0 || in->N < 0) return geo_error(entry, "negative size");
  if (in->M > max_m) return geo_error(entry, "M above GEO_LO_MAX_MATCHES");
  return in->B == 0 ? 0 : GEO_RUN;
}

// The pointer and workspace checks that follow, in order: null outputs (masks, the [B, M] ones, may have no storage
// when M == 0), null intrinsics, null inputs (in1, image 1's keypoints or 3D points, only when N > 0), and a workspace
// of at least need bytes.  Returns GEO_RUN or the error code.
template <class In>
int geo_check_buffers(const char* entry, const In* in, std::initializer_list<const void*> outputs,
                      std::initializer_list<const void*> masks, std::initializer_list<const void*> intrinsics,
                      const void* in1, const void* workspace, size_t workspace_bytes, size_t need) {
  bool missing = false;
  for (const void* p : outputs) missing = missing || !p;
  for (const void* p : masks) missing = missing || (in->M > 0 && !p);
  if (missing) return geo_error(entry, "null output");
  for (const void* p : intrinsics)
    if (!p) return geo_error(entry, "null intrinsics");
  if (in->M > 0 && (!in->kpts0 || !in->matches0 || (in->N > 0 && !in1))) return geo_error(entry, "null input");
  if (!workspace || workspace_bytes < need) return geo_error(entry, "workspace too small");
  return GEO_RUN;
}

// The carving base of a workspace: its first 256-byte boundary (the *_workspace_bytes entry points add 256 for it)
char* geo_workspace_base(void* workspace) { return (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255); }

int geo_chunks(int max_iters) { return (max_iters + GEO_CHUNK - 1) / GEO_CHUNK; }

}  // namespace
