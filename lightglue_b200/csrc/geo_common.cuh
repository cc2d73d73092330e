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
