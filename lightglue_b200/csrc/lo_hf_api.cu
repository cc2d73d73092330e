// Batched LO-RANSAC homography and fundamental matrix on the matcher's output: MSAC-scored four-point (H) or
// eight-point (F) sampling with Levenberg-Marquardt local optimisation and a final refinement (include/geometry_b200.h,
// steps LH1-LH8 and LF1-LF8).  H is refined at unit norm in the tangent space of the sphere, F at rank 2 in its
// orthonormal representation (U, V, sigma).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  geo_api.cu's compaction and Hartley normalisation kernel (geo_hf.cuh)
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair, one thread per sample: the minimal solve of step 4, fp32
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against the chunk's
//            models, one thread per sample, and adds count << 40 | MSAC score with one 64-bit atomic per sample
//     lo     one CTA per pair: the chunk's lowest (score, h); when it beats the pair's model, LM on the truncated
//            transfer (H) or Sampson (F) cost and a re-score; then the adaptive stop.  Otherwise it returns at once.
//   final    one CTA per pair: the final LM refinement, the model and its inliers
// A stopped pair's CTAs return at once.  Compiled with -fmad=false: oracle/lo_homography_oracle.py and
// oracle/lo_fundamental_oracle.py take the same steps.
#include <stdint.h>

#include "geo_hf.cuh"
#include "lg_internal.h"
#include "lo_common.cuh"

namespace {

struct LoHfPair {
  double model[9];           // the pair's model in pixels, scaled as step 4
  unsigned long long score;  // its LH3 / LF3 score
  int count;                 // its inliers
  int h;                     // the hypothesis that seeded it; -1: none yet
  int nlo;                   // local optimisations adopted
};

struct LoHfWs {
  LoHfPair* pair;           // [B]
  unsigned long long* acc;  // [B, GEO_CHUNK] count << 40 | score of the current chunk's hypotheses
};

size_t lohf_carve(char* base, int B, int M, GeoWs* w, LoHfWs* l) {
  WsBump b{base, carve(base, B, M, w)};
  l->pair = b.take<LoHfPair>(B);
  l->acc = b.take<unsigned long long>((size_t)B * GEO_CHUNK);
  return b.bytes();
}

struct LoHfArgs {
  GeoArgs g;
  LoHfWs l;
  int32_t* num_lo;
  int64_t* cost;
};

// Step 4's hypotheses of chunk c (a.g.kind and a.g.s pick H or F), one thread per sample
__global__ void __launch_bounds__(GEO_CHUNK, 1) lohf_hyp_kernel(LoHfArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c == 0 && t == 0) {
    LoHfPair& L = a.l.pair[b];
    L.score = 0;
    L.count = 0;
    L.h = -1;
    L.nlo = 0;
  }
  const GeoPair& P = a.g.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  double m[9];
  const bool ok = P.stop == 0 && h < a.g.max_iters && geo_hypothesis(a.g, P, a.g.w.pts + (long)b * a.g.M, h, m);
  if (ok) {
    float* hm = a.g.w.hyp + ((long)b * GEO_CHUNK + t) * 9;
    for (int i = 0; i < 9; ++i) hm[i] = (float)m[i];
    a.l.acc[(long)b * GEO_CHUNK + t] = 0;
  }
  a.g.w.count[(long)b * GEO_CHUNK + t] = ok ? 0 : -1;
}

// The chunk's LH3 / LF3 scores, count << 40 | MSAC score
template <int KIND>
struct LoHfScore {
  using Args = LoHfArgs;
  using Acc = unsigned long long;
  static constexpr int SOLS = 1, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const GeoWs& ws(const LoHfArgs& a) { return a.g.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  __device__ LoHfScore(const LoHfArgs& a, const GeoPair&, int b)
      : src{a.g.w.pts + (long)b * a.g.M}, sums(a.l.acc), thr2(a.g.thr2), w((float)GEO_LO_QSCALE / a.g.thr2) {}
  __device__ unsigned long long term(const float* h, const float4* p) const {
    return lo_term(geo_err(KIND, h, p[0]), thr2, w);
  }
};

// T1^-1 X T0 (H) or (T1^T X) T0 (F), unscaled: the first half of denormalise
template <int KIND>
__device__ void to_pixels(const GeoPair& P, const double* X, double* out) {
  double L[9];
  if (KIND == GEO_HOMOGRAPHY) {
    const double r = 1.0 / P.s1;
    const double Li[9] = {r, 0.0, P.cx1, 0.0, r, P.cy1, 0.0, 0.0, 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Li[i];
  } else {
    const double Lt[9] = {P.s1, 0.0, 0.0, 0.0, P.s1, 0.0, -(P.s1 * P.cx1), -(P.s1 * P.cy1), 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Lt[i];
  }
  const double T0[9] = {P.s0, 0.0, -(P.s0 * P.cx0), 0.0, P.s0, -(P.s0 * P.cy0), 0.0, 0.0, 1.0};
  double tmp[9];
  mm3(L, X, tmp);
  mm3(tmp, T0, out);
}

// The columns j != m of the Householder reflection I - (2 / v.v) v v^T, v = e_m - Hn, which maps e_m to Hn: an
// orthonormal basis of the tangent space of the unit sphere at Hn (header step LH7)
__device__ void householder_basis(const double* Hn, double (*B)[9]) {
  int m = 0;
  for (int i = 1; i < 9; ++i)
    if (fabs(Hn[i]) < fabs(Hn[m])) m = i;
  double v[9], vv = 0.0;
  for (int i = 0; i < 9; ++i) v[i] = (i == m ? 1.0 : 0.0) - Hn[i];
  for (int i = 0; i < 9; ++i) vv = vv + v[i] * v[i];
  const double c = 2.0 / vv;
  for (int j = 0, k = 0; j < 9; ++j) {
    if (j == m) continue;
    for (int i = 0; i < 9; ++i) B[k][i] = (i == j ? 1.0 : 0.0) - c * v[i] * v[j];
    ++k;
  }
}

// The homography for lo_common.cuh's LM loop and re-score: x = Hn, the unit-norm normalised model (header step LH7)
struct HomographyLo {
  static constexpr int KIND = GEO_HOMOGRAPHY, DOF = 8, TERMS = 45, GROUP = 15, NP = 9, NF = 9;
  struct Scratch {
    double basis[DOF][9];     // tangent basis at the model being summed or updated
    double Hu[9], G[DOF][9];  // T1^-1 Hn T0 and its derivatives along the basis
  };

  // Hn = T1 H T0^-1 at unit Frobenius norm of a pixel H; thread 0 only
  static __device__ void start(LoShared<HomographyLo>& s, const GeoPair& P, const double* H) {
    const double T1[9] = {P.s1, 0.0, -(P.s1 * P.cx1), 0.0, P.s1, -(P.s1 * P.cy1), 0.0, 0.0, 1.0};
    const double r = 1.0 / P.s0;
    const double T0i[9] = {r, 0.0, P.cx0, 0.0, r, P.cy0, 0.0, 0.0, 1.0};
    double tmp[9];
    mm3(T1, H, tmp);
    mm3(tmp, T0i, s.x);
    double f = 0.0;
    for (int i = 0; i < 9; ++i) f = f + s.x[i] * s.x[i];
    f = sqrt(f);
    for (int i = 0; i < 9; ++i) s.x[i] = s.x[i] / f;
  }

  static __device__ void terms(LoShared<HomographyLo>& s, const GeoPair& P, const double* X, const float4* pts, int n,
                               double thr2, double* out, int tid) {
    if (tid == 0) {
      householder_basis(X, s.m.basis);
      to_pixels<KIND>(P, X, s.m.Hu);
      for (int k = 0; k < DOF; ++k) to_pixels<KIND>(P, s.m.basis[k], s.m.G[k]);
    }
    __syncthreads();
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    const double* h = s.m.Hu;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts[k];
      const double x = p.x, y = p.y, u = p.z, v = p.w;
      const double w = 1.0 / ((h[6] * x + h[7] * y) + h[8]);
      const double px = ((h[0] * x + h[1] * y) + h[2]) * w, py = ((h[3] * x + h[4] * y) + h[5]) * w;
      const double dx = u - px, dy = v - py;
      const double err = dx * dx + dy * dy;
      const bool in = err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (!in) continue;
      double jx[DOF], jy[DOF];
#pragma unroll
      for (int q = 0; q < DOF; ++q) {
        const volatile double* g = s.m.G[q];  // re-read per point: held in registers, the 72 entries spill
        const double da = (g[0] * x + g[1] * y) + g[2], db = (g[3] * x + g[4] * y) + g[5];
        const double dc = (g[6] * x + g[7] * y) + g[8];
        jx[q] = -((da - px * dc) * w);
        jy[q] = -((db - py * dc) * w);
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + (jx[i] * jx[j] + jy[i] * jy[j]);
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[36 + i] = acc[36 + i] + (jx[i] * dx + jy[i] * dy);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // X' = normalize(X + sum_k d_k basis_k), the basis taken at X
  static __device__ void update(LoShared<HomographyLo>& s, const double* X, const double* d, double* out) {
    householder_basis(X, s.m.basis);
    double f = 0.0;
    for (int i = 0; i < 9; ++i) {
      double v = X[i];
      for (int k = 0; k < DOF; ++k) v = v + d[k] * s.m.basis[k][i];
      out[i] = v;
      f = f + v * v;
    }
    f = sqrt(f);
    for (int i = 0; i < 9; ++i) out[i] = out[i] / f;
  }

  static __device__ void pixels(LoShared<HomographyLo>&, const GeoPair& P, const double* X, double* out) {
    denormalise(KIND, P, X, out);
  }

  static __device__ __forceinline__ float err(const float* h, float4 p) { return geo_err(KIND, h, p); }
};

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Fn_ab = u1_a*v1_b + sig*u2_a*v2_b of x = (U, V, sig)
__device__ void compose(const double* x, double* Fn) {
  const double* U = x;
  const double* V = x + 9;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) Fn[a * 3 + b] = U[a * 3] * V[b * 3] + x[18] * U[a * 3 + 1] * V[b * 3 + 1];
}

// The fundamental matrix for lo_common.cuh's LM loop and re-score: x = U (0-8), V (9-17) and sig (18), the orthonormal
// representation Fn = u1 v1^T + sig u2 v2^T of the normalised model, u_k, v_k columns of U, V (header step LF7)
struct FundamentalLo {
  static constexpr int KIND = GEO_FUNDAMENTAL, DOF = 7, TERMS = 36, GROUP = 18, NP = 19, NF = 9;
  struct Scratch {
    double Fu[9], G[DOF][9];  // T1^T Fn T0 and the directions at Fn in pixels
  };

  // x of a pixel F: Fn = (T1^-T F) T0^-1, then U, V and sig by step 4's one-sided Jacobi; thread 0 only
  static __device__ void start(LoShared<FundamentalLo>& s, const GeoPair& P, const double* F) {
    const double r1 = 1.0 / P.s1, r0 = 1.0 / P.s0;
    const double T1it[9] = {r1, 0.0, 0.0, 0.0, r1, 0.0, P.cx1, P.cy1, 1.0};
    const double T0i[9] = {r0, 0.0, P.cx0, 0.0, r0, P.cy0, 0.0, 0.0, 1.0};
    double tmp[9], A[9], W[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    mm3(T1it, F, tmp);
    mm3(tmp, T0i, A);
    jacobi_columns3(A, W);
    double nrm[3];
    int m = 0;
    for (int j = 0; j < 3; ++j) {
      double nj = 0.0;
      for (int i = 0; i < 3; ++i) nj = nj + A[i * 3 + j] * A[i * 3 + j];
      nrm[j] = nj;
      if (nj < nrm[m]) m = j;
    }
    int p = m == 0 ? 1 : 0, q = m == 2 ? 1 : 2;
    if (nrm[q] > nrm[p]) {
      const int t = p;
      p = q;
      q = t;
    }
    const double s1 = sqrt(nrm[p]), s2 = sqrt(nrm[q]);
    double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
    for (int r = 0; r < 3; ++r) {
      u1[r] = A[r * 3 + p] / s1;
      u2[r] = A[r * 3 + q] / s2;
      v1[r] = W[r * 3 + p];
      v2[r] = W[r * 3 + q];
    }
    cross3(u1, u2, u3);
    cross3(v1, v2, v3);
    double* U = s.x;
    double* V = s.x + 9;
    for (int r = 0; r < 3; ++r) {
      U[r * 3] = u1[r]; U[r * 3 + 1] = u2[r]; U[r * 3 + 2] = u3[r];
      V[r * 3] = v1[r]; V[r * 3 + 1] = v2[r]; V[r * 3 + 2] = v3[r];
    }
    s.x[18] = s2 / s1;
  }

  static __device__ void terms(LoShared<FundamentalLo>& s, const GeoPair& P, const double* X, const float4* pts, int n,
                               double thr2, double* out, int tid) {
    if (tid == 0) {
      double Fn[9], D[9];
      compose(X, Fn);
      to_pixels<KIND>(P, Fn, s.m.Fu);
      for (int k = 0; k < 3; ++k) {
        const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
        double w[3], c[3];
        for (int j = 0; j < 3; ++j) {  // [e_k]x Fn: column j is e_k x Fn[:, j]
          for (int i = 0; i < 3; ++i) w[i] = Fn[i * 3 + j];
          cross3(e, w, c);
          for (int i = 0; i < 3; ++i) D[i * 3 + j] = c[i];
        }
        to_pixels<KIND>(P, D, s.m.G[k]);
        for (int i = 0; i < 3; ++i) cross3(e, Fn + i * 3, D + i * 3);  // -Fn [e_k]x: row i is e_k x Fn[i, :]
        to_pixels<KIND>(P, D, s.m.G[3 + k]);
      }
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) D[a * 3 + b] = X[a * 3 + 1] * X[9 + b * 3 + 1];
      to_pixels<KIND>(P, D, s.m.G[6]);
    }
    __syncthreads();
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    const double* f = s.m.Fu;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts[k];
      const double x = p.x, y = p.y, u = p.z, v = p.w;
      const double a0 = (f[0] * x + f[1] * y) + f[2], a1 = (f[3] * x + f[4] * y) + f[5];
      const double a2 = (f[6] * x + f[7] * y) + f[8];
      const double d = (u * a0 + v * a1) + a2;
      const double b0 = (f[0] * u + f[3] * v) + f[6], b1 = (f[1] * u + f[4] * v) + f[7];
      const double den = ((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1;
      const double err = (d * d) / den;
      const bool in = err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (!in) continue;
      const double sq = sqrt(den), r = d / sq;
      double J[DOF];
#pragma unroll
      for (int q = 0; q < DOF; ++q) {
        const volatile double* g = s.m.G[q];  // re-read per point, as the homography's LM does
        const double da0 = (g[0] * x + g[1] * y) + g[2], da1 = (g[3] * x + g[4] * y) + g[5];
        const double da2 = (g[6] * x + g[7] * y) + g[8];
        const double dd = (u * da0 + v * da1) + da2;
        const double db0 = (g[0] * u + g[3] * v) + g[6], db1 = (g[1] * u + g[4] * v) + g[7];
        const double dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1;
        J[q] = (dd - d * dden / den) / sq;
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + J[i] * J[j];
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[28 + i] = acc[28 + i] + J[i] * r;
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // U' = Q(d0..2) U, V' = Q(d3..5) V, sig' = sig + d6
  static __device__ void update(LoShared<FundamentalLo>&, const double* X, const double* d, double* out) {
    double Q[9];
    quat_rotation(d, Q);
    mm3(Q, X, out);
    quat_rotation(d + 3, Q);
    mm3(Q, X + 9, out + 9);
    out[18] = X[18] + d[6];
  }

  static __device__ void pixels(LoShared<FundamentalLo>&, const GeoPair& P, const double* X, double* out) {
    double Fn[9];
    compose(X, Fn);
    denormalise(KIND, P, Fn, out);
  }

  static __device__ __forceinline__ float err(const float* h, float4 p) { return geo_err(KIND, h, p); }
};

// After chunk c: the chunk's best hypothesis, the local optimisation when it beats the pair's model, the stop
template <class Model>
__global__ void __launch_bounds__(RED, 1) lohf_lo_kernel(LoHfArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  GeoPair& P = a.g.w.pair[b];
  if (P.stop) return;
  LoHfPair& L = a.l.pair[b];
  __shared__ LoShared<Model> s;
  if (t == 0) s.key = ~0ull;
  __syncthreads();
  if (t < GEO_CHUNK && a.g.w.count[(long)b * GEO_CHUNK + t] >= 0)
    atomicMin(&s.key, (a.l.acc[(long)b * GEO_CHUNK + t] & LO_SCORE_MASK) << 28 | (unsigned)(c * GEO_CHUNK + t));
  __syncthreads();
  const unsigned long long key = s.key;
  const float4* pts = a.g.w.pts + (long)b * a.g.M;
  if (t == 0) s.take = key != ~0ull && (L.h < 0 || (key >> 28) < L.score);
  __syncthreads();
  if (s.take) {
    if (t == 0) {
      const unsigned h = (unsigned)(key & 0xfffffffu);
      geo_hypothesis(a.g, P, pts, h, L.model);
      L.score = key >> 28;
      L.count = (int)(a.l.acc[(long)b * GEO_CHUNK + h - c * GEO_CHUNK] >> 40);
      L.h = (int)h;
      Model::start(s, P, L.model);
    }
    __syncthreads();
    lo_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_STEPS, t);
    lo_rescore(s, P, pts, P.n, a.g.thr2, t);
    if (t == 0 && (s.score & LO_SCORE_MASK) < L.score) {
      for (int i = 0; i < 9; ++i) L.model[i] = s.px[i];
      L.score = s.score & LO_SCORE_MASK;
      L.count = (int)(s.score >> 40);
      L.nlo = L.nlo + 1;
    }
  }
  if (t == 0) {
    const int drawn = min((c + 1) * GEO_CHUNK, a.g.max_iters);
    const int cnt = L.h >= 0 ? L.count : 0;
    P.drawn = drawn;
    P.stop = drawn >= a.g.max_iters ||
             drawn >= update_num_iters(a.g.confidence, 1.0 - (double)cnt / P.n, a.g.s, a.g.max_iters);
  }
}

// Final refinement and the outputs (header steps LH6 and LH8, LF6 and LF8)
template <class Model>
__global__ void __launch_bounds__(RED, 1) lohf_final_kernel(LoHfArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  const GeoPair& P = a.g.w.pair[b];
  const LoHfPair& L = a.l.pair[b];
  const GeoOutputs& o = a.g.out;
  uint8_t* inl = o.inliers + (long)b * a.g.M;
  for (int i = t; i < a.g.M; i += RED) inl[i] = 0;
  if (!P.ok || L.h < 0) {
    if (t < 9) o.model[(long)b * 9 + t] = 0.0;
    if (t == 0) {
      o.num_inliers[b] = 0;
      o.success[b] = 0;
      o.best_hypothesis[b] = -1;
      o.num_hypotheses[b] = P.drawn;
      a.num_lo[b] = 0;
      a.cost[b] = 0;
    }
    return;
  }
  __shared__ LoShared<Model> s;
  const float4* pts = a.g.w.pts + (long)b * a.g.M;
  const int* idx = a.g.w.idx + (long)b * a.g.M;
  if (t == 0) Model::start(s, P, L.model);
  __syncthreads();
  lo_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_FINAL_STEPS, t);
  lo_rescore(s, P, pts, P.n, a.g.thr2, t);
  if (t == 0 && (s.score & LO_SCORE_MASK) > L.score) {  // the refinement is kept unless its score rises
    for (int i = 0; i < 9; ++i) {
      s.px[i] = L.model[i];
      s.fm[i] = (float)L.model[i];
    }
    s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
  }
  __syncthreads();
  for (int k = t; k < P.n; k += RED)
    if (Model::err(s.fm, pts[k]) < a.g.thr2) inl[idx[k]] = 1;
  if (t < 9) o.model[(long)b * 9 + t] = s.px[t];
  if (t == 0) {
    o.num_inliers[b] = (int)(s.score >> 40);
    o.success[b] = 1;
    o.best_hypothesis[b] = L.h;
    o.num_hypotheses[b] = P.drawn;
    a.num_lo[b] = L.nlo;
    a.cost[b] = (int64_t)(s.score & LO_SCORE_MASK);
  }
}

size_t lohf_workspace_bytes(int B, int M) {
  if (B < 0 || M < 0) return 0;
  GeoWs w;
  LoHfWs l;
  return lohf_carve(nullptr, B, M, &w, &l) + 256;
}

// geo_homography_lo and geo_fundamental_lo: name for the error strings, s the points per sample
template <class Model>
int lohf_estimate(const char* name, int s, const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out,
                  void* workspace, size_t workspace_bytes, void* stream_) {
  int rc = geo_check_config(name, cfg, in, out, GEO_LO_MAX_MATCHES, [&] {
    return cfg->model == Model::KIND          ? nullptr
           : Model::KIND == GEO_HOMOGRAPHY ? "model must be GEO_HOMOGRAPHY"
                                           : "model must be GEO_FUNDAMENTAL";
  }, geo_no_check);
  if (rc == GEO_RUN) {
    const GeoOutputs& o = out->geo;
    rc = geo_check_buffers(name, in, {o.model, o.num_inliers, o.success, o.best_hypothesis, o.num_hypotheses,
                                      out->num_local_optimizations, out->cost}, {o.inliers}, {}, in->kpts1,
                           workspace, workspace_bytes, lohf_workspace_bytes(in->B, in->M));
  }
  if (rc != GEO_RUN) return rc;
  LoHfArgs a{};
  lohf_carve(geo_workspace_base(workspace), in->B, in->M, &a.g.w, &a.l);
  GeoArgs& g = a.g;
  g.B = in->B; g.M = in->M; g.N = in->N;
  g.kind = Model::KIND;
  g.s = s;
  g.max_iters = cfg->max_iters;
  g.chunks = geo_chunks(cfg->max_iters);
  g.seed = cfg->seed;
  g.thr2 = (float)(cfg->threshold * cfg->threshold);
  g.confidence = cfg->confidence;
  g.kpts0 = in->kpts0; g.kpts1 = in->kpts1; g.matches0 = in->matches0;
  g.out = out->geo;
  a.num_lo = out->num_local_optimizations;
  a.cost = out->cost;
  const int splits = geo_score_splits(g.B, g.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  geo_prepare_kernel<<<g.B, 1024, 0, stream>>>(g);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < g.chunks; ++c) {
    lohf_hyp_kernel<<<g.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<LoHfScore<Model::KIND>><<<dim3(g.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
    lohf_lo_kernel<Model><<<g.B, RED, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
  }
  lohf_final_kernel<Model><<<g.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}

}  // namespace

extern "C" size_t geo_lo_homography_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lohf_workspace_bytes(B, M);
}

extern "C" size_t geo_lo_fundamental_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lohf_workspace_bytes(B, M);
}

extern "C" int geo_homography_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return lohf_estimate<HomographyLo>("geo_homography_lo", 4, cfg, in, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_fundamental_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return lohf_estimate<FundamentalLo>("geo_fundamental_lo", 8, cfg, in, out, workspace, workspace_bytes, stream);
}
