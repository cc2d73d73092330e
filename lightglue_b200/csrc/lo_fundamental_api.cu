// Batched LO-RANSAC fundamental matrix on the matcher's output: MSAC-scored eight-point sampling with Levenberg-Marquardt
// local optimisation of a rank-2 F and a final refinement (include/geometry_b200.h, steps LF1-LF8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  geo_api.cu's compaction and Hartley normalisation kernel (geo_hf.cuh)
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair, one thread per sample: the eight-point solve and rank 2 of step 4, fp32 (lo_hf.cuh)
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against the chunk's
//            models, one thread per sample, and adds count << 40 | MSAC score with one 64-bit atomic per sample
//            (lo_hf.cuh)
//     lo     one CTA per pair: the chunk's lowest (score, h); when it beats the pair's model, LM on the truncated
//            Sampson cost and a re-score; then the adaptive stop.  Otherwise it returns at once.
//   final    one CTA per pair: the final LM refinement, F and its inliers
// A stopped pair's CTAs return at once.  Compiled with -fmad=false: oracle/lo_fundamental_oracle.py takes the same steps.
#include <stdint.h>

#include "geo_lm.cuh"
#include "lg_internal.h"
#include "lo_hf.cuh"

namespace {

constexpr int LOF_DOF = 7;
constexpr int LOF_TERMS = 36;  // J^T J upper triangle (28), J^T r (7), truncated cost
constexpr int LOF_GROUP = 18;  // terms per pass of the fixed-order sums: two passes keep red within static shared

// Shared state of one pair's CTA in the LO and final kernels
struct LofShared {
  double red[LOF_GROUP][RED];
  double U[9], V[9], sig;        // the model being refined: Fn = u1 v1^T + sig u2 v2^T, u_k, v_k columns of U, V
  double cU[9], cV[9], csig;     // the LM step's candidate
  double sums[LOF_TERMS], csum[LOF_TERMS];
  double Fu[9], G[LOF_DOF][9];   // T1^T Fn T0 and the directions at Fn in pixels
  double Fo[9];                  // the scaled pixel model of the last re-scored Fn
  float fm[9];                   // a model rounded to float
  unsigned long long key, score;
  int take, step_ok;
};

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Fn = (T1^-T F) T0^-1 of a pixel F (header step LF7)
__device__ void normalised_model(const GeoPair& P, const double* F, double* Fn) {
  const double r1 = 1.0 / P.s1, r0 = 1.0 / P.s0;
  const double T1it[9] = {r1, 0.0, 0.0, 0.0, r1, 0.0, P.cx1, P.cy1, 1.0};
  const double T0i[9] = {r0, 0.0, P.cx0, 0.0, r0, P.cy0, 0.0, 0.0, 1.0};
  double tmp[9];
  mm3(T1it, F, tmp);
  mm3(tmp, T0i, Fn);
}

// (T1^T X) T0, unscaled (the first half of denormalise for F)
__device__ void to_pixels(const GeoPair& P, const double* X, double* out) {
  const double L[9] = {P.s1, 0.0, 0.0, 0.0, P.s1, 0.0, -(P.s1 * P.cx1), -(P.s1 * P.cy1), 1.0};
  const double T0[9] = {P.s0, 0.0, -(P.s0 * P.cx0), 0.0, P.s0, -(P.s0 * P.cy0), 0.0, 0.0, 1.0};
  double tmp[9];
  mm3(L, X, tmp);
  mm3(tmp, T0, out);
}

// U, V and sig of Fn by step 4's one-sided Jacobi (header step LF7); thread 0 only
__device__ void factorise(const double* Fn, double* U, double* V, double* sig) {
  double A[9], W[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) A[i] = Fn[i];
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
  for (int r = 0; r < 3; ++r) {
    U[r * 3] = u1[r]; U[r * 3 + 1] = u2[r]; U[r * 3 + 2] = u3[r];
    V[r * 3] = v1[r]; V[r * 3 + 1] = v2[r]; V[r * 3 + 2] = v3[r];
  }
  *sig = s2 / s1;
}

// Fn_ab = u1_a*v1_b + sig*u2_a*v2_b
__device__ void compose(const double* U, const double* V, double sig, double* Fn) {
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) Fn[a * 3 + b] = U[a * 3] * V[b * 3] + sig * U[a * 3 + 1] * V[b * 3 + 1];
}

// The LOF_TERMS sums at the model (U, V, sig) (header step LF7) into out
__device__ void lof_terms(LofShared& s, const GeoPair& P, const double* U, const double* V, double sig,
                          const float4* pts, int n, double thr2, double* out, int tid) {
  if (tid == 0) {
    double Fn[9], D[9];
    compose(U, V, sig, Fn);
    to_pixels(P, Fn, s.Fu);
    for (int k = 0; k < 3; ++k) {
      const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
      double w[3], c[3];
      for (int j = 0; j < 3; ++j) {  // [e_k]x Fn: column j is e_k x Fn[:, j]
        for (int i = 0; i < 3; ++i) w[i] = Fn[i * 3 + j];
        cross3(e, w, c);
        for (int i = 0; i < 3; ++i) D[i * 3 + j] = c[i];
      }
      to_pixels(P, D, s.G[k]);
      for (int i = 0; i < 3; ++i) cross3(e, Fn + i * 3, D + i * 3);  // -Fn [e_k]x: row i is e_k x Fn[i, :]
      to_pixels(P, D, s.G[3 + k]);
    }
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) D[a * 3 + b] = U[a * 3 + 1] * V[b * 3 + 1];
    to_pixels(P, D, s.G[6]);
  }
  __syncthreads();
  double acc[LOF_TERMS];
#pragma unroll
  for (int i = 0; i < LOF_TERMS; ++i) acc[i] = 0.0;
  const double* f = s.Fu;
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
    acc[LOF_TERMS - 1] = acc[LOF_TERMS - 1] + (in ? err : thr2);
    if (!in) continue;
    const double sq = sqrt(den), r = d / sq;
    double J[LOF_DOF];
#pragma unroll
    for (int q = 0; q < LOF_DOF; ++q) {
      const volatile double* g = s.G[q];  // re-read per point, as the homography's LM does
      const double da0 = (g[0] * x + g[1] * y) + g[2], da1 = (g[3] * x + g[4] * y) + g[5];
      const double da2 = (g[6] * x + g[7] * y) + g[8];
      const double dd = (u * da0 + v * da1) + da2;
      const double db0 = (g[0] * u + g[3] * v) + g[6], db1 = (g[1] * u + g[4] * v) + g[7];
      const double dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1;
      J[q] = (dd - d * dden / den) / sq;
    }
    int e = 0;
#pragma unroll
    for (int i = 0; i < LOF_DOF; ++i)
#pragma unroll
      for (int j = i; j < LOF_DOF; ++j, ++e) acc[e] = acc[e] + J[i] * J[j];
#pragma unroll
    for (int i = 0; i < LOF_DOF; ++i) acc[28 + i] = acc[28 + i] + J[i] * r;
  }
#pragma unroll
  for (int g = 0; g < LOF_TERMS; g += LOF_GROUP) lo_tree_sums<LOF_GROUP>(acc + g, s.red, out + g, tid);
}

// U' = Q(d0..2) U, V' = Q(d3..5) V, sig' = sig + d6 (header step LF7); thread 0 only
__device__ void lof_update(LofShared& s, const double* d) {
  double Q[9];
  quat_rotation(d, Q);
  mm3(Q, s.U, s.cU);
  quat_rotation(d + 3, Q);
  mm3(Q, s.V, s.cV);
  s.csig = s.sig + d[6];
}

// steps LM steps from (s.U, s.V, s.sig), in place (header step LF7); every thread of the CTA calls it
__device__ void lof_refine(LofShared& s, const GeoPair& P, const float4* pts, int n, double thr2, int steps, int tid) {
  lof_terms(s, P, s.U, s.V, s.sig, pts, n, thr2, s.sums, tid);
  double lam = GEO_LO_LAMBDA0;  // every thread keeps the same schedule
  for (int it = 0; it < steps; ++it) {
    if (tid == 0) {
      double d[LOF_DOF];
      s.step_ok = lm_solve<LOF_DOF>(s.sums, s.sums + 28, lam, d);
      if (s.step_ok) lof_update(s, d);
    }
    __syncthreads();
    if (!s.step_ok) {
      lam = lam * 10.0;
      __syncthreads();
      continue;
    }
    lof_terms(s, P, s.cU, s.cV, s.csig, pts, n, thr2, s.csum, tid);
    const bool better = s.csum[LOF_TERMS - 1] < s.sums[LOF_TERMS - 1];
    __syncthreads();
    if (better) {
      if (tid < 9) {
        s.U[tid] = s.cU[tid];
        s.V[tid] = s.cV[tid];
      }
      if (tid == 0) s.sig = s.csig;
      if (tid < LOF_TERMS) s.sums[tid] = s.csum[tid];
      lam = lam / 10.0;
    } else {
      lam = lam * 10.0;
    }
    __syncthreads();
  }
}

// LF3 score and count of (s.U, s.V, s.sig) in pixels, scaled as step 4 (s.Fo) and rounded to float (s.fm)
__device__ void lof_rescore(LofShared& s, const GeoPair& P, const float4* pts, float thr2, int tid) {
  if (tid == 0) {
    double Fn[9];
    compose(s.U, s.V, s.sig, Fn);
    denormalise(GEO_FUNDAMENTAL, P, Fn, s.Fo);
    for (int i = 0; i < 9; ++i) s.fm[i] = (float)s.Fo[i];
    s.score = 0;
  }
  __syncthreads();
  const float w = (float)GEO_LO_QSCALE / thr2;
  unsigned long long acc = 0;
  for (int k = tid; k < P.n; k += RED) acc += lo_term(geo_err(GEO_FUNDAMENTAL, s.fm, pts[k]), thr2, w);
  if (acc) atomicAdd(&s.score, acc);
  __syncthreads();
}

// (s.U, s.V, s.sig) of a pixel model; thread 0 only
__device__ void lof_start(LofShared& s, const GeoPair& P, const double* F) {
  double Fn[9];
  normalised_model(P, F, Fn);
  factorise(Fn, s.U, s.V, &s.sig);
}

// After chunk c: the chunk's best hypothesis, the local optimisation when it beats the pair's model, the stop
__global__ void __launch_bounds__(RED, 1) lof_kernel(LoHfArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  GeoPair& P = a.g.w.pair[b];
  if (P.stop) return;
  LoHfPair& L = a.l.pair[b];
  __shared__ LofShared s;
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
      lof_start(s, P, L.model);
    }
    __syncthreads();
    lof_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_STEPS, t);
    lof_rescore(s, P, pts, a.g.thr2, t);
    if (t == 0 && (s.score & LO_SCORE_MASK) < L.score) {
      for (int i = 0; i < 9; ++i) L.model[i] = s.Fo[i];
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

// Final refinement and the outputs (header steps LF6, LF8)
__global__ void __launch_bounds__(RED, 1) lof_final_kernel(LoHfArgs a) {
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
  __shared__ LofShared s;
  const float4* pts = a.g.w.pts + (long)b * a.g.M;
  const int* idx = a.g.w.idx + (long)b * a.g.M;
  if (t == 0) lof_start(s, P, L.model);
  __syncthreads();
  lof_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_FINAL_STEPS, t);
  lof_rescore(s, P, pts, a.g.thr2, t);
  if (t == 0 && (s.score & LO_SCORE_MASK) > L.score) {  // the refinement is kept unless its score rises
    for (int i = 0; i < 9; ++i) {
      s.Fo[i] = L.model[i];
      s.fm[i] = (float)L.model[i];
    }
    s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
  }
  __syncthreads();
  for (int k = t; k < P.n; k += RED)
    if (geo_err(GEO_FUNDAMENTAL, s.fm, pts[k]) < a.g.thr2) inl[idx[k]] = 1;
  if (t < 9) o.model[(long)b * 9 + t] = s.Fo[t];
  if (t == 0) {
    o.num_inliers[b] = (int)(s.score >> 40);
    o.success[b] = 1;
    o.best_hypothesis[b] = L.h;
    o.num_hypotheses[b] = P.drawn;
    a.num_lo[b] = L.nlo;
    a.cost[b] = (int64_t)(s.score & LO_SCORE_MASK);
  }
}

}  // namespace

extern "C" size_t geo_lo_fundamental_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  GeoWs w;
  LoHfWs l;
  return lohf_carve(nullptr, B, M, &w, &l) + 256;
}

extern "C" int geo_fundamental_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  if (!cfg || !in || !out) return lg_set_error("geo_fundamental_lo: null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return lg_set_error("geo_fundamental_lo: ABI version mismatch");
  if (cfg->model != GEO_FUNDAMENTAL) return lg_set_error("geo_fundamental_lo: model must be GEO_FUNDAMENTAL");
  if (cfg->max_iters < 1 || cfg->max_iters > GEO_MAX_ITERS)
    return lg_set_error("geo_fundamental_lo: max_iters outside [1, 2^24]");
  if (!(cfg->threshold > 0.0) || !isfinite(cfg->threshold))
    return lg_set_error("geo_fundamental_lo: threshold must be positive");
  if (!(cfg->confidence >= 0.0 && cfg->confidence <= 1.0))
    return lg_set_error("geo_fundamental_lo: confidence outside [0, 1]");
  if (in->B < 0 || in->M < 0 || in->N < 0) return lg_set_error("geo_fundamental_lo: negative size");
  if (in->M > GEO_LO_MAX_MATCHES) return lg_set_error("geo_fundamental_lo: M above GEO_LO_MAX_MATCHES");
  if (in->B == 0) return 0;
  const GeoOutputs& o = out->geo;
  if (!o.model || !o.num_inliers || !o.success || !o.best_hypothesis || !o.num_hypotheses ||
      !out->num_local_optimizations || !out->cost || (in->M > 0 && !o.inliers))  // an empty mask may have no storage
    return lg_set_error("geo_fundamental_lo: null output");
  if (in->M > 0 && (!in->kpts0 || !in->matches0 || (in->N > 0 && !in->kpts1)))
    return lg_set_error("geo_fundamental_lo: null input");
  if (!workspace || workspace_bytes < geo_lo_fundamental_workspace_bytes(in->B, in->M, cfg->max_iters))
    return lg_set_error("geo_fundamental_lo: workspace too small");
  LoHfArgs a{};
  lohf_carve((char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255), in->B, in->M, &a.g.w, &a.l);
  GeoArgs& g = a.g;
  g.B = in->B; g.M = in->M; g.N = in->N;
  g.kind = GEO_FUNDAMENTAL;
  g.s = 8;
  g.max_iters = cfg->max_iters;
  g.chunks = (cfg->max_iters + GEO_CHUNK - 1) / GEO_CHUNK;
  g.seed = cfg->seed;
  g.thr2 = (float)(cfg->threshold * cfg->threshold);
  g.confidence = cfg->confidence;
  g.kpts0 = in->kpts0; g.kpts1 = in->kpts1; g.matches0 = in->matches0;
  g.out = o;
  a.num_lo = out->num_local_optimizations;
  a.cost = out->cost;
  // the score CTAs of geo_estimate
  const int want = (2 * lg_num_sms() + g.B - 1) / g.B;
  int splits = (g.M + 127) / 128;
  if (splits > want) splits = want;
  if (splits < 1) splits = 1;
  const cudaStream_t stream = (cudaStream_t)stream_;
  geo_prepare_kernel<<<g.B, 1024, 0, stream>>>(g);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < g.chunks; ++c) {
    lohf_hyp_kernel<<<g.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    lohf_score_kernel<GEO_FUNDAMENTAL><<<dim3(g.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
    lof_kernel<<<g.B, RED, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
  }
  lof_final_kernel<<<g.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
