// Batched LO-RANSAC homography on the matcher's output: MSAC-scored four-point sampling with Levenberg-Marquardt local
// optimisation and a final refinement (include/geometry_b200.h, steps LH1-LH8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  geo_api.cu's compaction and Hartley normalisation kernel (geo_hf.cuh)
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair, one thread per sample: the four-point DLT of step 4, fp32 (lo_hf.cuh)
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against the chunk's
//            models, one thread per sample, and adds count << 40 | MSAC score with one 64-bit atomic per sample
//            (lo_hf.cuh)
//     lo     one CTA per pair: the chunk's lowest (score, h); when it beats the pair's model, LM on the truncated
//            transfer cost and a re-score; then the adaptive stop.  Otherwise it returns at once.
//   final    one CTA per pair: the final LM refinement, H and its inliers
// A stopped pair's CTAs return at once.  Compiled with -fmad=false: oracle/lo_homography_oracle.py takes the same steps.
#include <stdint.h>

#include "geo_lm.cuh"
#include "lg_internal.h"
#include "lo_hf.cuh"

namespace {

constexpr int LOH_DOF = 8;
constexpr int LOH_TERMS = 45;  // J^T J upper triangle (36), J^T r (8), truncated cost
constexpr int LOH_GROUP = 15;  // terms per pass of the fixed-order sums: three passes keep red within static shared

// Shared state of one pair's CTA in the LO and final kernels
struct LohShared {
  double red[LOH_GROUP][RED];
  double Hn[9], cand[9];              // unit-norm normalised model being refined and the LM step's candidate
  double sums[LOH_TERMS], csum[LOH_TERMS];
  double basis[LOH_DOF][9];           // tangent basis at the model being summed or updated
  double Hu[9], G[LOH_DOF][9];        // T1^-1 Hn T0 and its derivatives along the basis
  double Ho[9];                       // the scaled pixel model of the last re-scored Hn
  float fm[9];                        // a model rounded to float
  unsigned long long key, score;
  int take, step_ok;
};

// Hn = T1 H T0^-1 at unit Frobenius norm (header step LH7)
__device__ void normalised_model(const GeoPair& P, const double* H, double* Hn) {
  const double T1[9] = {P.s1, 0.0, -(P.s1 * P.cx1), 0.0, P.s1, -(P.s1 * P.cy1), 0.0, 0.0, 1.0};
  const double r = 1.0 / P.s0;
  const double T0i[9] = {r, 0.0, P.cx0, 0.0, r, P.cy0, 0.0, 0.0, 1.0};
  double tmp[9];
  mm3(T1, H, tmp);
  mm3(tmp, T0i, Hn);
  double f = 0.0;
  for (int i = 0; i < 9; ++i) f = f + Hn[i] * Hn[i];
  f = sqrt(f);
  for (int i = 0; i < 9; ++i) Hn[i] = Hn[i] / f;
}

// T1^-1 X T0, unscaled (the first half of denormalise)
__device__ void to_pixels(const GeoPair& P, const double* X, double* out) {
  const double r = 1.0 / P.s1;
  const double L[9] = {r, 0.0, P.cx1, 0.0, r, P.cy1, 0.0, 0.0, 1.0};
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

// The LOH_TERMS sums at the normalised model X (header step LH7) into out
__device__ void loh_terms(LohShared& s, const GeoPair& P, const double* X, const float4* pts, int n, double thr2,
                          double* out, int tid) {
  if (tid == 0) {
    householder_basis(X, s.basis);
    to_pixels(P, X, s.Hu);
    for (int k = 0; k < LOH_DOF; ++k) to_pixels(P, s.basis[k], s.G[k]);
  }
  __syncthreads();
  double acc[LOH_TERMS];
#pragma unroll
  for (int i = 0; i < LOH_TERMS; ++i) acc[i] = 0.0;
  const double* h = s.Hu;
  for (int k = tid; k < n; k += RED) {
    const float4 p = pts[k];
    const double x = p.x, y = p.y, u = p.z, v = p.w;
    const double w = 1.0 / ((h[6] * x + h[7] * y) + h[8]);
    const double px = ((h[0] * x + h[1] * y) + h[2]) * w, py = ((h[3] * x + h[4] * y) + h[5]) * w;
    const double dx = u - px, dy = v - py;
    const double err = dx * dx + dy * dy;
    const bool in = err < thr2;
    acc[LOH_TERMS - 1] = acc[LOH_TERMS - 1] + (in ? err : thr2);
    if (!in) continue;
    double jx[LOH_DOF], jy[LOH_DOF];
#pragma unroll
    for (int q = 0; q < LOH_DOF; ++q) {
      const volatile double* g = s.G[q];  // re-read per point: held in registers, the 72 entries spill
      const double da = (g[0] * x + g[1] * y) + g[2], db = (g[3] * x + g[4] * y) + g[5];
      const double dc = (g[6] * x + g[7] * y) + g[8];
      jx[q] = -((da - px * dc) * w);
      jy[q] = -((db - py * dc) * w);
    }
    int e = 0;
#pragma unroll
    for (int i = 0; i < LOH_DOF; ++i)
#pragma unroll
      for (int j = i; j < LOH_DOF; ++j, ++e) acc[e] = acc[e] + (jx[i] * jx[j] + jy[i] * jy[j]);
#pragma unroll
    for (int i = 0; i < LOH_DOF; ++i) acc[36 + i] = acc[36 + i] + (jx[i] * dx + jy[i] * dy);
  }
#pragma unroll
  for (int g = 0; g < LOH_TERMS; g += LOH_GROUP) lo_tree_sums<LOH_GROUP>(acc + g, s.red, out + g, tid);
}

// X' = normalize(X + sum_k d_k basis_k), the basis taken at X (header step LH7); thread 0 only
__device__ void loh_update(LohShared& s, const double* X, const double* d, double* out) {
  householder_basis(X, s.basis);
  double f = 0.0;
  for (int i = 0; i < 9; ++i) {
    double v = X[i];
    for (int k = 0; k < LOH_DOF; ++k) v = v + d[k] * s.basis[k][i];
    out[i] = v;
    f = f + v * v;
  }
  f = sqrt(f);
  for (int i = 0; i < 9; ++i) out[i] = out[i] / f;
}

// steps LM steps from s.Hn, in place (header step LH7); every thread of the CTA calls it
__device__ void loh_refine(LohShared& s, const GeoPair& P, const float4* pts, int n, double thr2, int steps, int tid) {
  loh_terms(s, P, s.Hn, pts, n, thr2, s.sums, tid);
  double lam = GEO_LO_LAMBDA0;  // every thread keeps the same schedule
  for (int it = 0; it < steps; ++it) {
    if (tid == 0) {
      double d[LOH_DOF];
      s.step_ok = lm_solve<LOH_DOF>(s.sums, s.sums + 36, lam, d);
      if (s.step_ok) loh_update(s, s.Hn, d, s.cand);
    }
    __syncthreads();
    if (!s.step_ok) {
      lam = lam * 10.0;
      __syncthreads();
      continue;
    }
    loh_terms(s, P, s.cand, pts, n, thr2, s.csum, tid);
    const bool better = s.csum[LOH_TERMS - 1] < s.sums[LOH_TERMS - 1];
    __syncthreads();
    if (better) {
      if (tid < 9) s.Hn[tid] = s.cand[tid];
      if (tid < LOH_TERMS) s.sums[tid] = s.csum[tid];
      lam = lam / 10.0;
    } else {
      lam = lam * 10.0;
    }
    __syncthreads();
  }
}

// LH3 score and count of s.Hn in pixels, scaled as step 4 (s.Ho) and rounded to float (s.fm)
__device__ void loh_rescore(LohShared& s, const GeoPair& P, const float4* pts, float thr2, int tid) {
  if (tid == 0) {
    denormalise(GEO_HOMOGRAPHY, P, s.Hn, s.Ho);
    for (int i = 0; i < 9; ++i) s.fm[i] = (float)s.Ho[i];
    s.score = 0;
  }
  __syncthreads();
  const float w = (float)GEO_LO_QSCALE / thr2;
  unsigned long long acc = 0;
  for (int k = tid; k < P.n; k += RED) acc += lo_term(geo_err(GEO_HOMOGRAPHY, s.fm, pts[k]), thr2, w);
  if (acc) atomicAdd(&s.score, acc);
  __syncthreads();
}

// After chunk c: the chunk's best hypothesis, the local optimisation when it beats the pair's model, the stop
__global__ void __launch_bounds__(RED, 1) loh_kernel(LoHfArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  GeoPair& P = a.g.w.pair[b];
  if (P.stop) return;
  LoHfPair& L = a.l.pair[b];
  __shared__ LohShared s;
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
      normalised_model(P, L.model, s.Hn);
    }
    __syncthreads();
    loh_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_STEPS, t);
    loh_rescore(s, P, pts, a.g.thr2, t);
    if (t == 0 && (s.score & LO_SCORE_MASK) < L.score) {
      for (int i = 0; i < 9; ++i) L.model[i] = s.Ho[i];
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
             drawn >= update_num_iters(a.g.confidence, 1.0 - (double)cnt / P.n, 4, a.g.max_iters);
  }
}

// Final refinement and the outputs (header steps LH6, LH8)
__global__ void __launch_bounds__(RED, 1) loh_final_kernel(LoHfArgs a) {
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
  __shared__ LohShared s;
  const float4* pts = a.g.w.pts + (long)b * a.g.M;
  const int* idx = a.g.w.idx + (long)b * a.g.M;
  if (t == 0) normalised_model(P, L.model, s.Hn);
  __syncthreads();
  loh_refine(s, P, pts, P.n, (double)a.g.thr2, GEO_LO_FINAL_STEPS, t);
  loh_rescore(s, P, pts, a.g.thr2, t);
  if (t == 0 && (s.score & LO_SCORE_MASK) > L.score) {  // the refinement is kept unless its score rises
    for (int i = 0; i < 9; ++i) {
      s.Ho[i] = L.model[i];
      s.fm[i] = (float)L.model[i];
    }
    s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
  }
  __syncthreads();
  for (int k = t; k < P.n; k += RED)
    if (geo_err(GEO_HOMOGRAPHY, s.fm, pts[k]) < a.g.thr2) inl[idx[k]] = 1;
  if (t < 9) o.model[(long)b * 9 + t] = s.Ho[t];
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

extern "C" size_t geo_lo_homography_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  GeoWs w;
  LoHfWs l;
  return lohf_carve(nullptr, B, M, &w, &l) + 256;
}

extern "C" int geo_homography_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  if (!cfg || !in || !out) return lg_set_error("geo_homography_lo: null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return lg_set_error("geo_homography_lo: ABI version mismatch");
  if (cfg->model != GEO_HOMOGRAPHY) return lg_set_error("geo_homography_lo: model must be GEO_HOMOGRAPHY");
  if (cfg->max_iters < 1 || cfg->max_iters > GEO_MAX_ITERS)
    return lg_set_error("geo_homography_lo: max_iters outside [1, 2^24]");
  if (!(cfg->threshold > 0.0) || !isfinite(cfg->threshold))
    return lg_set_error("geo_homography_lo: threshold must be positive");
  if (!(cfg->confidence >= 0.0 && cfg->confidence <= 1.0))
    return lg_set_error("geo_homography_lo: confidence outside [0, 1]");
  if (in->B < 0 || in->M < 0 || in->N < 0) return lg_set_error("geo_homography_lo: negative size");
  if (in->M > GEO_LO_MAX_MATCHES) return lg_set_error("geo_homography_lo: M above GEO_LO_MAX_MATCHES");
  if (in->B == 0) return 0;
  const GeoOutputs& o = out->geo;
  if (!o.model || !o.num_inliers || !o.success || !o.best_hypothesis || !o.num_hypotheses ||
      !out->num_local_optimizations || !out->cost || (in->M > 0 && !o.inliers))  // an empty mask may have no storage
    return lg_set_error("geo_homography_lo: null output");
  if (in->M > 0 && (!in->kpts0 || !in->matches0 || (in->N > 0 && !in->kpts1)))
    return lg_set_error("geo_homography_lo: null input");
  if (!workspace || workspace_bytes < geo_lo_homography_workspace_bytes(in->B, in->M, cfg->max_iters))
    return lg_set_error("geo_homography_lo: workspace too small");
  LoHfArgs a{};
  lohf_carve((char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255), in->B, in->M, &a.g.w, &a.l);
  GeoArgs& g = a.g;
  g.B = in->B; g.M = in->M; g.N = in->N;
  g.kind = GEO_HOMOGRAPHY;
  g.s = 4;
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
    lohf_score_kernel<GEO_HOMOGRAPHY><<<dim3(g.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
    loh_kernel<<<g.B, RED, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
  }
  loh_final_kernel<<<g.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
