// Batched absolute pose on the matcher's 2D-3D matches: Lambda Twist P3P RANSAC, then Levenberg-Marquardt on the
// inliers (include/geometry_b200.h, steps A1-A8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  one 1024-thread CTA per pair: ordered compaction of the valid matches, calibrated coordinates, K check
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold), decides the
//            adaptive stop, then one thread per sample solves it: up to 4 fp32 projections
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against every solution
//            of the chunk, one thread per sample, and adds the inlier counts
//   refit    one CTA per pair: folds the last chunk, Levenberg-Marquardt from the best solution, recount, R and t
//   mask     one thread per row of matches0: the final inlier mask
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/pnp_oracle.py takes the same
// steps in numpy.
#include <stdint.h>

#include "pnp_common.cuh"

namespace {

constexpr int MASK_THREADS = 256;

__global__ void __launch_bounds__(GEO_CHUNK, 1) pnp_hyp_kernel(PnpArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c > 0) geo_fold<SOLS>(a, S, b, c - 1);
  const PnpPair& P = a.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  int ns = 0;
  int id[S];
  if (P.stop == 0 && h < a.max_iters && geo_sample(a.seed, h, P.n, S, id) == S) {
    double Rs[SOLS][9], ts[SOLS][3];
    ns = p3p(a.w.pts + (long)b * a.M, a.w.wld + (long)b * a.M, id, Rs, ts);
    const double* K = a.K0 + (long)b * 9;
    float* hm = a.w.hyp + ((long)b * GEO_CHUNK + t) * SOLS * 12;
    for (int r = 0; r < ns; ++r) {
      double Pm[12];
      projection(K, Rs[r], ts[r], Pm);
      for (int i = 0; i < 12; ++i) hm[r * 12 + i] = (float)Pm[i];
      a.w.count[((long)b * GEO_CHUNK + t) * SOLS + r] = 0;
    }
  }
  a.w.nsol[(long)b * GEO_CHUNK + t] = ns;
}

// Inlier counts of every projection, on a tile of pixels and world points
struct PnpScore {
  using Args = PnpArgs;
  using Acc = int;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const PnpArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  float thr2;
  __device__ PnpScore(const PnpArgs& a, const PnpPair& P, int b)
      : src{a.w.pts + (long)b * a.M, a.w.wld + (long)b * a.M}, sums(a.w.count), thr2(P.thr2) {}
  __device__ int term(const float* g, const float4* p) const { return reproj_inlier(g, p[0], p[1], thr2); }
};

constexpr int LM_TERMS = 28;  // J^T J upper triangle (21), J^T r (6), cost

// This thread's partial sums of the refit's terms at (R, t) over the inliers k = t, t + RED, ... (header step A7)
__device__ void lm_partials(const double* K, const double* R, const double* t, const float4* pts, const float4* wld,
                            const uint8_t* inl, int n, int tid, double* acc) {
  const double fx = K[0], s = K[1], cx = K[2], fy = K[4], cy = K[5];
  for (int i = 0; i < LM_TERMS; ++i) acc[i] = 0.0;
  for (int k = tid; k < n; k += RED) {
    if (!inl[k]) continue;
    const float4 p = pts[k], q = wld[k];
    const double u = p.x, v = p.y, W[3] = {q.x, q.y, q.z};
    double Xc[3];
    for (int i = 0; i < 3; ++i) Xc[i] = R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i];
    const double iz = 1.0 / Xc[2];
    const double ax = Xc[0] * iz, bx = Xc[1] * iz;
    const double pu = fx * ax + s * bx;
    const double ru = pu + cx - u, rv = fy * bx + cy - v;
    const double gu[3] = {fx * iz, s * iz, -(pu * iz)};
    const double gv[3] = {0.0, fy * iz, -(fy * bx * iz)};
    const double ju[6] = {gu[2] * Xc[1] - gu[1] * Xc[2], gu[0] * Xc[2] - gu[2] * Xc[0], gu[1] * Xc[0] - gu[0] * Xc[1],
                          gu[0], gu[1], gu[2]};
    const double jv[6] = {gv[2] * Xc[1] - gv[1] * Xc[2], gv[0] * Xc[2] - gv[2] * Xc[0], gv[1] * Xc[0] - gv[0] * Xc[1],
                          gv[0], gv[1], gv[2]};
    int e = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = i; j < 6; ++j, ++e) acc[e] = acc[e] + (ju[i] * ju[j] + jv[i] * jv[j]);
#pragma unroll
    for (int i = 0; i < 6; ++i) acc[21 + i] = acc[21 + i] + (ju[i] * ru + jv[i] * rv);
    acc[27] = acc[27] + (ru * ru + rv * rv);
  }
}

__global__ void __launch_bounds__(RED, 1) pnp_refit_kernel(PnpArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  geo_fold<SOLS>(a, S, b, a.chunks - 1);
  PnpPair& P = a.w.pair[b];
  const float4* pts = a.w.pts + (long)b * a.M;
  const float4* wld = a.w.wld + (long)b * a.M;
  const double* K = a.K0 + (long)b * 9;
  __shared__ double red[RED];
  __shared__ double pose[2][12];  // R, t of the best solution and of the refit
  __shared__ double cand[12];     // the LM step's candidate
  __shared__ double sums[LM_TERMS], csum[LM_TERMS];
  __shared__ float fm[2][12];
  __shared__ int count[2];
  __shared__ int step_ok;
  const unsigned long long key = P.best;
  if (!P.ok || key == 0) {
    if (t < 9) a.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.out.t[(long)b * 3 + t] = 0.0;
    if (t == 0) {
      a.out.num_inliers[b] = 0;
      a.out.success[b] = 0;
      a.out.best_hypothesis[b] = a.out.best_solution[b] = -1;
      a.out.num_hypotheses[b] = P.drawn;
    }
    return;
  }
  const unsigned hr = ~(unsigned)(key & 0xffffffffu);
  const int hcount = (int)(key >> 32) - 1;
  const float thr2 = P.thr2;
  if (t == 0) {
    int id[S];
    double Rs[SOLS][9], ts[SOLS][3], Pm[12];
    geo_sample(a.seed, hr >> 4, P.n, S, id);
    p3p(pts, wld, id, Rs, ts);
    for (int i = 0; i < 9; ++i) pose[0][i] = pose[1][i] = Rs[hr & 15][i];
    for (int i = 0; i < 3; ++i) pose[0][9 + i] = pose[1][9 + i] = ts[hr & 15][i];
    projection(K, pose[0], pose[0] + 9, Pm);
    for (int i = 0; i < 12; ++i) fm[0][i] = (float)Pm[i];
    count[0] = hcount;
    count[1] = -1;
  }
  __syncthreads();
  if (hcount >= GEO_PNP_REFIT_MIN) {
    uint8_t* inl = a.w.inl + (long)b * a.M;
    for (int k = t; k < P.n; k += RED) inl[k] = reproj_inlier(fm[0], pts[k], wld[k], thr2);
    __syncthreads();
    double acc[LM_TERMS];
    lm_partials(K, pose[1], pose[1] + 9, pts, wld, inl, P.n, t, acc);
    for (int i = 0; i < LM_TERMS; ++i) {
      const double s = tree_sum(acc[i], red, t);
      if (t == 0) sums[i] = s;
    }
    double lam = GEO_PNP_LM_LAMBDA0;  // every thread keeps the same schedule
    for (int it = 0; it < GEO_PNP_LM_STEPS; ++it) {
      if (t == 0) {
        double d[6];
        step_ok = lm_solve<6>(sums, sums + 21, lam, d);
        if (step_ok) lm_update(pose[1], pose[1] + 9, d, cand, cand + 9);
      }
      __syncthreads();
      if (!step_ok) {
        lam = lam * 10.0;
        __syncthreads();
        continue;
      }
      lm_partials(K, cand, cand + 9, pts, wld, inl, P.n, t, acc);
      for (int i = 0; i < LM_TERMS; ++i) {
        const double s = tree_sum(acc[i], red, t);
        if (t == 0) csum[i] = s;
      }
      __syncthreads();
      const bool better = csum[27] < sums[27];
      __syncthreads();
      if (better) {
        if (t < 12) pose[1][t] = cand[t];
        if (t < LM_TERMS) sums[t] = csum[t];
        lam = lam / 10.0;
      } else {
        lam = lam * 10.0;
      }
      __syncthreads();
    }
    if (t == 0) {
      double Pm[12];
      projection(K, pose[1], pose[1] + 9, Pm);
      for (int i = 0; i < 12; ++i) fm[1][i] = (float)Pm[i];
      count[1] = 0;
    }
    __syncthreads();
    int k1 = 0;
    for (int k = t; k < P.n; k += RED) k1 += reproj_inlier(fm[1], pts[k], wld[k], thr2);
    if (k1) atomicAdd(&count[1], k1);
    __syncthreads();
  }
  const int u = count[1] >= count[0] ? 1 : 0;
  if (t < 12) P.P[t] = fm[u][t];
  if (t < 9) a.out.R[(long)b * 9 + t] = pose[u][t];
  if (t < 3) a.out.t[(long)b * 3 + t] = pose[u][9 + t];
  if (t == 0) {
    a.out.num_inliers[b] = count[u];
    a.out.success[b] = 1;
    a.out.best_hypothesis[b] = (int)(hr >> 4);
    a.out.best_solution[b] = (int)(hr & 15);
    a.out.num_hypotheses[b] = P.drawn;
    P.success = 1;
  }
}

__global__ void __launch_bounds__(MASK_THREADS) pnp_mask_kernel(PnpArgs a) {
  const int b = blockIdx.x, i = blockIdx.y * MASK_THREADS + threadIdx.x;
  if (i >= a.M) return;
  const PnpPair& P = a.w.pair[b];
  const int k = a.w.slot[(long)b * a.M + i];
  bool in = false;
  if (P.success && k >= 0) in = reproj_inlier(P.P, a.w.pts[(long)b * a.M + k], a.w.wld[(long)b * a.M + k], P.thr2);
  a.out.inliers[(long)b * a.M + i] = in;
}

}  // namespace

extern "C" size_t geo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  PnpWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_absolute_pose(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoPnpOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_absolute_pose";
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, geo_no_check, geo_no_check);
  if (rc == GEO_RUN)
    rc = geo_check_buffers(entry, in, {out->R, out->t, out->num_inliers, out->success, out->best_hypothesis,
                                       out->best_solution, out->num_hypotheses}, {out->inliers}, {in->K0},
                           in->points3d1, workspace, workspace_bytes,
                           geo_pnp_workspace_bytes(in->B, in->M, cfg->max_iters));
  if (rc != GEO_RUN) return rc;
  PnpArgs a{};
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.threshold = cfg->threshold;
  a.confidence = cfg->confidence;
  a.kpts0 = in->kpts0; a.points3d1 = in->points3d1; a.matches0 = in->matches0;
  a.K0 = in->K0;
  a.out = *out;
  const int splits = geo_score_splits(a.B, a.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  pnp_prepare_kernel<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    pnp_hyp_kernel<<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<PnpScore><<<dim3(a.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  pnp_refit_kernel<<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  if (a.M > 0) {
    pnp_mask_kernel<<<dim3(a.B, (a.M + MASK_THREADS - 1) / MASK_THREADS), MASK_THREADS, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  return 0;
}
