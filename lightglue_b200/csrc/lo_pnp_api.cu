// Batched LO-RANSAC absolute pose on the matcher's 2D-3D matches: MSAC-scored Lambda Twist P3P sampling with
// Levenberg-Marquardt local optimisation of (R, t) and a final refinement (include/geometry_b200.h, steps LA1-LA8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  pnp_api.cu's compaction and calibration kernel (pnp_common.cuh)
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair, one thread per sample: up to 4 P3P solutions as fp32 projections
//     score  (B, splits) CTAs: each streams a slice of the pair's pixels and world points through shared memory against
//            every solution of the chunk, one thread per sample, and adds count << 40 | MSAC score with one 64-bit
//            atomic per solution
//     lo     one CTA per pair: the chunk's lowest (score, h, r); when it beats the pair's model, the solution re-solved
//            in double, LM on the truncated reprojection cost and a re-score; then the adaptive stop.  Otherwise it
//            only decides the stop.
//   final    one CTA per pair: the final LM refinement, R, t and the inlier mask of every row of matches0
// A stopped pair's CTAs return at once.  Compiled with -fmad=false: oracle/lo_pnp_oracle.py takes the same steps.
#include <stdint.h>

#include "lo_common.cuh"
#include "pnp_common.cuh"

namespace {

struct LoPnpPair {
  double R[9], t[3];         // the pair's model
  unsigned long long score;  // its LA3 score
  int count;                 // its inliers
  int hr;                    // h * 16 + r of the solution that seeded it; -1: none yet
  int nlo;                   // local optimisations adopted
};

struct LoPnpWs {
  LoPnpPair* pair;          // [B]
  unsigned long long* acc;  // [B, GEO_CHUNK, SOLS] count << 40 | score of the current chunk's solutions
};

size_t lopnp_carve(char* base, int B, int M, PnpWs* w, LoPnpWs* l) {
  WsBump b{base, carve(base, B, M, w)};
  l->pair = b.take<LoPnpPair>(B);
  l->acc = b.take<unsigned long long>((size_t)B * GEO_CHUNK * SOLS);
  return b.bytes();
}

struct LoPnpArgs {
  PnpArgs p;
  LoPnpWs l;
  int32_t* num_lo;
  int64_t* cost;
};

// One compacted point: its pixel (u, v, x, y) and world point (X, Y, Z, 0)
struct PnpPoint {
  float4 p, q;
};

// A pair's compacted points as lo_common.cuh's LM loop and re-score read them
struct PnpPoints {
  const float4* pix;
  const float4* wld;
  __device__ __forceinline__ PnpPoint operator[](int k) const { return {pix[k], wld[k]}; }
};

// The absolute pose for lo_common.cuh's LM loop and re-score: x = R (0-8, row-major) and t (9-11); the pair's
// constants are its K0 (header step LA7)
struct PnpLo {
  static constexpr int DOF = 6, TERMS = 28, GROUP = 14, NP = 12, NF = 12;
  struct Scratch {};

  // The TERMS sums at x: A7's Jacobian over the points in front of the camera with err < thr2, and the truncated cost
  static __device__ void terms(LoShared<PnpLo>& s, const double* K, const double* x, PnpPoints pts, int n, double thr2,
                               double* out, int tid) {
    const double fx = K[0], sk = K[1], cx = K[2], fy = K[4], cy = K[5];
    const double* R = x;
    const double* t = x + 9;
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts.pix[k], q = pts.wld[k];
      const double u = p.x, v = p.y, W[3] = {q.x, q.y, q.z};
      double Xc[3];
      for (int i = 0; i < 3; ++i) Xc[i] = R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i];
      const double iz = 1.0 / Xc[2];
      const double ax = Xc[0] * iz, bx = Xc[1] * iz;
      const double pu = fx * ax + sk * bx;
      const double ru = pu + cx - u, rv = fy * bx + cy - v;
      const double err = ru * ru + rv * rv;
      const bool in = Xc[2] > 0.0 && err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (!in) continue;
      const double gu[3] = {fx * iz, sk * iz, -(pu * iz)};
      const double gv[3] = {0.0, fy * iz, -(fy * bx * iz)};
      const double ju[6] = {gu[2] * Xc[1] - gu[1] * Xc[2], gu[0] * Xc[2] - gu[2] * Xc[0], gu[1] * Xc[0] - gu[0] * Xc[1],
                            gu[0], gu[1], gu[2]};
      const double jv[6] = {gv[2] * Xc[1] - gv[1] * Xc[2], gv[0] * Xc[2] - gv[2] * Xc[0], gv[1] * Xc[0] - gv[0] * Xc[1],
                            gv[0], gv[1], gv[2]};
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + (ju[i] * ju[j] + jv[i] * jv[j]);
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[21 + i] = acc[21 + i] + (ju[i] * ru + jv[i] * rv);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // R' = Q R, t' = Q t + d3..5 (A7's step)
  static __device__ void update(LoShared<PnpLo>&, const double* x, const double* d, double* out) {
    lm_update(x, x + 9, d, out, out + 9);
  }

  // P = K0 [R | t] (A5)
  static __device__ void pixels(LoShared<PnpLo>&, const double* K, const double* x, double* out) {
    projection(K, x, x + 9, out);
  }

  static __device__ __forceinline__ float err(const float* g, PnpPoint pt) { return reproj_err(g, pt.p, pt.q); }
};

__global__ void __launch_bounds__(GEO_CHUNK, 1) lopnp_hyp_kernel(LoPnpArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c == 0 && t == 0) {
    LoPnpPair& L = a.l.pair[b];
    L.score = 0;
    L.count = 0;
    L.hr = -1;
    L.nlo = 0;
  }
  const PnpPair& P = a.p.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  int ns = 0;
  int id[S];
  if (P.stop == 0 && h < a.p.max_iters && geo_sample(a.p.seed, h, P.n, S, id) == S) {
    double Rs[SOLS][9], ts[SOLS][3];
    ns = p3p(a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M, id, Rs, ts);
    const double* K = a.p.K0 + (long)b * 9;
    float* hm = a.p.w.hyp + ((long)b * GEO_CHUNK + t) * SOLS * 12;
    for (int r = 0; r < ns; ++r) {
      double Pm[12];
      projection(K, Rs[r], ts[r], Pm);
      for (int i = 0; i < 12; ++i) hm[r * 12 + i] = (float)Pm[i];
      a.l.acc[((long)b * GEO_CHUNK + t) * SOLS + r] = 0;
    }
  }
  a.p.w.nsol[(long)b * GEO_CHUNK + t] = ns;
}

// The chunk's LA3 scores of every projection, count << 40 | MSAC score, on a tile of pixels and world points
struct LoPnpScore {
  using Args = LoPnpArgs;
  using Acc = unsigned long long;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const LoPnpArgs& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  __device__ LoPnpScore(const LoPnpArgs& a, const PnpPair& P, int b)
      : src{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M}, sums(a.l.acc), thr2(P.thr2),
        w((float)GEO_LO_QSCALE / P.thr2) {}
  __device__ unsigned long long term(const float* g, const float4* p) const {
    return lo_term(reproj_err(g, p[0], p[1]), thr2, w);
  }
};

// After chunk c: the chunk's best solution, the local optimisation when it beats the pair's model, the stop
__global__ void __launch_bounds__(RED, 1) lopnp_lo_kernel(LoPnpArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  PnpPair& P = a.p.w.pair[b];
  if (P.stop) return;
  LoPnpPair& L = a.l.pair[b];
  __shared__ LoShared<PnpLo> s;
  if (t == 0) s.key = ~0ull;
  __syncthreads();
  if (t < GEO_CHUNK) {
    const int ns = a.p.w.nsol[(long)b * GEO_CHUNK + t];
    const unsigned h = c * GEO_CHUNK + t;
    for (int r = 0; r < ns; ++r) {
      const unsigned long long v = a.l.acc[((long)b * GEO_CHUNK + t) * SOLS + r];
      atomicMin(&s.key, (v & LO_SCORE_MASK) << 28 | (h * 16u + (unsigned)r));
    }
  }
  __syncthreads();
  const unsigned long long key = s.key;
  const PnpPoints pts{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M};
  const double* K = a.p.K0 + (long)b * 9;
  if (t == 0) s.take = key != ~0ull && (L.hr < 0 || (key >> 28) < L.score);
  __syncthreads();
  if (s.take) {
    if (t == 0) {  // LA4: re-solve sample h in double, as the score's projections were solved
      const unsigned hr = (unsigned)(key & 0xfffffffu);
      int id[S];
      double Rs[SOLS][9], ts[SOLS][3];
      geo_sample(a.p.seed, hr >> 4, P.n, S, id);
      p3p(pts.pix, pts.wld, id, Rs, ts);
      for (int i = 0; i < 9; ++i) s.x[i] = L.R[i] = Rs[hr & 15][i];
      for (int i = 0; i < 3; ++i) s.x[9 + i] = L.t[i] = ts[hr & 15][i];
      L.score = key >> 28;
      L.count = (int)(a.l.acc[((long)b * GEO_CHUNK + (hr >> 4) - c * GEO_CHUNK) * SOLS + (hr & 15)] >> 40);
      L.hr = (int)hr;
    }
    __syncthreads();
    lo_refine(s, K, pts, P.n, (double)P.thr2, GEO_LO_STEPS, t);
    lo_rescore(s, K, pts, P.n, P.thr2, t);
    if (t == 0 && (s.score & LO_SCORE_MASK) < L.score) {
      for (int i = 0; i < 9; ++i) L.R[i] = s.x[i];
      for (int i = 0; i < 3; ++i) L.t[i] = s.x[9 + i];
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
             drawn >= update_num_iters(a.p.confidence, 1.0 - (double)cnt / P.n, S, a.p.max_iters);
  }
}

// Final refinement and the outputs (header steps LA6 and LA8)
__global__ void __launch_bounds__(RED, 1) lopnp_final_kernel(LoPnpArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  const PnpPair& P = a.p.w.pair[b];
  const LoPnpPair& L = a.l.pair[b];
  const GeoPnpOutputs& o = a.p.out;
  uint8_t* inl = o.inliers + (long)b * a.p.M;
  if (!P.ok || L.hr < 0) {
    for (int i = t; i < a.p.M; i += RED) inl[i] = 0;
    if (t < 9) o.R[(long)b * 9 + t] = 0.0;
    if (t < 3) o.t[(long)b * 3 + t] = 0.0;
    if (t == 0) {
      o.num_inliers[b] = 0;
      o.success[b] = 0;
      o.best_hypothesis[b] = o.best_solution[b] = -1;
      o.num_hypotheses[b] = P.drawn;
      a.num_lo[b] = 0;
      a.cost[b] = 0;
    }
    return;
  }
  __shared__ LoShared<PnpLo> s;
  const PnpPoints pts{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M};
  const double* K = a.p.K0 + (long)b * 9;
  if (t < 9) s.x[t] = L.R[t];
  if (t < 3) s.x[9 + t] = L.t[t];
  __syncthreads();
  lo_refine(s, K, pts, P.n, (double)P.thr2, GEO_LO_FINAL_STEPS, t);
  lo_rescore(s, K, pts, P.n, P.thr2, t);
  if (t == 0 && (s.score & LO_SCORE_MASK) > L.score) {  // the refinement is kept unless its score rises
    for (int i = 0; i < 9; ++i) s.x[i] = L.R[i];
    for (int i = 0; i < 3; ++i) s.x[9 + i] = L.t[i];
    projection(K, L.R, L.t, s.px);
    for (int i = 0; i < 12; ++i) s.fm[i] = (float)s.px[i];
    s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
  }
  __syncthreads();
  const int* slot = a.p.w.slot + (long)b * a.p.M;
  for (int i = t; i < a.p.M; i += RED) {  // A5's test per row of matches0, as pnp_mask_kernel
    const int k = slot[i];
    inl[i] = k >= 0 && reproj_inlier(s.fm, pts.pix[k], pts.wld[k], P.thr2);
  }
  if (t < 9) o.R[(long)b * 9 + t] = s.x[t];
  if (t < 3) o.t[(long)b * 3 + t] = s.x[9 + t];
  if (t == 0) {
    o.num_inliers[b] = (int)(s.score >> 40);
    o.success[b] = 1;
    o.best_hypothesis[b] = L.hr >> 4;
    o.best_solution[b] = L.hr & 15;
    o.num_hypotheses[b] = P.drawn;
    a.num_lo[b] = L.nlo;
    a.cost[b] = (int64_t)(s.score & LO_SCORE_MASK);
  }
}

}  // namespace

extern "C" size_t geo_lo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  PnpWs w;
  LoPnpWs l;
  return lopnp_carve(nullptr, B, M, &w, &l) + 256;
}

extern "C" int geo_absolute_pose_lo(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoLoPnpOutputs* out,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_absolute_pose_lo";
  int rc = geo_check_config(entry, cfg, in, out, GEO_LO_MAX_MATCHES, geo_no_check, geo_no_check);
  if (rc == GEO_RUN) {
    const GeoPnpOutputs& o = out->pnp;
    rc = geo_check_buffers(entry, in, {o.R, o.t, o.num_inliers, o.success, o.best_hypothesis, o.best_solution,
                                       o.num_hypotheses, out->num_local_optimizations, out->cost}, {o.inliers},
                           {in->K0}, in->points3d1, workspace, workspace_bytes,
                           geo_lo_pnp_workspace_bytes(in->B, in->M, cfg->max_iters));
  }
  if (rc != GEO_RUN) return rc;
  LoPnpArgs a{};
  lopnp_carve(geo_workspace_base(workspace), in->B, in->M, &a.p.w, &a.l);
  PnpArgs& p = a.p;
  p.B = in->B; p.M = in->M; p.N = in->N;
  p.max_iters = cfg->max_iters;
  p.chunks = geo_chunks(cfg->max_iters);
  p.seed = cfg->seed;
  p.threshold = cfg->threshold;
  p.confidence = cfg->confidence;
  p.kpts0 = in->kpts0; p.points3d1 = in->points3d1; p.matches0 = in->matches0;
  p.K0 = in->K0;
  p.out = out->pnp;
  a.num_lo = out->num_local_optimizations;
  a.cost = out->cost;
  const int splits = geo_score_splits(p.B, p.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  pnp_prepare_kernel<<<p.B, 1024, 0, stream>>>(p);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < p.chunks; ++c) {
    lopnp_hyp_kernel<<<p.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<LoPnpScore><<<dim3(p.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
    lopnp_lo_kernel<<<p.B, RED, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
  }
  lopnp_final_kernel<<<p.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
