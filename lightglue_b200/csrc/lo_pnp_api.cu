// Batched LO-RANSAC absolute pose on the matcher's 2D-3D matches: MSAC-scored Lambda Twist P3P sampling with
// Levenberg-Marquardt local optimisation of (R, t) and a final refinement (include/geometry_b200.h, steps LA1-LA8), on
// lo_common.cuh's schedule.  pnp_api.cu's compaction and calibration kernel prepares the pair; geo_hyp_kernel draws up
// to 4 P3P solutions as fp32 projections; a local optimisation starts from its solution re-solved in double and runs LM
// on the truncated reprojection cost; the final kernel writes the inlier mask of every row of matches0.  With lens
// distortion (geo_absolute_pose_lo_dist, steps AD1-AD4) PnpDistLo runs the same schedule in distorted pixels.  Compiled
// with -fmad=false: oracle/lo_pnp_oracle.py takes the same steps.
#include <stdint.h>

#include "lo_common.cuh"
#include "pnp_common.cuh"

namespace {

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

// The chunk's LA3 scores of every projection, count << 40 | MSAC score, on a tile of pixels and world points
struct LoPnpScore {
  using Args = LoArgs<PnpArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  __device__ LoPnpScore(const Args& a, const PnpPair& P, int b)
      : src{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M}, sums(a.l.acc), thr2(P.thr2),
        w((float)GEO_LO_QSCALE / P.thr2) {}
  __device__ unsigned long long term(const float* g, const float4* p) const {
    return lo_term(reproj_err(g, p[0], p[1]), thr2, w);
  }
};

// The absolute pose for lo_common.cuh's LM loop, re-score and schedule: x = R (0-8, row-major) and t (9-11); the
// pair's constants are its K0 (header step LA7)
struct PnpLo {
  static constexpr int DOF = 6, TERMS = 28, GROUP = 14, NP = 12, NF = 12, S = ::S, SOLS = ::SOLS;
  using Base = PnpArgs;
  using Args = LoArgs<PnpArgs>;
  using Solver = PnpSolver;
  using Score = LoPnpScore;
  struct Scratch {};

  // The TERMS sums at x: A7's Jacobian over the points in front of the camera with err < thr2, and the truncated cost
  static __device__ void terms(LoShared<PnpLo>& s, const double* K, const double* x, PnpPoints pts, int n, double thr2,
                               double* out, int tid) {
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const PnpResidual e = pnp_residual(K, x, x + 9, pts.pix[k], pts.wld[k]);
      const double err = e.ru * e.ru + e.rv * e.rv;
      const bool in = e.Xc[2] > 0.0 && err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (in) pnp_add_normal(K, e, acc);
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

  static __device__ PnpPoints points(const Args& a, int b) {
    return {a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M};
  }
  static __device__ const double* consts(const Args& a, int b) { return a.p.K0 + (long)b * 9; }
  static __device__ float thr2(const Args& a, int b) { return a.p.w.pair[b].thr2; }

  // LA4: sample h re-solved in double, as the score's projections were solved
  static __device__ void seed(LoShared<PnpLo>& s, const Args& a, int b, unsigned hr, long, LoPair& L, int t) {
    if (t == 0) {
      double x[SOLS][12];
      PnpSolver::solve(a.p, b, hr >> 4, x);
      for (int i = 0; i < 12; ++i) s.x[i] = L.model[i] = x[hr & 15][i];
    }
  }

  static __device__ void store(LoShared<PnpLo>& s, LoPair& L) {
    for (int i = 0; i < 12; ++i) L.model[i] = s.x[i];
  }

  static __device__ void load(LoShared<PnpLo>& s, const Args&, int, const LoPair& L, int t) {
    if (t < 12) s.x[t] = L.model[t];
  }

  static __device__ void restore(LoShared<PnpLo>& s, const Args& a, int b, const LoPair& L, int t) {
    if (t == 0) {
      for (int i = 0; i < 12; ++i) s.x[i] = L.model[i];
      projection(consts(a, b), L.model, L.model + 9, s.px);
      for (int i = 0; i < 12; ++i) s.fm[i] = (float)s.px[i];
      s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
    }
    __syncthreads();
  }

  static __device__ void fail(const Args& a, int b, int t) {
    if (t < 9) a.p.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.p.out.t[(long)b * 3 + t] = 0.0;
  }

  // LA8: A5's test per row of matches0, as pnp_mask_kernel
  static __device__ void write(LoShared<PnpLo>& s, const Args& a, int b, int t) {
    const PnpPoints pts = points(a, b);
    const int* slot = a.p.w.slot + (long)b * a.p.M;
    uint8_t* inl = a.p.out.inliers + (long)b * a.p.M;
    for (int i = t; i < a.p.M; i += RED) {
      const int k = slot[i];
      inl[i] = k >= 0 && reproj_inlier(s.fm, pts.pix[k], pts.wld[k], a.p.w.pair[b].thr2);
    }
    if (t < 9) a.p.out.R[(long)b * 9 + t] = s.x[t];
    if (t < 3) a.p.out.t[(long)b * 3 + t] = s.x[9 + t];
  }
};

// ---- with lens distortion (header steps AD1-AD4 on LA1-LA8) ----

// One compacted point and the pair's camera for AD2's test
struct PnpDistPoint {
  float4 p, q;
  const Camera<float>* cam;
};

struct PnpDistPoints {
  const float4* pix;
  const float4* wld;
  Camera<float> cam;
  __device__ __forceinline__ PnpDistPoint operator[](int k) const { return {pix[k], wld[k], &cam}; }
};

// LoPnpScore with AD2's error of every [R | t]
struct LoPnpDistScore {
  using Args = LoArgs<PnpDistArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  Camera<float> cam;
  __device__ LoPnpDistScore(const Args& a, const PnpPair& P, int b)
      : src{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M}, sums(a.l.acc), thr2(P.thr2),
        w((float)GEO_LO_QSCALE / P.thr2), cam(pair_camera<float>(a.p, b)) {}
  __device__ unsigned long long term(const float* g, const float4* p) const {
    return lo_term(dist_reproj_err(g, cam, p[0], p[1]), thr2, w);
  }
};

// PnpLo with AD2's error and AD3's residuals: x = R (0-8, row-major) and t (9-11), scored as [R | t]; the pair's
// constants are its camera in double
struct PnpDistLo {
  static constexpr int DOF = 6, TERMS = 28, GROUP = 14, NP = 12, NF = 12, S = ::S, SOLS = ::SOLS;
  using Base = PnpDistArgs;
  using Args = LoArgs<PnpDistArgs>;
  using Solver = PnpDistSolver;
  using Score = LoPnpDistScore;
  struct Scratch {};

  static __device__ void terms(LoShared<PnpDistLo>& s, const Camera<double>& c, const double* x,
                               const PnpDistPoints& pts, int n, double thr2, double* out, int tid) {
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const PnpDistResidual e = pnp_dist_residual(c, x, x + 9, pts.pix[k], pts.wld[k]);
      const double err = e.ru * e.ru + e.rv * e.rv;
      const bool in = e.Xc[2] > 0.0 && err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (in) pnp_dist_add_normal(c, e, acc);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  static __device__ void update(LoShared<PnpDistLo>&, const double* x, const double* d, double* out) {
    lm_update(x, x + 9, d, out, out + 9);
  }

  static __device__ void pixels(LoShared<PnpDistLo>&, const Camera<double>&, const double* x, double* out) {
    rt_matrix(x, out);
  }

  static __device__ __forceinline__ float err(const float* g, PnpDistPoint pt) {
    return dist_reproj_err(g, *pt.cam, pt.p, pt.q);
  }

  static __device__ PnpDistPoints points(const Args& a, int b) {
    return {a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M, pair_camera<float>(a.p, b)};
  }
  static __device__ Camera<double> consts(const Args& a, int b) { return pair_camera<double>(a.p, b); }
  static __device__ float thr2(const Args& a, int b) { return a.p.w.pair[b].thr2; }

  static __device__ void seed(LoShared<PnpDistLo>& s, const Args& a, int b, unsigned hr, long, LoPair& L, int t) {
    if (t == 0) {
      double x[SOLS][12];
      PnpDistSolver::solve(a.p, b, hr >> 4, x);
      for (int i = 0; i < 12; ++i) s.x[i] = L.model[i] = x[hr & 15][i];
    }
  }

  static __device__ void store(LoShared<PnpDistLo>& s, LoPair& L) {
    for (int i = 0; i < 12; ++i) L.model[i] = s.x[i];
  }

  static __device__ void load(LoShared<PnpDistLo>& s, const Args&, int, const LoPair& L, int t) {
    if (t < 12) s.x[t] = L.model[t];
  }

  static __device__ void restore(LoShared<PnpDistLo>& s, const Args&, int, const LoPair& L, int t) {
    if (t == 0) {
      for (int i = 0; i < 12; ++i) s.x[i] = L.model[i];
      rt_matrix(L.model, s.px);
      for (int i = 0; i < 12; ++i) s.fm[i] = (float)s.px[i];
      s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
    }
    __syncthreads();
  }

  static __device__ void fail(const Args& a, int b, int t) {
    if (t < 9) a.p.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.p.out.t[(long)b * 3 + t] = 0.0;
  }

  // AD4: AD2's test per row of matches0
  static __device__ void write(LoShared<PnpDistLo>& s, const Args& a, int b, int t) {
    const PnpDistPoints pts = points(a, b);
    const int* slot = a.p.w.slot + (long)b * a.p.M;
    uint8_t* inl = a.p.out.inliers + (long)b * a.p.M;
    for (int i = t; i < a.p.M; i += RED) {
      const int k = slot[i];
      inl[i] = k >= 0 && err(s.fm, pts[k]) < a.p.w.pair[b].thr2;
    }
    if (t < 9) a.p.out.R[(long)b * 9 + t] = s.x[t];
    if (t < 3) a.p.out.t[(long)b * 3 + t] = s.x[9 + t];
  }
};

}  // namespace

extern "C" size_t geo_lo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lo_workspace_bytes<PnpLo>(B, M);
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
  PnpArgs p = pnp_args(cfg, in);
  p.out = out->pnp;
  return lo_launch<PnpLo>(p, out->num_local_optimizations, out->cost, workspace, pnp_prepare_kernel, stream_);
}

extern "C" int geo_absolute_pose_lo_dist(const GeoPnpConfig* cfg, const GeoPnpDistInputs* din, GeoLoPnpOutputs* out,
                                         void* workspace, size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_absolute_pose_lo_dist";
  const GeoPnpInputs* in = din ? &din->pnp : nullptr;
  int rc = geo_check_config(entry, cfg, in, out, GEO_LO_MAX_MATCHES, geo_no_check,
                            [&] { return dist_count_check(din->num_dist); });
  if (rc == GEO_RUN) {
    const GeoPnpOutputs& o = out->pnp;
    rc = geo_check_buffers(entry, in, {o.R, o.t, o.num_inliers, o.success, o.best_hypothesis, o.best_solution,
                                       o.num_hypotheses, out->num_local_optimizations, out->cost}, {o.inliers},
                           {in->K0, din->dist0}, in->points3d1, workspace, workspace_bytes,
                           geo_lo_pnp_workspace_bytes(in->B, in->M, cfg->max_iters));
  }
  if (rc != GEO_RUN) return rc;
  PnpDistArgs p{pnp_args(cfg, in), din->dist0, din->num_dist};
  p.out = out->pnp;
  return lo_launch<PnpDistLo>(p, out->num_local_optimizations, out->cost, workspace, pnp_dist_prepare_kernel, stream_);
}
