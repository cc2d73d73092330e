// Batched LO-RANSAC absolute pose on the matcher's 2D-3D matches: MSAC-scored Lambda Twist P3P sampling with
// Levenberg-Marquardt local optimisation of (R, t) and a final refinement (include/geometry_b200.h, steps LA1-LA8), on
// lo_common.cuh's schedule.  pnp_common.cuh's compaction and calibration kernel prepares the pair; geo_hyp_kernel draws
// up to 4 P3P solutions as fp32 models; a local optimisation starts from its solution re-solved in double and runs LM
// on the truncated reprojection cost; the final kernel writes the inlier mask of every row of matches0.  Every piece is
// a template on pnp_common.cuh's camera policy: PnpLo<Pinhole> for geo_absolute_pose_lo, PnpLo<Distorted> for
// geo_absolute_pose_lo_dist (steps AD1-AD4, in distorted pixels), PnpLo<Fisheye> for geo_absolute_pose_lo_fisheye
// (AE1-AE4, in fisheye pixels).  Compiled with -fmad=false:
// oracle/lo_pnp_oracle.py takes the same steps.
#include <stdint.h>

#include "lo_common.cuh"
#include "pnp_common.cuh"

namespace {

// One compacted point: its pixel (u, v, x, y), world point (X, Y, Z, 0) and the pair's fp32 test state
template <class Cam>
struct PnpPoint {
  float4 p, q;
  const typename Cam::Test* cam;
};

// A pair's compacted points as lo_common.cuh's LM loop and re-score read them
template <class Cam>
struct PnpPoints {
  const float4* pix;
  const float4* wld;
  typename Cam::Test cam;
  __device__ __forceinline__ PnpPoint<Cam> operator[](int k) const { return {pix[k], wld[k], &cam}; }
};

// The chunk's LA3 scores of every model, count << 40 | MSAC score, on a tile of pixels and world points
template <class Cam>
struct LoPnpScore {
  using Args = LoArgs<PnpArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  typename Cam::Test cam;
  __device__ LoPnpScore(const Args& a, const PnpPair& P, int b)
      : src{a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M}, sums(a.l.acc), thr2(P.thr2),
        w((float)GEO_LO_QSCALE / P.thr2), cam(Cam::test(a.p, b)) {}
  __device__ unsigned long long term(const float* g, const float4* p) const {
    return lo_term(Cam::err(cam, g, p[0], p[1]), thr2, w);
  }
};

// The absolute pose for lo_common.cuh's LM loop, re-score and schedule: x = R (0-8, row-major) and t (9-11); the
// pair's constants are Cam's (header step LA7)
template <class Cam>
struct PnpLo {
  static constexpr int DOF = 6, TERMS = 28, GROUP = 14, NP = 12, NF = 12, S = ::S, SOLS = ::SOLS;
  using Base = PnpArgs;
  using Args = LoArgs<PnpArgs>;
  using Solver = PnpSolver<Cam>;
  using Score = LoPnpScore<Cam>;
  struct Scratch {};

  // The TERMS sums at x: A7's Jacobian over the points in front of the camera with err < thr2, and the truncated cost
  static __device__ void terms(LoShared<PnpLo>& s, const typename Cam::Consts& c, const double* x,
                               const PnpPoints<Cam>& pts, int n, double thr2, double* out, int tid) {
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const auto e = Cam::residual(c, x, pts.pix[k], pts.wld[k]);
      const double err = e.ru * e.ru + e.rv * e.rv;
      const bool in = e.Xc[2] > 0.0 && err < thr2;
      acc[TERMS - 1] = acc[TERMS - 1] + (in ? err : thr2);
      if (in) Cam::add_normal(c, e, acc);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // R' = Q R, t' = Q t + d3..5 (A7's step)
  static __device__ void update(LoShared<PnpLo>&, const double* x, const double* d, double* out) {
    lm_update(x, x + 9, d, out, out + 9);
  }

  // Cam's scored model of x (A5, AD2)
  static __device__ void pixels(LoShared<PnpLo>&, const typename Cam::Consts& c, const double* x, double* out) {
    Cam::model(c, x, out);
  }

  static __device__ __forceinline__ float err(const float* g, PnpPoint<Cam> pt) {
    return Cam::err(*pt.cam, g, pt.p, pt.q);
  }

  static __device__ PnpPoints<Cam> points(const Args& a, int b) {
    return {a.p.w.pts + (long)b * a.p.M, a.p.w.wld + (long)b * a.p.M, Cam::test(a.p, b)};
  }
  static __device__ typename Cam::Consts consts(const Args& a, int b) { return Cam::consts(a.p, b); }
  static __device__ Msac loss(const Args& a, int b) { return {a.p.w.pair[b].thr2}; }

  // LA4: sample h re-solved in double, as the score's models were solved
  static __device__ void seed(LoShared<PnpLo>& s, const Args& a, int b, unsigned hr, long, LoPair& L, int t) {
    if (t == 0) {
      double x[SOLS][12];
      Solver::solve(a.p, b, hr >> 4, x);
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
      Cam::model(consts(a, b), L.model, s.px);
      for (int i = 0; i < 12; ++i) s.fm[i] = (float)s.px[i];
      s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
    }
    __syncthreads();
  }

  static __device__ void fail(const Args& a, int b, int t) {
    if (t < 9) a.p.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.p.out.t[(long)b * 3 + t] = 0.0;
  }

  // LA8 (and AD4): the fp32 test per row of matches0, as pnp_mask_kernel
  static __device__ void write(LoShared<PnpLo>& s, const Args& a, int b, int t) {
    const PnpPoints<Cam> pts = points(a, b);
    const int* slot = a.p.w.slot + (long)b * a.p.M;
    uint8_t* inl = a.p.out.inliers + (long)b * a.p.M;
    for (int i = t; i < a.p.M; i += RED) {
      const int k = slot[i];
      inl[i] = k >= 0 && Cam::inlier(pts.cam, s.fm, pts.pix[k], pts.wld[k], a.p.w.pair[b].thr2);
    }
    if (t < 9) a.p.out.R[(long)b * 9 + t] = s.x[t];
    if (t < 3) a.p.out.t[(long)b * 3 + t] = s.x[9 + t];
  }
};

// geo_absolute_pose_lo, geo_absolute_pose_lo_dist and geo_absolute_pose_lo_fisheye: the checks, then the launches
template <class Cam>
int absolute_pose(const char* entry, const GeoPnpConfig* cfg, const GeoPnpInputs* in, const double* dist0,
                  int num_dist, GeoLoPnpOutputs* out, void* workspace, size_t workspace_bytes, void* stream_) {
  int rc = geo_check_config(entry, cfg, in, out, GEO_LO_MAX_MATCHES, geo_no_check,
                            [&] { return Cam::count_check(num_dist); });
  if (rc == GEO_RUN) {
    const GeoPnpOutputs& o = out->pnp;
    const auto buffers = [&](std::initializer_list<const void*> intrinsics) {
      return geo_check_buffers(entry, in, {o.R, o.t, o.num_inliers, o.success, o.best_hypothesis, o.best_solution,
                                           o.num_hypotheses, out->num_local_optimizations, out->cost}, {o.inliers},
                               intrinsics, in->points3d1, workspace, workspace_bytes,
                               geo_lo_pnp_workspace_bytes(in->B, in->M, cfg->max_iters));
    };
    rc = Cam::COEFFS ? buffers({in->K0, dist0}) : buffers({in->K0});
  }
  if (rc != GEO_RUN) return rc;
  PnpArgs p = pnp_args(cfg, in, dist0, num_dist);
  p.out = out->pnp;
  return lo_launch<PnpLo<Cam>>(p, out->num_local_optimizations, out->cost, workspace, pnp_prepare_kernel<Cam>, stream_);
}

}  // namespace

extern "C" size_t geo_lo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lo_workspace_bytes<PnpLo<Pinhole>>(B, M);
}

extern "C" int geo_absolute_pose_lo(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoLoPnpOutputs* out,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  return absolute_pose<Pinhole>("geo_absolute_pose_lo", cfg, in, nullptr, 0, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_absolute_pose_lo_dist(const GeoPnpConfig* cfg, const GeoPnpDistInputs* din, GeoLoPnpOutputs* out,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  // a null din goes on as a null in, which geo_check_config reports
  return absolute_pose<Distorted>("geo_absolute_pose_lo_dist", cfg, din ? &din->pnp : nullptr,
                                  din ? din->dist0 : nullptr, din ? din->num_dist : 0, out, workspace, workspace_bytes,
                                  stream);
}

extern "C" int geo_absolute_pose_lo_fisheye(const GeoPnpConfig* cfg, const GeoPnpDistInputs* din,
                                            GeoLoPnpOutputs* out, void* workspace, size_t workspace_bytes,
                                            void* stream) {
  return absolute_pose<Fisheye>("geo_absolute_pose_lo_fisheye", cfg, din ? &din->pnp : nullptr,
                                din ? din->dist0 : nullptr, din ? din->num_dist : 0, out, workspace, workspace_bytes,
                                stream);
}
