// Batched absolute pose on the matcher's 2D-3D matches: Lambda Twist P3P RANSAC, then Levenberg-Marquardt on the
// inliers (include/geometry_b200.h, steps A1-A8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  pnp_prepare_kernel<Cam>, one 1024-thread CTA per pair: ordered compaction of the valid matches,
//            calibrated coordinates, camera check
//   per chunk of GEO_CHUNK samples:
//     hyp    geo_hyp_kernel, one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold),
//            decides the adaptive stop, then one thread per sample solves it: up to 4 fp32 models
//     score  geo_score_kernel<PnpScore<Cam>>, (B, splits) CTAs: each streams a slice of the pair's points through
//            shared memory against every solution of the chunk, one thread per sample, and adds the inlier counts
//   final    geo_final_kernel<PnpRansac<Cam>>, one CTA per pair: folds the last chunk, Levenberg-Marquardt from the
//            best solution (lo_common.cuh's loop), recount, R and t
//   mask     pnp_mask_kernel<Cam>, one thread per row of matches0: the final inlier mask
// A stopped pair's CTAs return at once.  Cam is pnp_common.cuh's camera policy: Pinhole for geo_absolute_pose (the
// float model is K0 [R | t]), Distorted for geo_absolute_pose_dist (steps AD1-AD4: D2's calibrated coordinates, the
// float model [R | t] and the test in distorted pixels), Fisheye for geo_absolute_pose_fisheye (AE1-AE4: FE3's
// calibrated coordinates, which may drop a match, and the test in fisheye pixels).  Compiled with -fmad=false, like geo_api.cu:
// oracle/pnp_oracle.py takes the same steps in numpy.
#include <stdint.h>

#include "lo_common.cuh"
#include "pnp_common.cuh"

namespace {

constexpr int MASK_THREADS = 256;

// Inlier counts of every model, on a tile of pixels and world points
template <class Cam>
struct PnpScore {
  using Args = PnpArgs;
  using Acc = int;
  static constexpr int SOLS = ::SOLS, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const PnpWs& ws(const PnpArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  float thr2;
  typename Cam::Test cam;
  __device__ PnpScore(const PnpArgs& a, const PnpPair& P, int b)
      : src{a.w.pts + (long)b * a.M, a.w.wld + (long)b * a.M}, sums(a.w.count), thr2(P.thr2), cam(Cam::test(a, b)) {}
  __device__ int term(const float* g, const float4* p) const { return Cam::inlier(cam, g, p[0], p[1], thr2); }
};

// The points of the refinement and its fixed inlier set: those of the float model fm (header step A7)
template <class Cam>
struct PnpFixed {
  const float4* pix;
  const float4* wld;
  const float* fm;
  typename Cam::Test cam;
};

// (R, t) for lo_common.cuh's LM loop on A7's fixed inliers: x = R (0-8, row-major) and t (9-11); the pair's constants
// are Cam's
template <class Cam>
struct PnpLm {
  static constexpr int DOF = 6, TERMS = 28, GROUP = 14, NP = 12, NF = 12;
  struct Scratch {};

  static __device__ void terms(LoShared<PnpLm>& s, const typename Cam::Consts& c, const double* x,
                               const PnpFixed<Cam>& pts, int n, double thr2, double* out, int tid) {
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts.pix[k], q = pts.wld[k];
      if (!Cam::inlier(pts.cam, pts.fm, p, q, (float)thr2)) continue;
      const auto e = Cam::residual(c, x, p, q);
      Cam::add_normal(c, e, acc);
      acc[TERMS - 1] = acc[TERMS - 1] + (e.ru * e.ru + e.rv * e.rv);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  static __device__ void update(LoShared<PnpLm>&, const double* x, const double* d, double* out) {
    lm_update(x, x + 9, d, out, out + 9);
  }
};

// The absolute pose for geo_final_kernel: GEO_PNP_LM_STEPS Levenberg-Marquardt steps on the best solution's inliers
// (header step A7)
template <class Cam>
struct PnpRansac : PnpSolver<Cam> {
  using Base = PnpArgs;
  using Score = PnpScore<Cam>;
  using Scratch = LoShared<PnpLm<Cam>>;

  static __device__ bool inlier(const PnpArgs& a, int b, const float* g, int k) {
    const long i = (long)b * a.M + k;
    return Cam::inlier(Cam::test(a, b), g, a.w.pts[i], a.w.wld[i], a.w.pair[b].thr2);
  }
  static __device__ void clear(const PnpArgs&, int, int) {}  // pnp_mask_kernel writes every row
  static __device__ void fail(const PnpArgs& a, int b, int t) {
    if (t < 9) a.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.out.t[(long)b * 3 + t] = 0.0;
  }
  static __device__ bool refits(const PnpArgs&, int hcount) { return hcount >= GEO_PNP_REFIT_MIN; }

  static __device__ void refit(GeoFinal<PnpRansac>& s, const PnpArgs& a, int b, int t) {
    if (t == 0)
      for (int i = 0; i < 12; ++i) s.m.x[i] = s.x[0][i];
    __syncthreads();
    const PnpFixed<Cam> pts{a.w.pts + (long)b * a.M, a.w.wld + (long)b * a.M, s.fm[0], Cam::test(a, b)};
    const float thr2 = a.w.pair[b].thr2;
    lo_refine(s.m, Cam::consts(a, b), pts, a.w.pair[b].n, (double)thr2, GEO_PNP_LM_STEPS, GEO_PNP_LM_LAMBDA0, t);
    if (t == 0)
      for (int i = 0; i < 12; ++i) s.x[1][i] = s.m.x[i];
  }

  // R, t, and the float model for pnp_mask_kernel
  static __device__ void write(GeoFinal<PnpRansac>& s, const PnpArgs& a, int b, int u, int t) {
    PnpPair& P = a.w.pair[b];
    if (t < 12) P.P[t] = s.fm[u][t];
    if (t < 9) a.out.R[(long)b * 9 + t] = s.x[u][t];
    if (t < 3) a.out.t[(long)b * 3 + t] = s.x[u][9 + t];
    if (t == 0) P.success = 1;
  }
};

template <class Cam>
__global__ void __launch_bounds__(MASK_THREADS) pnp_mask_kernel(PnpArgs a) {
  const int b = blockIdx.x, i = blockIdx.y * MASK_THREADS + threadIdx.x;
  if (i >= a.M) return;
  const PnpPair& P = a.w.pair[b];
  const int k = a.w.slot[(long)b * a.M + i];
  bool in = false;
  if (P.success && k >= 0)
    in = Cam::inlier(Cam::test(a, b), P.P, a.w.pts[(long)b * a.M + k], a.w.wld[(long)b * a.M + k], P.thr2);
  a.out.inliers[(long)b * a.M + i] = in;
}

// geo_absolute_pose, geo_absolute_pose_dist and geo_absolute_pose_fisheye: the checks, then the launches
template <class Cam>
int absolute_pose(const char* entry, const GeoPnpConfig* cfg, const GeoPnpInputs* in, const double* dist0,
                  int num_dist, GeoPnpOutputs* out, void* workspace, size_t workspace_bytes, void* stream_) {
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, geo_no_check,
                            [&] { return Cam::count_check(num_dist); });
  if (rc == GEO_RUN) {
    const auto buffers = [&](std::initializer_list<const void*> intrinsics) {
      return geo_check_buffers(entry, in, {out->R, out->t, out->num_inliers, out->success, out->best_hypothesis,
                                           out->best_solution, out->num_hypotheses}, {out->inliers}, intrinsics,
                               in->points3d1, workspace, workspace_bytes,
                               geo_pnp_workspace_bytes(in->B, in->M, cfg->max_iters));
    };
    rc = Cam::COEFFS ? buffers({in->K0, dist0}) : buffers({in->K0});
  }
  if (rc != GEO_RUN) return rc;
  PnpArgs a = pnp_args(cfg, in, dist0, num_dist);
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.out = *out;
  const cudaStream_t stream = (cudaStream_t)stream_;
  if (int rc = geo_launch<PnpRansac<Cam>>(a, pnp_prepare_kernel<Cam>, stream)) return rc;
  if (a.M > 0) {
    pnp_mask_kernel<Cam><<<dim3(a.B, (a.M + MASK_THREADS - 1) / MASK_THREADS), MASK_THREADS, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  return 0;
}

}  // namespace

extern "C" size_t geo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  PnpWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_absolute_pose(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoPnpOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return absolute_pose<Pinhole>("geo_absolute_pose", cfg, in, nullptr, 0, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_absolute_pose_dist(const GeoPnpConfig* cfg, const GeoPnpDistInputs* din, GeoPnpOutputs* out,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  // a null din goes on as a null in, which geo_check_config reports
  return absolute_pose<Distorted>("geo_absolute_pose_dist", cfg, din ? &din->pnp : nullptr, din ? din->dist0 : nullptr,
                                  din ? din->num_dist : 0, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_absolute_pose_fisheye(const GeoPnpConfig* cfg, const GeoPnpDistInputs* din, GeoPnpOutputs* out,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  return absolute_pose<Fisheye>("geo_absolute_pose_fisheye", cfg, din ? &din->pnp : nullptr,
                                din ? din->dist0 : nullptr, din ? din->num_dist : 0, out, workspace, workspace_bytes,
                                stream);
}
