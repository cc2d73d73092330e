// Batched affine (6 degrees of freedom) and partial affine (rotation, uniform scale, translation) RANSAC on the
// matcher's output, with Levenberg-Marquardt refinement on the best hypothesis's inliers (include/geometry_b200.h,
// steps AF1-AF7).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  geo_prepare_kernel of geo_hf.cuh: ordered compaction, Hartley normalisation
//   per chunk of GEO_CHUNK hypotheses:
//     hyp    geo_hyp_kernel, one CTA per pair: folds the previous chunk's counts (geo_fold), decides the adaptive
//            stop, then one thread per hypothesis draws and solves its sample in double
//     score  geo_score_kernel with AfScore: the inlier counts of the chunk's fp32 models
//   final    geo_final_kernel<AfRansac>, one CTA per pair: folds the last chunk, LM refinement through
//            lo_common.cuh's loop, re-score, outputs
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/affine_oracle.py takes the
// same steps in numpy.
#include "geo_hf.cuh"
#include "lo_common.cuh"

namespace {

// The pixel model's six floats [a00, a01, a02, a10, a11, a12]; step 5's H error with the bottom row (0, 0, 1), where
// w = 1 / ((0*x0 + 0*y0) + 1) is exactly 1, so this is geo_err(GEO_HOMOGRAPHY) bit for bit without the division
__device__ __forceinline__ float af_err(const float* g, float4 p) {
  const float dx = p.z - ((g[0] * p.x + g[1] * p.y) + g[2]);
  const float dy = p.w - ((g[3] * p.x + g[4] * p.y) + g[5]);
  return dx * dx + dy * dy;
}

// The normalised model (affine: a..f of u = (a x + b y) + c, v = (d x + e y) + f; partial: a, b, tx, ty of
// u = (a x - b y) + tx, v = (b x + a y) + ty) -> the pixel model (header step AF3)
template <bool PARTIAL>
__device__ void af_pixels(const GeoPair& P, const double* X, double* A) {
  const double r = 1.0 / P.s1;
  if (PARTIAL) {
    const double kx = P.s0 * P.cx0, ky = P.s0 * P.cy0;
    A[0] = (X[0] * P.s0) * r;
    A[3] = (X[1] * P.s0) * r;
    A[1] = -A[3];
    A[4] = A[0];
    A[2] = (X[2] - (X[0] * kx - X[1] * ky)) * r + P.cx1;
    A[5] = (X[3] - (X[1] * kx + X[0] * ky)) * r + P.cy1;
    return;
  }
  const double T0[9] = {P.s0, 0.0, -(P.s0 * P.cx0), 0.0, P.s0, -(P.s0 * P.cy0), 0.0, 0.0, 1.0};
  const double L[9] = {r, 0.0, P.cx1, 0.0, r, P.cy1, 0.0, 0.0, 1.0};
  const double An[9] = {X[0], X[1], X[2], X[3], X[4], X[5], 0.0, 0.0, 1.0};
  double tmp[9], out[9];
  mm3(L, An, tmp);
  mm3(tmp, T0, out);
  for (int i = 0; i < 6; ++i) A[i] = out[i];
}

// |D| <= GEO_FLT_EPS * (((|dxj| + |dyj|) + |dxk|) + |dyk|): OpenCV's haveCollinearPoints on one triple
__device__ __forceinline__ bool af_collinear(double dxj, double dyj, double dxk, double dyk, double D) {
  return fabs(D) <= GEO_FLT_EPS * (((fabs(dxj) + fabs(dyj)) + fabs(dxk)) + fabs(dyk));
}

// Hypothesis h of a pair: its sample (header step 3), minimal solve on normalised coordinates (X) and pixel model (A).
// False for a degenerate sample.
template <bool PARTIAL>
__device__ bool af_hypothesis(const GeoArgs& a, const GeoPair& P, const float4* pts, unsigned h, double* X,
                              double* A) {
  constexpr int S = PARTIAL ? 2 : 3, NP = PARTIAL ? 4 : 6;
  int id[S];
  if (geo_sample(a.seed, h, P.n, S, id) < S) return false;
  double x[S], y[S], u[S], v[S];
  for (int q = 0; q < S; ++q) {
    const float4 p = pts[id[q]];
    x[q] = ((double)p.x - P.cx0) * P.s0;
    y[q] = ((double)p.y - P.cy0) * P.s0;
    u[q] = ((double)p.z - P.cx1) * P.s1;
    v[q] = ((double)p.w - P.cy1) * P.s1;
  }
  if (PARTIAL) {
    const double dx = x[1] - x[0], dy = y[1] - y[0], du = u[1] - u[0], dv = v[1] - v[0];
    const double dd = dx * dx + dy * dy;
    if (!(dd > 0.0) || (du == 0.0 && dv == 0.0)) return false;
    X[0] = (dx * du + dy * dv) / dd;
    X[1] = (dx * dv - dy * du) / dd;
    X[2] = u[0] - (X[0] * x[0] - X[1] * y[0]);
    X[3] = v[0] - (X[1] * x[0] + X[0] * y[0]);
  } else {
    const double dxj = x[1] - x[0], dyj = y[1] - y[0], dxk = x[2] - x[0], dyk = y[2] - y[0];
    const double D = dxj * dyk - dxk * dyj;
    const double duj = u[1] - u[0], dvj = v[1] - v[0], duk = u[2] - u[0], dvk = v[2] - v[0];
    if (af_collinear(dxj, dyj, dxk, dyk, D) || af_collinear(duj, dvj, duk, dvk, duj * dvk - duk * dvj)) return false;
    X[0] = (duj * dyk - duk * dyj) / D;
    X[1] = (dxj * duk - dxk * duj) / D;
    X[2] = u[0] - (X[0] * x[0] + X[1] * y[0]);
    X[3] = (dvj * dyk - dvk * dyj) / D;
    X[4] = (dxj * dvk - dxk * dvj) / D;
    X[5] = v[0] - (X[3] * x[0] + X[4] * y[0]);
  }
  af_pixels<PARTIAL>(P, X, A);
  bool fin = true;
  for (int i = 0; i < NP; ++i) fin = fin && isfinite(X[i]);
  for (int i = 0; i < 6; ++i) fin = fin && isfinite(A[i]);
  return fin;
}

// geo_hyp_kernel's solver: X of af_hypothesis per sample, scored as its pixel model
template <bool PARTIAL>
struct AfSolver {
  static constexpr int SOLS = 1, NX = PARTIAL ? 4 : 6, NF = 6;
  static __device__ int s(const GeoArgs& a) { return a.s; }
  static __device__ int solve(const GeoArgs& a, int b, unsigned h, double (*x)[NX]) {
    double A[6];
    return af_hypothesis<PARTIAL>(a, a.w.pair[b], a.w.pts + (long)b * a.M, h, x[0], A);
  }
  static __device__ void pixels(const GeoArgs& a, int b, const double* x, double* px) {
    af_pixels<PARTIAL>(a.w.pair[b], x, px);
  }
};

// Affine inlier counts of the chunk's six-float models
struct AfScore {
  using Args = GeoArgs;
  using Acc = int;
  static constexpr int SOLS = 1, NF = 6, K = 1, TILE = ::TILE;
  static __device__ const GeoWs& ws(const GeoArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  float thr2;
  __device__ AfScore(const GeoArgs& a, const GeoPair&, int b)
      : src{a.w.pts + (long)b * a.M}, sums(a.w.count), thr2(a.thr2) {}
  __device__ int term(const float* g, const float4* p) const { return af_err(g, p[0]) < thr2; }
};

// The points of the refinement and its fixed inlier set: those of the float model fm (header step AF6)
struct AfPoints {
  const float4* pts;
  const float* fm;
};

// The normalised model for lo_common.cuh's LM loop: x = X of af_hypothesis, residuals in normalised image-1 units
template <bool PARTIAL>
struct AffineLm {
  static constexpr int DOF = PARTIAL ? 4 : 6, TERMS = DOF * (DOF + 1) / 2 + DOF + 1, GROUP = PARTIAL ? 15 : 14,
                       NP = DOF, NF = 6;
  struct Scratch {};

  static __device__ void terms(LoShared<AffineLm>& s, const GeoPair& P, const double* X, AfPoints pts, int n,
                               double thr2, double* out, int tid) {
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts.pts[k];
      if (!(af_err(pts.fm, p) < (float)thr2)) continue;
      const double x = ((double)p.x - P.cx0) * P.s0, y = ((double)p.y - P.cy0) * P.s0;
      const double u = ((double)p.z - P.cx1) * P.s1, v = ((double)p.w - P.cy1) * P.s1;
      double rx, ry, jx[DOF], jy[DOF];
      if (PARTIAL) {
        rx = ((X[0] * x - X[1] * y) + X[2]) - u;
        ry = ((X[1] * x + X[0] * y) + X[3]) - v;
        const double ex[4] = {x, -y, 1.0, 0.0}, ey[4] = {y, x, 0.0, 1.0};
#pragma unroll
        for (int i = 0; i < DOF; ++i) { jx[i] = ex[i]; jy[i] = ey[i]; }
      } else {
        rx = ((X[0] * x + X[1] * y) + X[2]) - u;
        ry = ((X[3] * x + X[4] * y) + X[5]) - v;
        const double ex[6] = {x, y, 1.0, 0.0, 0.0, 0.0}, ey[6] = {0.0, 0.0, 0.0, x, y, 1.0};
#pragma unroll
        for (int i = 0; i < DOF; ++i) { jx[i] = ex[i]; jy[i] = ey[i]; }
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + (jx[i] * jx[j] + jy[i] * jy[j]);
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[e + i] = acc[e + i] + (jx[i] * rx + jy[i] * ry);
      acc[TERMS - 1] = acc[TERMS - 1] + (rx * rx + ry * ry);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  static __device__ void update(LoShared<AffineLm>&, const double* X, const double* d, double* out) {
    for (int i = 0; i < NP; ++i) out[i] = X[i] + d[i];
  }
};

// The affine model for geo_final_kernel: refine_iters LM steps on the best hypothesis's inliers (header step AF6)
template <bool PARTIAL>
struct AfRansac : AfSolver<PARTIAL> {
  using Base = GeoArgs;
  using Score = AfScore;
  using Scratch = LoShared<AffineLm<PARTIAL>>;

  static __device__ bool inlier(const GeoArgs& a, int b, const float* g, int k) {
    return af_err(g, a.w.pts[(long)b * a.M + k]) < a.thr2;
  }
  static __device__ void clear(const GeoArgs& a, int b, int t) {
    for (int i = t; i < a.M; i += RED) a.out.inliers[(long)b * a.M + i] = 0;
  }
  static __device__ void fail(const GeoArgs& a, int b, int t) {
    if (t < 9) a.out.model[(long)b * 9 + t] = 0.0;
  }
  static __device__ bool refits(const GeoArgs& a, int hcount) { return hcount >= a.s && a.refine_iters > 0; }

  static __device__ void refit(GeoFinal<AfRansac>& s, const GeoArgs& a, int b, int t) {
    constexpr int NP = AfSolver<PARTIAL>::NX;
    if (t == 0)
      for (int i = 0; i < NP; ++i) s.m.x[i] = s.x[0][i];
    __syncthreads();
    const GeoPair& P = a.w.pair[b];
    lo_refine(s.m, P, AfPoints{a.w.pts + (long)b * a.M, s.fm[0]}, P.n, (double)a.thr2, a.refine_iters,
              GEO_LO_LAMBDA0, t);
    if (t == 0)
      for (int i = 0; i < NP; ++i) s.x[1][i] = s.m.x[i];
  }

  // [A; 0 0 1] and its inliers
  static __device__ void write(GeoFinal<AfRansac>& s, const GeoArgs& a, int b, int u, int t) {
    geo_write_mask<AfRansac>(a, b, s.fm[u], t);
    if (t < 9) a.out.model[(long)b * 9 + t] = t < 6 ? s.px[u][t] : t == 8 ? 1.0 : 0.0;
  }
};

}  // namespace

extern "C" size_t geo_affine_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  GeoWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_estimate_affine(const GeoAffineConfig* cfg, const GeoInputs* in, GeoOutputs* out, void* workspace,
                                   size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_estimate_affine";
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, [&] {
    return cfg->model != GEO_AFFINE && cfg->model != GEO_AFFINE_PARTIAL ? "unknown model" : nullptr;
  }, [&] {
    return cfg->refine_iters < 0 || cfg->refine_iters > GEO_AFFINE_MAX_REFINE
               ? "refine_iters outside [0, GEO_AFFINE_MAX_REFINE]" : nullptr;
  });
  if (rc == GEO_RUN)
    rc = geo_check_buffers(entry, in, {out->model, out->num_inliers, out->success, out->best_hypothesis,
                                       out->num_hypotheses}, {out->inliers}, {}, in->kpts1, workspace, workspace_bytes,
                           geo_affine_workspace_bytes(in->B, in->M, cfg->max_iters));
  if (rc != GEO_RUN) return rc;
  GeoArgs a{};
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.kind = cfg->model;
  a.s = cfg->model == GEO_AFFINE ? 3 : 2;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.thr2 = (float)(cfg->threshold * cfg->threshold);
  a.confidence = cfg->confidence;
  a.kpts0 = in->kpts0; a.kpts1 = in->kpts1; a.matches0 = in->matches0;
  a.out = *out;
  a.refine_iters = cfg->refine_iters;
  const cudaStream_t stream = (cudaStream_t)stream_;
  return cfg->model == GEO_AFFINE ? geo_launch<AfRansac<false>>(a, geo_prepare_kernel, stream)
                                  : geo_launch<AfRansac<true>>(a, geo_prepare_kernel, stream);
}
