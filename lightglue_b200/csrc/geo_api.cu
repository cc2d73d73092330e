// Batched RANSAC on the matcher's output (include/geometry_b200.h, which states the algorithm step by step).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  geo_prepare_kernel, one 1024-thread CTA per pair: ordered compaction of the valid matches, Hartley
//            normalisation
//   per chunk of GEO_CHUNK hypotheses:
//     hyp    geo_hyp_kernel, one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold),
//            decides the adaptive stop, then one thread per hypothesis draws and solves its sample in double
//     score  geo_score_kernel<HfScore>, (B, splits) CTAs: each streams a slice of the pair's points through shared
//            memory against the chunk's fp32 models, one thread per hypothesis, and adds its inlier counts
//   final    geo_final_kernel<HfRansac>, one CTA per pair: folds the last chunk, least-squares refit on the best
//            hypothesis's inliers, recount, outputs
// A stopped pair's CTAs return at once.  This file is compiled with -fmad=false: every multiply and add rounds on its
// own, as numpy's do in oracle/geometry_oracle.py.
#include "geo_hf.cuh"
#include "lg_internal.h"

namespace {

// H or F inlier counts, the model kind read at run time
struct HfScore {
  using Args = GeoArgs;
  using Acc = int;
  static constexpr int SOLS = 1, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const GeoWs& ws(const GeoArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  int kind;
  float thr2;
  __device__ HfScore(const GeoArgs& a, const GeoPair&, int b)
      : src{a.w.pts + (long)b * a.M}, sums(a.w.count), kind(a.kind), thr2(a.thr2) {}
  __device__ int term(const float* h, const float4* p) const { return geo_err(kind, h, p[0]) < thr2; }
};

// Normalised DLT / 8-point rows of one correspondence; returns the number of rows (header step 4)
__device__ __forceinline__ int geo_rows(int kind, const GeoPair& P, float4 p, double* ra, double* rb) {
  const double x = ((double)p.x - P.cx0) * P.s0, y = ((double)p.y - P.cy0) * P.s0;
  const double u = ((double)p.z - P.cx1) * P.s1, v = ((double)p.w - P.cy1) * P.s1;
  if (kind == GEO_HOMOGRAPHY) {
    const double A[9] = {x, y, 1.0, 0.0, 0.0, 0.0, -u * x, -u * y, -u};
    const double Bv[9] = {0.0, 0.0, 0.0, x, y, 1.0, -v * x, -v * y, -v};
    for (int i = 0; i < 9; ++i) { ra[i] = A[i]; rb[i] = Bv[i]; }
    return 2;
  }
  const double A[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
  for (int i = 0; i < 9; ++i) ra[i] = A[i];
  return 1;
}

// H or F for geo_final_kernel: least-squares refit on the best hypothesis's inliers (header step 7)
struct HfRansac : HfSolver {
  using Base = GeoArgs;
  using Score = HfScore;
  struct Scratch {
    double red[RED];
    double ata[45];
  };

  static __device__ bool inlier(const GeoArgs& a, int b, const float* g, int k) {
    return geo_err(a.kind, g, a.w.pts[(long)b * a.M + k]) < a.thr2;
  }
  static __device__ void clear(const GeoArgs& a, int b, int t) {
    for (int i = t; i < a.M; i += RED) a.out.inliers[(long)b * a.M + i] = 0;
  }
  static __device__ void fail(const GeoArgs& a, int b, int t) {
    if (t < 9) a.out.model[(long)b * 9 + t] = 0.0;
  }
  static __device__ bool refits(const GeoArgs& a, int hcount) { return hcount >= a.s; }

  static __device__ void refit(GeoFinal<HfRansac>& s, const GeoArgs& a, int b, int t) {
    const GeoPair& P = a.w.pair[b];
    const float4* pts = a.w.pts + (long)b * a.M;
    geo_ata(P.n, [&](int k) { return inlier(a, b, s.fm[0], k); },
            [&](int k, double* ra, double* rb) { return geo_rows(a.kind, P, pts[k], ra, rb); }, s.m.red, s.m.ata, t);
    if (t == 0) {
      double v[9];
      ata_null_vector(s.m.ata, v);
      if (a.kind == GEO_FUNDAMENTAL) rank2(v);
      denormalise(a.kind, P, v, s.x[1]);
    }
  }

  static __device__ void write(GeoFinal<HfRansac>& s, const GeoArgs& a, int b, int u, int t) {
    geo_write_mask<HfRansac>(a, b, s.fm[u], t);
    if (t < 9) a.out.model[(long)b * 9 + t] = s.px[u][t];
  }
};

}  // namespace

extern "C" size_t geo_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  GeoWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_estimate(const GeoConfig* cfg, const GeoInputs* in, GeoOutputs* out, void* workspace,
                            size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_estimate";
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, [&] {
    return cfg->model != GEO_HOMOGRAPHY && cfg->model != GEO_FUNDAMENTAL ? "unknown model" : nullptr;
  }, geo_no_check);
  if (rc == GEO_RUN)
    rc = geo_check_buffers(entry, in, {out->model, out->num_inliers, out->success, out->best_hypothesis,
                                       out->num_hypotheses}, {out->inliers}, {}, in->kpts1, workspace, workspace_bytes,
                           geo_workspace_bytes(in->B, in->M, cfg->max_iters));
  if (rc != GEO_RUN) return rc;
  GeoArgs a{};
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.kind = cfg->model;
  a.s = cfg->model == GEO_HOMOGRAPHY ? 4 : 8;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.thr2 = (float)(cfg->threshold * cfg->threshold);
  a.confidence = cfg->confidence;
  a.kpts0 = in->kpts0; a.kpts1 = in->kpts1; a.matches0 = in->matches0;
  a.out = *out;
  return geo_launch<HfRansac>(a, geo_prepare_kernel, (cudaStream_t)stream_);
}
