// Batched RANSAC on the matcher's output (include/geometry_b200.h, which states the algorithm step by step).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  one 1024-thread CTA per pair: ordered compaction of the valid matches, Hartley normalisation
//   per chunk of GEO_CHUNK hypotheses:
//     hyp    one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold), decides the
//            adaptive stop, then one thread per hypothesis draws and solves its sample in double
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against the chunk's
//            fp32 models, one thread per hypothesis, and adds its inlier counts
//   refit    one CTA per pair: folds the last chunk, least-squares refit on the best hypothesis's inliers, recount,
//            outputs
// A stopped pair's CTAs return at once.  This file is compiled with -fmad=false: every multiply and add rounds on its
// own, as numpy's do in oracle/geometry_oracle.py.
#include "geo_hf.cuh"
#include "lg_internal.h"

namespace {

__global__ void __launch_bounds__(GEO_CHUNK, 1) geo_hyp_kernel(GeoArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c > 0) geo_fold<1>(a, a.s, b, c - 1);
  const GeoPair& P = a.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  double m[9];
  const bool ok = P.stop == 0 && h < a.max_iters && geo_hypothesis(a, P, a.w.pts + (long)b * a.M, h, m);
  if (ok) {
    float* hm = a.w.hyp + ((long)b * GEO_CHUNK + t) * 9;
    for (int i = 0; i < 9; ++i) hm[i] = (float)m[i];
  }
  a.w.count[(long)b * GEO_CHUNK + t] = ok ? 0 : -1;
}

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

__global__ void __launch_bounds__(RED, 1) geo_refit_kernel(GeoArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  geo_fold<1>(a, a.s, b, a.chunks - 1);
  const GeoPair& P = a.w.pair[b];
  const float4* pts = a.w.pts + (long)b * a.M;
  const int* idx = a.w.idx + (long)b * a.M;
  uint8_t* inl = a.out.inliers + (long)b * a.M;
  __shared__ double red[RED];
  __shared__ double ata[45];
  __shared__ double model[2][9];
  __shared__ float fm[2][9];
  __shared__ int count[2];
  for (int i = t; i < a.M; i += RED) inl[i] = 0;
  const unsigned long long key = P.best;
  if (!P.ok || key == 0) {
    if (t < 9) a.out.model[(long)b * 9 + t] = 0.0;
    if (t == 0) {
      a.out.num_inliers[b] = 0;
      a.out.success[b] = 0;
      a.out.best_hypothesis[b] = -1;
      a.out.num_hypotheses[b] = P.drawn;
    }
    return;
  }
  const unsigned hb = ~(unsigned)(key & 0xffffffffu) >> 4;
  const int hcount = (int)(key >> 32) - 1;
  if (t == 0) {
    geo_hypothesis(a, P, pts, hb, model[0]);
    for (int i = 0; i < 9; ++i) fm[0][i] = (float)model[0][i];
    count[0] = hcount;
    count[1] = -1;
  }
  __syncthreads();
  if (hcount >= a.s) {
    // one pass over the points per row i of the upper triangle keeps 9 accumulators in registers
    for (int i = 0, e0 = 0; i < 9; e0 += 9 - i, ++i) {
      double acc[9];
#pragma unroll
      for (int j = 0; j < 9; ++j) acc[j] = 0.0;
      for (int k = t; k < P.n; k += RED) {
        const float4 p = pts[k];
        if (!(geo_err(a.kind, fm[0], p) < a.thr2)) continue;
        double ra[9], rb[9];
        const int rows = geo_rows(a.kind, P, p, ra, rb);
#pragma unroll
        for (int j = 0; j < 9; ++j)
          if (j >= i) acc[j] = acc[j] + (rows == 2 ? ra[i] * ra[j] + rb[i] * rb[j] : ra[i] * ra[j]);
      }
#pragma unroll
      for (int j = 0; j < 9; ++j)
        if (j >= i) {
          const double s = tree_sum(acc[j], red, t);
          if (t == 0) ata[e0 + j - i] = s;
        }
    }
    if (t == 0) {
      double A[9][9], v[9];
      for (int i = 0, e = 0; i < 9; ++i)
        for (int j = i; j < 9; ++j, ++e) A[i][j] = A[j][i] = ata[e];
      smallest_eigvec<9>(A, v);
      if (a.kind == GEO_FUNDAMENTAL) rank2(v);
      denormalise(a.kind, P, v, model[1]);
      for (int i = 0; i < 9; ++i) fm[1][i] = (float)model[1][i];
      count[1] = 0;
    }
    __syncthreads();
    int k1 = 0;
    for (int k = t; k < P.n; k += RED) k1 += geo_err(a.kind, fm[1], pts[k]) < a.thr2;
    if (k1) atomicAdd(&count[1], k1);
    __syncthreads();
  }
  const int u = count[1] >= count[0] ? 1 : 0;
  for (int k = t; k < P.n; k += RED)
    if (geo_err(a.kind, fm[u], pts[k]) < a.thr2) inl[idx[k]] = 1;
  if (t < 9) a.out.model[(long)b * 9 + t] = model[u][t];
  if (t == 0) {
    a.out.num_inliers[b] = count[u];
    a.out.success[b] = 1;
    a.out.best_hypothesis[b] = (int)hb;
    a.out.num_hypotheses[b] = P.drawn;
  }
}

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
  const int splits = geo_score_splits(a.B, a.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  geo_prepare_kernel<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    geo_hyp_kernel<<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<HfScore><<<dim3(a.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  geo_refit_kernel<<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
