// Batched relative pose on the matcher's output: five-point RANSAC for E, then recoverPose's cheirality test
// (include/geometry_b200.h, steps P1-P8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  pose_prepare_kernel, one 1024-thread CTA per pair: ordered compaction of the valid matches, calibrated
//            coordinates, K checks
//   per chunk of GEO_CHUNK samples:
//     hyp    geo_hyp_kernel, one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold),
//            decides the adaptive stop, then one thread per sample solves it: up to 10 fp32 models
//     score  geo_score_kernel<PoseScore>, (B, splits) CTAs: each streams a slice of the pair's points through shared
//            memory against every solution of the chunk, one thread per sample, and adds the inlier counts
//   final    geo_final_kernel<PoseRansac>, one CTA per pair: folds the last chunk, least-squares refit projected on the
//            essential manifold, recount, E and the inliers
//   pose     pose_kernel, one CTA per pair: the four (R, t) of E, linear triangulation of every inlier, the cheirality
//            test
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/pose_oracle.py takes the same
// steps in numpy.
#include <stdint.h>

#include "lg_internal.h"
#include "pose_common.cuh"

namespace {

// Inlier counts of every solution
struct PoseScore {
  using Args = PoseArgs;
  using Acc = int;
  static constexpr int SOLS = ::SOLS, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const PoseWs& ws(const PoseArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  float thr2;
  __device__ PoseScore(const PoseArgs& a, const PosePair& P, int b)
      : src{a.w.pts + (long)b * a.M}, sums(a.w.count), thr2(P.thr2) {}
  __device__ int term(const float* g, const float4* p) const { return sampson(g, p[0]) < thr2; }
};

// The relative pose for geo_final_kernel: least-squares refit projected on the essential manifold (header step P5)
struct PoseRansac : PoseSolver {
  using Base = PoseArgs;
  using Score = PoseScore;
  struct Scratch {
    double red[RED];
    double ata[45];
  };

  static __device__ bool inlier(const PoseArgs& a, int b, const float* g, int k) {
    return sampson(g, a.w.pts[(long)b * a.M + k]) < a.w.pair[b].thr2;
  }
  static __device__ void clear(const PoseArgs& a, int b, int t) {
    for (int i = t; i < a.M; i += RED) a.out.inliers[(long)b * a.M + i] = a.out.pose_inliers[(long)b * a.M + i] = 0;
  }
  static __device__ void fail(const PoseArgs& a, int b, int t) {
    if (t < 9) a.out.E[(long)b * 9 + t] = a.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.out.t[(long)b * 3 + t] = 0.0;
    if (t == 0) a.out.num_pose_inliers[b] = 0;
  }
  static __device__ bool refits(const PoseArgs&, int hcount) { return hcount >= GEO_REFIT_MIN; }

  static __device__ void refit(GeoFinal<PoseRansac>& s, const PoseArgs& a, int b, int t) {
    const float4* pts = a.w.pts + (long)b * a.M;
    geo_ata(a.w.pair[b].n, [&](int k) { return inlier(a, b, s.fm[0], k); },
            [&](int k, double* ra, double*) {
              const float4 p = pts[k];
              const double x = p.x, y = p.y, u = p.z, v = p.w;
              const double r[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
              for (int i = 0; i < 9; ++i) ra[i] = r[i];
              return 1;
            }, s.m.red, s.m.ata, t);
    if (t == 0) {
      double v[9], u1[3], u2[3], v1[3], v2[3];
      ata_null_vector(s.m.ata, v);
      svd2(v, u1, u2, v1, v2);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) s.x[1][r * 3 + c] = u1[r] * v1[c] + u2[r] * v2[c];
      unit_scale(s.x[1]);
    }
  }

  // E and its inliers, and E for pose_kernel
  static __device__ void write(GeoFinal<PoseRansac>& s, const PoseArgs& a, int b, int u, int t) {
    PosePair& P = a.w.pair[b];
    geo_write_mask<PoseRansac>(a, b, s.fm[u], t);
    if (t < 9) a.out.E[(long)b * 9 + t] = P.E[t] = s.px[u][t];
    if (t == 0) P.success = 1;
  }
};

__global__ void __launch_bounds__(POSE_THREADS, 1) pose_kernel(PoseArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  const PosePair& P = a.w.pair[b];
  if (!P.success) return;
  __shared__ double Rs[2][9], ts[3];
  __shared__ int good[4];
  if (t == 0) pose_candidates(P.E, Rs, ts);
  if (t < 4) good[t] = 0;
  __syncthreads();
  const float4* pts = a.w.pts + (long)b * a.M;
  const int* idx = a.w.idx + (long)b * a.M;
  const uint8_t* inl = a.out.inliers + (long)b * a.M;
  uint8_t* flags = a.w.flags + (long)b * a.M;
  int cnt[4] = {0, 0, 0, 0};
  for (int k = t; k < P.n; k += POSE_THREADS) {
    if (!inl[idx[k]]) continue;
    const float4 p = pts[k];
    const double x = p.x, y = p.y, u = p.z, v = p.w;
    unsigned bits = 0;
    for (int c = 0; c < 4; ++c) {  // recoverPose's order: (R1, t), (R2, t), (R1, -t), (R2, -t)
      const double* R = Rs[c & 1];
      const double sg = c < 2 ? 1.0 : -1.0;
      const double tv[3] = {sg * ts[0], sg * ts[1], sg * ts[2]};
      const double P1[3][4] = {{R[0], R[1], R[2], tv[0]}, {R[3], R[4], R[5], tv[1]}, {R[6], R[7], R[8], tv[2]}};
      double r[4][4] = {{-1.0, 0.0, x, 0.0}, {0.0, -1.0, y, 0.0}};
      for (int j = 0; j < 4; ++j) {
        r[2][j] = u * P1[2][j] - P1[0][j];
        r[3][j] = v * P1[2][j] - P1[1][j];
      }
      double Nm[4][4], Q[4];
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) Nm[i][j] = ((r[0][i] * r[0][j] + r[1][i] * r[1][j]) + r[2][i] * r[2][j]) + r[3][i] * r[3][j];
      smallest_eigvec<4>(Nm, Q);
      const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
      const double z1 = ((R[6] * X + R[7] * Y) + R[8] * Z) + tv[2];
      if (Q[2] * Q[3] > 0.0 && Z < a.distance && z1 > 0.0 && z1 < a.distance) {
        bits |= 1u << c;
        ++cnt[c];
      }
    }
    flags[k] = (uint8_t)bits;
  }
  for (int c = 0; c < 4; ++c)
    if (cnt[c]) atomicAdd(&good[c], cnt[c]);
  __syncthreads();
  int best = 0;
  for (int c = 1; c < 4; ++c)
    if (good[c] > good[best]) best = c;
  uint8_t* pinl = a.out.pose_inliers + (long)b * a.M;
  for (int k = t; k < P.n; k += POSE_THREADS)
    if (inl[idx[k]] && (flags[k] >> best & 1)) pinl[idx[k]] = 1;
  const double sg = best < 2 ? 1.0 : -1.0;
  if (t < 9) a.out.R[(long)b * 9 + t] = Rs[best & 1][t];
  if (t < 3) a.out.t[(long)b * 3 + t] = sg * ts[t];
  if (t == 0) a.out.num_pose_inliers[b] = good[best];
}


}  // namespace

extern "C" size_t geo_pose_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  PoseWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_relative_pose(const GeoPoseConfig* cfg, const GeoPoseInputs* in, GeoPoseOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_relative_pose";
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, geo_no_check, [&] {
    return !(cfg->distance_threshold > 0.0) || !isfinite(cfg->distance_threshold) ? "distance_threshold must be positive"
                                                                                   : nullptr;
  });
  if (rc == GEO_RUN)
    rc = geo_check_buffers(entry, in, {out->E, out->R, out->t, out->num_inliers, out->num_pose_inliers, out->success,
                                       out->best_hypothesis, out->best_solution, out->num_hypotheses},
                           {out->inliers, out->pose_inliers}, {in->K0, in->K1}, in->kpts1, workspace, workspace_bytes,
                           geo_pose_workspace_bytes(in->B, in->M, cfg->max_iters));
  if (rc != GEO_RUN) return rc;
  PoseArgs a{};
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.threshold = cfg->threshold;
  a.confidence = cfg->confidence;
  a.distance = cfg->distance_threshold;
  a.kpts0 = in->kpts0; a.kpts1 = in->kpts1; a.matches0 = in->matches0;
  a.K0 = in->K0; a.K1 = in->K1;
  a.out = *out;
  const cudaStream_t stream = (cudaStream_t)stream_;
  if (int rc = geo_launch<PoseRansac>(a, pose_prepare_kernel, stream)) return rc;
  pose_kernel<<<a.B, POSE_THREADS, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
