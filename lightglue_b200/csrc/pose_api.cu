// Batched relative pose on the matcher's output: five-point RANSAC for E, then recoverPose's cheirality test
// (include/geometry_b200.h, steps P1-P8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  one 1024-thread CTA per pair: ordered compaction of the valid matches, calibrated coordinates, K checks
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair: folds the previous chunk's counts into the pair's best (geo_fold), decides the
//            adaptive stop, then one thread per sample solves it: up to 10 fp32 models
//     score  (B, splits) CTAs: each streams a slice of the pair's points through shared memory against every solution
//            of the chunk, one thread per sample, and adds the inlier counts
//   refit    one CTA per pair: folds the last chunk, least-squares refit projected on the essential manifold, recount,
//            E and the inliers
//   pose     one CTA per pair: the four (R, t) of E, linear triangulation of every inlier, the cheirality test
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/pose_oracle.py takes the same
// steps in numpy.
#include <stdint.h>

#include "lg_internal.h"
#include "pose_common.cuh"

namespace {

__global__ void __launch_bounds__(GEO_CHUNK, 1) pose_hyp_kernel(PoseArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c > 0) geo_fold<SOLS>(a, S, b, c - 1);
  const PosePair& P = a.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  int ns = 0;
  int id[S];
  if (P.stop == 0 && h < a.max_iters && geo_sample(a.seed, h, P.n, S, id) == S) {
    double sol[SOLS][9];
    ns = five_point(a.w.pts + (long)b * a.M, id, sol);
    float* hm = a.w.hyp + ((long)b * GEO_CHUNK + t) * SOLS * 9;
    for (int r = 0; r < ns; ++r) {
      for (int i = 0; i < 9; ++i) hm[r * 9 + i] = (float)sol[r][i];
      a.w.count[((long)b * GEO_CHUNK + t) * SOLS + r] = 0;
    }
  }
  a.w.nsol[(long)b * GEO_CHUNK + t] = ns;
}

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

__global__ void __launch_bounds__(RED, 1) pose_refit_kernel(PoseArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  geo_fold<SOLS>(a, S, b, a.chunks - 1);
  PosePair& P = a.w.pair[b];
  const float4* pts = a.w.pts + (long)b * a.M;
  const int* idx = a.w.idx + (long)b * a.M;
  uint8_t* inl = a.out.inliers + (long)b * a.M;
  uint8_t* pinl = a.out.pose_inliers + (long)b * a.M;
  __shared__ double red[RED];
  __shared__ double ata[45];
  __shared__ double model[2][9];
  __shared__ float fm[2][9];
  __shared__ int count[2];
  for (int i = t; i < a.M; i += RED) inl[i] = pinl[i] = 0;
  const unsigned long long key = P.best;
  if (!P.ok || key == 0) {
    if (t < 9) a.out.E[(long)b * 9 + t] = a.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.out.t[(long)b * 3 + t] = 0.0;
    if (t == 0) {
      a.out.num_inliers[b] = a.out.num_pose_inliers[b] = 0;
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
    double sol[SOLS][9];
    geo_sample(a.seed, hr >> 4, P.n, S, id);
    five_point(pts, id, sol);
    for (int i = 0; i < 9; ++i) {
      model[0][i] = sol[hr & 15][i];
      fm[0][i] = (float)model[0][i];
    }
    count[0] = hcount;
    count[1] = -1;
  }
  __syncthreads();
  if (hcount >= GEO_REFIT_MIN) {
    for (int i = 0, e0 = 0; i < 9; e0 += 9 - i, ++i) {
      double acc[9];
#pragma unroll
      for (int j = 0; j < 9; ++j) acc[j] = 0.0;
      for (int k = t; k < P.n; k += RED) {
        const float4 p = pts[k];
        if (!(sampson(fm[0], p) < thr2)) continue;
        const double x = p.x, y = p.y, u = p.z, v = p.w;
        const double ra[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
#pragma unroll
        for (int j = 0; j < 9; ++j)
          if (j >= i) acc[j] = acc[j] + ra[i] * ra[j];
      }
#pragma unroll
      for (int j = 0; j < 9; ++j)
        if (j >= i) {
          const double s = tree_sum(acc[j], red, t);
          if (t == 0) ata[e0 + j - i] = s;
        }
    }
    if (t == 0) {
      double A[9][9], v[9], u1[3], u2[3], v1[3], v2[3];
      for (int i = 0, e = 0; i < 9; ++i)
        for (int j = i; j < 9; ++j, ++e) A[i][j] = A[j][i] = ata[e];
      smallest_eigvec<9>(A, v);
      svd2(v, u1, u2, v1, v2);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) model[1][r * 3 + c] = u1[r] * v1[c] + u2[r] * v2[c];
      unit_scale(model[1]);
      for (int i = 0; i < 9; ++i) fm[1][i] = (float)model[1][i];
      count[1] = 0;
    }
    __syncthreads();
    int k1 = 0;
    for (int k = t; k < P.n; k += RED) k1 += sampson(fm[1], pts[k]) < thr2;
    if (k1) atomicAdd(&count[1], k1);
    __syncthreads();
  }
  const int u = count[1] >= count[0] ? 1 : 0;
  for (int k = t; k < P.n; k += RED)
    if (sampson(fm[u], pts[k]) < thr2) inl[idx[k]] = 1;
  if (t < 9) a.out.E[(long)b * 9 + t] = P.E[t] = model[u][t];
  if (t == 0) {
    a.out.num_inliers[b] = count[u];
    a.out.success[b] = 1;
    a.out.best_hypothesis[b] = (int)(hr >> 4);
    a.out.best_solution[b] = (int)(hr & 15);
    a.out.num_hypotheses[b] = P.drawn;
    P.success = 1;
  }
}

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
  const int splits = geo_score_splits(a.B, a.M);
  const cudaStream_t stream = (cudaStream_t)stream_;
  pose_prepare_kernel<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    pose_hyp_kernel<<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<PoseScore><<<dim3(a.B, splits), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  pose_refit_kernel<<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  pose_kernel<<<a.B, POSE_THREADS, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
