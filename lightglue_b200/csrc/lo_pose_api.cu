// Batched LO-RANSAC relative pose on the matcher's output: MSAC-scored five-point sampling with Levenberg-Marquardt
// local optimisation and a final refinement (include/geometry_b200.h, steps L1-L8), on lo_common.cuh's schedule.
// pose_api.cu's compaction kernel prepares the pair; geo_hyp_kernel draws the five-point solutions; a local
// optimisation starts from P7's pose choice of its E and runs LM on the truncated Sampson cost; the final kernel adds
// the cheirality test of the chosen (R, t).  Compiled with -fmad=false: oracle/lo_pose_oracle.py takes the same steps.
#include <stdint.h>

#include "geo_lm.cuh"
#include "lg_internal.h"
#include "lo_common.cuh"
#include "pose_common.cuh"

namespace {

// recoverPose's cheirality test of the calibrated point (x, y) <-> (u, v) for P1 = [R | t] (header step P7).
// pose_kernel (pose_api.cu) writes the same steps inline: routed through this function its register allocation
// changes.
__device__ __forceinline__ bool cheirality_pass(const double (&P1)[3][4], double x, double y, double u, double v,
                                                double distance) {
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
  const double z1 = ((P1[2][0] * X + P1[2][1] * Y) + P1[2][2] * Z) + P1[2][3];
  return Q[2] * Q[3] > 0.0 && Z < distance && z1 > 0.0 && z1 < distance;
}

// [R | t] of a row-major R and t
__device__ __forceinline__ void projection34(const double* R, const double* tv, double (&P1)[3][4]) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) P1[i][j] = R[3 * i + j];
    P1[i][3] = tv[i];
  }
}

// Column-wise cross product: column j of out is a x M[:, j] ([a]x M), M and out row-major
__device__ __forceinline__ void cross_columns(const double* a, const double* M, double* out) {
  for (int j = 0; j < 3; ++j) {
    const double col[3] = {M[j], M[3 + j], M[6 + j]};
    double c[3];
    cross3(a, col, c);
    for (int i = 0; i < 3; ++i) out[3 * i + j] = c[i];
  }
}

__device__ void tangent_basis(const double* t, double* b1, double* b2) {
  int m = 0;
  for (int i = 1; i < 3; ++i)
    if (fabs(t[i]) < fabs(t[m])) m = i;
  const double e[3] = {m == 0 ? 1.0 : 0.0, m == 1 ? 1.0 : 0.0, m == 2 ? 1.0 : 0.0};
  double c[3];
  cross3(t, e, c);
  const double nc = sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]);
  for (int i = 0; i < 3; ++i) b1[i] = c[i] / nc;
  cross3(t, b1, b2);
}

__device__ __forceinline__ void lo_epipolar(const double* E, double x, double y, double u, double v, double* a0, double* a1,
                                            double* b0, double* b1, double* d) {
  *a0 = (E[0] * x + E[1] * y) + E[2];
  *a1 = (E[3] * x + E[4] * y) + E[5];
  const double a2 = (E[6] * x + E[7] * y) + E[8];
  *d = (u * *a0 + v * *a1) + a2;
  *b0 = (E[0] * u + E[3] * v) + E[6];
  *b1 = (E[1] * u + E[4] * v) + E[7];
}

// The chunk's L3 scores of every solution, count << 40 | MSAC score
struct LoPoseScore {
  using Args = LoArgs<PoseArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = ::SOLS, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const PoseWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  __device__ LoPoseScore(const Args& a, const PosePair& P, int b)
      : src{a.p.w.pts + (long)b * a.p.M}, sums(a.l.acc), thr2(P.thr2), w((float)GEO_LO_QSCALE / P.thr2) {}
  __device__ unsigned long long term(const float* g, const float4* p) const {
    return lo_term(sampson(g, p[0]), thr2, w);
  }
};

// The relative pose for lo_common.cuh's LM loop, re-score and schedule: x = R, t (header step L7)
struct PoseLo {
  static constexpr int DOF = 5, TERMS = 21, GROUP = 21, NP = 12, NF = 9, S = ::S, SOLS = ::SOLS;
  using Base = PoseArgs;
  using Args = LoArgs<PoseArgs>;
  using Solver = PoseSolver;
  using Score = LoPoseScore;
  struct Scratch {
    double E[9], dE[5][9];   // [t]x R and its derivatives at the pose being summed
    double Rs[2][9], ts[3];  // P7 candidates
    int good[4], count;
  };

  // The TERMS sums at pose (R, t) (header step L7) into out
  static __device__ void terms(LoShared<PoseLo>& s, const PosePair&, const double* pose, const float4* pts, int n,
                               double thr2, double* out, int tid) {
    if (tid == 0) {
      const double* R = pose;
      const double* t = pose + 9;
      cross_columns(t, R, s.m.E);
      for (int k = 0; k < 3; ++k) {
        const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
        double G[9];
        cross_columns(e, R, G);
        cross_columns(t, G, s.m.dE[k]);
      }
      double b1[3], b2[3];
      tangent_basis(t, b1, b2);
      cross_columns(b1, R, s.m.dE[3]);
      cross_columns(b2, R, s.m.dE[4]);
    }
    __syncthreads();
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts[k];
      const double x = p.x, y = p.y, u = p.z, v = p.w;
      double a0, a1, b0, b1, d;
      lo_epipolar(s.m.E, x, y, u, v, &a0, &a1, &b0, &b1, &d);
      const double den = ((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1;
      const double err = (d * d) / den;
      const bool in = err < thr2;
      acc[20] = acc[20] + (in ? err : thr2);
      if (!in) continue;
      const double sq = sqrt(den);
      const double r = d / sq;
      double J[5];
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        double da0, da1, db0, db1, dd;
        lo_epipolar(s.m.dE[q], x, y, u, v, &da0, &da1, &db0, &db1, &dd);
        const double dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1;
        J[q] = (dd - d * dden / den) / sq;
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < 5; ++i)
#pragma unroll
        for (int j = i; j < 5; ++j, ++e) acc[e] = acc[e] + J[i] * J[j];
#pragma unroll
      for (int i = 0; i < 5; ++i) acc[15 + i] = acc[15 + i] + J[i] * r;
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // R' = Q(d0..2) R, t' = normalize(t + d3 b1 + d4 b2) (header step L7)
  static __device__ void update(LoShared<PoseLo>&, const double* pose, const double* d, double* out) {
    double Q[9], b1[3], b2[3], v[3];
    quat_rotation(d, Q);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        out[3 * i + j] = Q[3 * i] * pose[j] + Q[3 * i + 1] * pose[3 + j] + Q[3 * i + 2] * pose[6 + j];
    tangent_basis(pose + 9, b1, b2);
    for (int i = 0; i < 3; ++i) v[i] = (pose[9 + i] + d[3] * b1[i]) + d[4] * b2[i];
    const double nv = sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    for (int i = 0; i < 3; ++i) out[9 + i] = v[i] / nv;
  }

  // E = [t]x R scaled as P3
  static __device__ void pixels(LoShared<PoseLo>&, const PosePair&, const double* pose, double* out) {
    cross_columns(pose + 9, pose, out);
    unit_scale(out);
  }

  static __device__ __forceinline__ float err(const float* h, float4 p) { return sampson(h, p); }

  static __device__ const float4* points(const Args& a, int b) { return a.p.w.pts + (long)b * a.p.M; }
  static __device__ const PosePair& consts(const Args& a, int b) { return a.p.w.pair[b]; }
  static __device__ Msac loss(const Args& a, int b) { return {a.p.w.pair[b].thr2}; }

  // L4's start: P7's pose choice of the solution's E (lo_choose_pose, below)
  static __device__ void seed(LoShared<PoseLo>& s, const Args& a, int b, unsigned hr, long m, LoPair& L, int t);

  static __device__ void store(LoShared<PoseLo>& s, LoPair& L) {
    for (int i = 0; i < 12; ++i) L.model[i] = s.x[i];
  }

  static __device__ void load(LoShared<PoseLo>& s, const Args&, int, const LoPair& L, int t) {
    if (t < 12) s.x[t] = L.model[t];
  }

  // The output E is [t]x R, not the sampled E: the stored (R, t) is scored again
  static __device__ void restore(LoShared<PoseLo>& s, const Args& a, int b, const LoPair& L, int t) {
    load(s, a, b, L, t);
    __syncthreads();
    lo_rescore(s, consts(a, b), points(a, b), a.p.w.pair[b].n, loss(a, b), t);
  }

  static __device__ void fail(const Args& a, int b, int t) {
    const GeoPoseOutputs& o = a.p.out;
    for (int i = t; i < a.p.M; i += RED) o.pose_inliers[(long)b * a.p.M + i] = 0;
    if (t < 9) o.E[(long)b * 9 + t] = o.R[(long)b * 9 + t] = 0.0;
    if (t < 3) o.t[(long)b * 3 + t] = 0.0;
    if (t == 0) o.num_pose_inliers[b] = 0;
  }

  // L8: the inliers of E and those that pass the cheirality test of (R, t)
  static __device__ void write(LoShared<PoseLo>& s, const Args& a, int b, int t) {
    const PosePair& P = a.p.w.pair[b];
    const GeoPoseOutputs& o = a.p.out;
    const float4* pts = points(a, b);
    const int* idx = a.p.w.idx + (long)b * a.p.M;
    uint8_t* inl = o.inliers + (long)b * a.p.M;
    uint8_t* pinl = o.pose_inliers + (long)b * a.p.M;
    for (int i = t; i < a.p.M; i += RED) inl[i] = pinl[i] = 0;
    if (t == 0) s.m.count = 0;
    __syncthreads();
    int cnt = 0;
    double P1[3][4];
    projection34(s.x, s.x + 9, P1);
    for (int k = t; k < P.n; k += RED) {
      const float4 p = pts[k];
      if (!(sampson(s.fm, p) < P.thr2)) continue;
      inl[idx[k]] = 1;
      if (cheirality_pass(P1, p.x, p.y, p.z, p.w, a.p.distance)) {
        pinl[idx[k]] = 1;
        ++cnt;
      }
    }
    if (cnt) atomicAdd(&s.m.count, cnt);
    __syncthreads();
    if (t < 9) {
      o.E[(long)b * 9 + t] = s.px[t];
      o.R[(long)b * 9 + t] = s.x[t];
    }
    if (t < 3) o.t[(long)b * 3 + t] = s.x[9 + t];
    if (t == 0) o.num_pose_inliers[b] = s.m.count;
  }
};

// P7's choice among the candidates of s.fm (widened) on s.fm's inliers, into s.x; every thread calls it
__device__ void lo_choose_pose(LoShared<PoseLo>& s, const float4* pts, int n, float thr2, double distance, int tid) {
  if (tid == 0) {
    double E[9];
    for (int i = 0; i < 9; ++i) E[i] = s.fm[i];
    pose_candidates(E, s.m.Rs, s.m.ts);
  }
  if (tid < 4) s.m.good[tid] = 0;
  __syncthreads();
  int cnt[4] = {0, 0, 0, 0};
  for (int k = tid; k < n; k += RED) {
    const float4 p = pts[k];
    if (!(sampson(s.fm, p) < thr2)) continue;
    for (int c = 0; c < 4; ++c) {
      const double sg = c < 2 ? 1.0 : -1.0;
      const double tv[3] = {sg * s.m.ts[0], sg * s.m.ts[1], sg * s.m.ts[2]};
      double P1[3][4];
      projection34(s.m.Rs[c & 1], tv, P1);
      cnt[c] += cheirality_pass(P1, p.x, p.y, p.z, p.w, distance);
    }
  }
  for (int c = 0; c < 4; ++c)
    if (cnt[c]) atomicAdd(&s.m.good[c], cnt[c]);
  __syncthreads();
  int best = 0;
  for (int c = 1; c < 4; ++c)
    if (s.m.good[c] > s.m.good[best]) best = c;
  if (tid < 9) s.x[tid] = s.m.Rs[best & 1][tid];
  if (tid < 3) s.x[9 + tid] = (best < 2 ? 1.0 : -1.0) * s.m.ts[tid];
  __syncthreads();
}

__device__ void PoseLo::seed(LoShared<PoseLo>& s, const Args& a, int b, unsigned, long m, LoPair& L, int t) {
  const PosePair& P = a.p.w.pair[b];
  if (t < 9) s.fm[t] = a.p.w.hyp[m * 9 + t];
  __syncthreads();
  lo_choose_pose(s, points(a, b), P.n, P.thr2, a.p.distance, t);
  if (t == 0) store(s, L);
}

}  // namespace

extern "C" size_t geo_lo_pose_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lo_workspace_bytes<PoseLo>(B, M);
}

extern "C" int geo_relative_pose_lo(const GeoLoPoseConfig* cfg, const GeoPoseInputs* in, GeoLoPoseOutputs* out,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_relative_pose_lo";
  int rc = geo_check_config(entry, cfg, in, out, GEO_LO_MAX_MATCHES, geo_no_check, [&] {
    return !(cfg->distance_threshold > 0.0) || !isfinite(cfg->distance_threshold) ? "distance_threshold must be positive"
                                                                                   : nullptr;
  });
  if (rc == GEO_RUN) {
    const GeoPoseOutputs& o = out->pose;
    rc = geo_check_buffers(entry, in, {o.E, o.R, o.t, o.num_inliers, o.num_pose_inliers, o.success, o.best_hypothesis,
                                       o.best_solution, o.num_hypotheses, out->num_local_optimizations, out->cost},
                           {o.inliers, o.pose_inliers}, {in->K0, in->K1}, in->kpts1, workspace, workspace_bytes,
                           geo_lo_pose_workspace_bytes(in->B, in->M, cfg->max_iters));
  }
  if (rc != GEO_RUN) return rc;
  PoseArgs p{};
  p.B = in->B; p.M = in->M; p.N = in->N;
  p.max_iters = cfg->max_iters;
  p.chunks = geo_chunks(cfg->max_iters);
  p.seed = cfg->seed;
  p.threshold = cfg->threshold;
  p.confidence = cfg->confidence;
  p.distance = cfg->distance_threshold;
  p.kpts0 = in->kpts0; p.kpts1 = in->kpts1; p.matches0 = in->matches0;
  p.K0 = in->K0; p.K1 = in->K1;
  p.out = out->pose;
  return lo_launch<PoseLo>(p, out->num_local_optimizations, out->cost, workspace, pose_prepare_kernel, stream_);
}
