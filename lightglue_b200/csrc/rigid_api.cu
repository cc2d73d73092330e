// Batched 3D-3D rigid (SE(3)) and similarity (Sim(3)) RANSAC on the matcher's output: Horn's closed-form quaternion
// solve on 3-point samples, and the same closed form on the best hypothesis's inliers (include/geometry_b200.h, steps
// RG1-RG7).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  rigid_prepare_kernel, one 1024-thread CTA per pair: ordered compaction of the valid matches
//   per chunk of GEO_CHUNK hypotheses:
//     hyp    geo_hyp_kernel, one CTA per pair: folds the previous chunk's counts (geo_fold), decides the adaptive
//            stop, then one thread per hypothesis draws and solves its sample in double
//     score  geo_score_kernel with RigidScore: the inlier counts of the chunk's fp32 models
//   final    geo_final_kernel<RigidRansac>, one CTA per pair: folds the last chunk, the closed-form refit on the
//            inliers, re-score, outputs
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/rigid_oracle.py takes the
// same steps in numpy.
#include <stdint.h>

#include "block_scan.cuh"
#include "geo_common.cuh"
#include "ws_bump.h"

namespace {

constexpr int S = 3;       // points per sample
constexpr int NX = 13;     // a solution: R (row-major, 0-8), t (9-11), scale (12)
constexpr int TILE = 256;  // points per shared-memory tile of the score kernel: one per thread, and no spills

struct RigidPair {
  unsigned long long best;  // (count + 1) << 32 | ~(h * 16) of the best hypothesis so far; 0: none
  int n;                    // valid matches
  int ok;                   // n >= 3
  int stop;                 // no further hypotheses are drawn
  int drawn;                // hypotheses drawn so far
};

struct RigidWs {
  RigidPair* pair;  // [B]
  float4* p;        // [B, M] compacted point of points0 (x, y, z, 0)
  float4* q;        // [B, M] compacted point of points1 (x, y, z, 0)
  int* idx;         // [B, M] row of matches0 of each compacted match
  float* hyp;       // [B, GEO_CHUNK, 12] the current chunk's models, fp32
  int* count;       // [B, GEO_CHUNK] their inlier counts; -1: degenerate or not drawn
};

size_t carve(char* base, int B, int M, RigidWs* w) {
  WsBump b{base, 0};
  w->pair = b.take<RigidPair>(B);
  w->p = b.take<float4>((size_t)B * M);
  w->q = b.take<float4>((size_t)B * M);
  w->idx = b.take<int>((size_t)B * M);
  w->hyp = b.take<float>((size_t)B * GEO_CHUNK * 12);
  w->count = b.take<int>((size_t)B * GEO_CHUNK);
  return b.bytes();
}

// One model per slot, valid when its count is >= 0, as the H/F workspace records it
__device__ __forceinline__ int geo_models(const RigidWs& w, long slot) { return w.count[slot] >= 0; }
__device__ __forceinline__ void geo_set_models(const RigidWs& w, long slot, int ns) { w.count[slot] = ns ? 0 : -1; }

struct RigidArgs {
  int B, M, N, kind, max_iters, chunks;
  unsigned seed;
  float thr2;
  double confidence;
  const float* pts0;
  const float* pts1;
  const int64_t* matches0;
  RigidWs w;
  GeoRigidOutputs out;
};

__device__ __forceinline__ double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// RG3's degeneracy rule on one triangle: collinear or coincident unless |d1 x d2|^2 > eps * |d1|^2 |d2|^2
__device__ bool rigid_collinear(const double (*x)[3]) {
  double d1[3], d2[3], c[3];
  for (int i = 0; i < 3; ++i) {
    d1[i] = x[1][i] - x[0][i];
    d2[i] = x[2][i] - x[0][i];
  }
  c[0] = d1[1] * d2[2] - d1[2] * d2[1];
  c[1] = d1[2] * d2[0] - d1[0] * d2[2];
  c[2] = d1[0] * d2[1] - d1[1] * d2[0];
  return !(dot3(c, c) > GEO_RIGID_COLLINEAR_EPS * (dot3(d1, d1) * dot3(d2, d2)));
}

// The closed form of RG3 and RG6 from the centroids pb, qb, the cross-covariance S3 (S3[i][j] = sum a_i b_j) and
// saa = sum |a|^2: Horn's quaternion, then the scale (kind GEO_SIMILARITY_3D) and t.  False for a degenerate fit.
__device__ bool rigid_fit(int kind, const double* pb, const double* qb, const double (*S3)[3], double saa, double* x) {
  const double sxx = S3[0][0], sxy = S3[0][1], sxz = S3[0][2], syx = S3[1][0], syy = S3[1][1], syz = S3[1][2];
  const double szx = S3[2][0], szy = S3[2][1], szz = S3[2][2];
  const double N[4][4] = {{(sxx + syy) + szz, syz - szy, szx - sxz, sxy - syx},
                          {syz - szy, (sxx - syy) - szz, sxy + syx, szx + sxz},
                          {szx - sxz, sxy + syx, (syy - sxx) - szz, syz + szy},
                          {sxy - syx, szx + sxz, syz + szy, (szz - sxx) - syy}};
  double A[4][4], v[4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) A[i][j] = -N[i][j];
  smallest_eigvec<4>(A, v);
  const double nq = sqrt(((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]) + v[3] * v[3]);
  const double w = v[0] / nq, qx = v[1] / nq, qy = v[2] / nq, qz = v[3] / nq;
  double* R = x;
  R[0] = 1.0 - 2.0 * (qy * qy + qz * qz);
  R[1] = 2.0 * (qx * qy - w * qz);
  R[2] = 2.0 * (qx * qz + w * qy);
  R[3] = 2.0 * (qx * qy + w * qz);
  R[4] = 1.0 - 2.0 * (qx * qx + qz * qz);
  R[5] = 2.0 * (qy * qz - w * qx);
  R[6] = 2.0 * (qx * qz - w * qy);
  R[7] = 2.0 * (qy * qz + w * qx);
  R[8] = 1.0 - 2.0 * (qx * qx + qy * qy);
  double sc = 1.0;
  if (kind == GEO_SIMILARITY_3D) {
    double num = 0.0;  // sum_k b_k . (R a_k) = sum_ij R_ij S_ji
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) num = num + R[i * 3 + j] * S3[j][i];
    sc = num / saa;
  }
  x[12] = sc;
  for (int i = 0; i < 3; ++i) x[9 + i] = qb[i] - sc * ((R[i * 3] * pb[0] + R[i * 3 + 1] * pb[1]) + R[i * 3 + 2] * pb[2]);
  bool fin = sc > 0.0 && isfinite(sc);
  for (int i = 0; i < 12; ++i) fin = fin && isfinite(x[i]);
  return fin;
}

// RG4's fp32 squared distance of q from the float model g = [sR | t] (row-major 3x4) applied to p
__device__ __forceinline__ float rigid_err(const float* g, float4 p, float4 q) {
  const float e0 = (((g[0] * p.x + g[1] * p.y) + g[2] * p.z) + g[3]) - q.x;
  const float e1 = (((g[4] * p.x + g[5] * p.y) + g[6] * p.z) + g[7]) - q.y;
  const float e2 = (((g[8] * p.x + g[9] * p.y) + g[10] * p.z) + g[11]) - q.z;
  return (e0 * e0 + e1 * e1) + e2 * e2;
}

// geo_hyp_kernel's solver: sample h of pair b (RG2) and its closed form (RG3), scored as [sR | t]
struct RigidSolver {
  static constexpr int SOLS = 1, NX = ::NX, NF = 12;
  static __device__ int s(const RigidArgs&) { return S; }
  static __device__ int solve(const RigidArgs& a, int b, unsigned h, double (*x)[NX]) {
    int id[S];
    if (geo_sample(a.seed, h, a.w.pair[b].n, S, id) < S) return 0;
    double p[S][3], q[S][3];
    for (int k = 0; k < S; ++k) {
      const float4 u = a.w.p[(long)b * a.M + id[k]], v = a.w.q[(long)b * a.M + id[k]];
      p[k][0] = u.x; p[k][1] = u.y; p[k][2] = u.z;
      q[k][0] = v.x; q[k][1] = v.y; q[k][2] = v.z;
    }
    if (rigid_collinear(p) || rigid_collinear(q)) return 0;
    double pb[3], qb[3], S3[3][3] = {}, saa = 0.0;
    for (int i = 0; i < 3; ++i) {
      pb[i] = ((p[0][i] + p[1][i]) + p[2][i]) / 3.0;
      qb[i] = ((q[0][i] + q[1][i]) + q[2][i]) / 3.0;
    }
    for (int k = 0; k < S; ++k) {
      double ak[3], bk[3];
      for (int i = 0; i < 3; ++i) {
        ak[i] = p[k][i] - pb[i];
        bk[i] = q[k][i] - qb[i];
      }
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) S3[i][j] = S3[i][j] + ak[i] * bk[j];
      saa = saa + dot3(ak, ak);
    }
    return rigid_fit(a.kind, pb, qb, S3, saa, x[0]);
  }
  static __device__ void pixels(const RigidArgs&, int, const double* x, double* px) {
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) px[i * 4 + j] = x[12] * x[i * 3 + j];
      px[i * 4 + 3] = x[9 + i];
    }
  }
};

// Inlier counts of the chunk's [sR | t] models, on a tile of point pairs
struct RigidScore {
  using Args = RigidArgs;
  using Acc = int;
  static constexpr int SOLS = 1, NF = 12, K = 2, TILE = ::TILE;
  static __device__ const RigidWs& ws(const RigidArgs& a) { return a.w; }
  const float4* src[K];
  int* sums;
  float thr2;
  __device__ RigidScore(const RigidArgs& a, const RigidPair&, int b)
      : src{a.w.p + (long)b * a.M, a.w.q + (long)b * a.M}, sums(a.w.count), thr2(a.thr2) {}
  __device__ int term(const float* g, const float4* p) const { return rigid_err(g, p[0], p[1]) < thr2; }
};

// The refit's shared state: step 2's partial sums and the inlier centroids
struct RigidScratch {
  double red[RED];
  double c[6];
};

// The rigid or similarity model for geo_final_kernel: RG3's closed form on the best hypothesis's inliers (RG6)
struct RigidRansac : RigidSolver {
  using Base = RigidArgs;
  using Score = RigidScore;
  using Scratch = RigidScratch;

  static __device__ bool inlier(const RigidArgs& a, int b, const float* g, int k) {
    const long i = (long)b * a.M + k;
    return rigid_err(g, a.w.p[i], a.w.q[i]) < a.thr2;
  }
  static __device__ void clear(const RigidArgs& a, int b, int t) {
    for (int i = t; i < a.M; i += RED) a.out.inliers[(long)b * a.M + i] = 0;
  }
  static __device__ void fail(const RigidArgs& a, int b, int t) {
    if (t < 9) a.out.R[(long)b * 9 + t] = 0.0;
    if (t < 3) a.out.t[(long)b * 3 + t] = 0.0;
    if (t == 0) a.out.scale[b] = 0.0;
  }
  static __device__ bool refits(const RigidArgs&, int hcount) { return hcount >= S; }

  // Two passes of step 2's sums over the inliers of s.fm[0]: the centroids, then S and sum |a|^2.  A degenerate fit
  // becomes NaN, which has no inliers, so the hypothesis stays.
  static __device__ void refit(GeoFinal<RigidRansac>& s, const RigidArgs& a, int b, int t) {
    const int n = a.w.pair[b].n;
    const float4* P = a.w.p + (long)b * a.M;
    const float4* Q = a.w.q + (long)b * a.M;
    double acc[10];
    for (int i = 0; i < 6; ++i) acc[i] = 0.0;
    for (int k = t; k < n; k += RED) {
      const float4 p = P[k], q = Q[k];
      if (!(rigid_err(s.fm[0], p, q) < a.thr2)) continue;
      const double v[6] = {p.x, p.y, p.z, q.x, q.y, q.z};
      for (int i = 0; i < 6; ++i) acc[i] = acc[i] + v[i];
    }
    const double cnt = (double)s.count[0];
    for (int i = 0; i < 6; ++i) {
      const double sum = tree_sum(acc[i], s.m.red, t);
      if (t == 0) s.m.c[i] = sum / cnt;
    }
    __syncthreads();
    double c[6];
    for (int i = 0; i < 6; ++i) c[i] = s.m.c[i];
    for (int i = 0; i < 10; ++i) acc[i] = 0.0;
    for (int k = t; k < n; k += RED) {
      const float4 p = P[k], q = Q[k];
      if (!(rigid_err(s.fm[0], p, q) < a.thr2)) continue;
      const double ak[3] = {(double)p.x - c[0], (double)p.y - c[1], (double)p.z - c[2]};
      const double bk[3] = {(double)q.x - c[3], (double)q.y - c[4], (double)q.z - c[5]};
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) acc[i * 3 + j] = acc[i * 3 + j] + ak[i] * bk[j];
      acc[9] = acc[9] + dot3(ak, ak);
    }
    double S3[3][3], saa = 0.0;
    for (int i = 0; i < 10; ++i) {
      const double sum = tree_sum(acc[i], s.m.red, t);
      if (i < 9) S3[i / 3][i % 3] = sum;
      else saa = sum;
    }
    if (t == 0 && !rigid_fit(a.kind, c, c + 3, S3, saa, s.x[1]))
      for (int i = 0; i < NX; ++i) s.x[1][i] = __longlong_as_double(0x7ff8000000000000ll);
  }

  static __device__ void write(GeoFinal<RigidRansac>& s, const RigidArgs& a, int b, int u, int t) {
    geo_write_mask<RigidRansac>(a, b, s.fm[u], t);
    if (t < 9) a.out.R[(long)b * 9 + t] = s.x[u][t];
    if (t < 3) a.out.t[(long)b * 3 + t] = s.x[u][9 + t];
    if (t == 0) a.out.scale[b] = s.x[u][12];
  }
};

// RG1: ordered compaction of the matches whose index is in [0, N) and whose six coordinates are finite
__global__ void __launch_bounds__(1024) rigid_prepare_kernel(RigidArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  const int64_t* m0 = a.matches0 + (long)b * a.M;
  for (int base = 0; base < a.M; base += 1024) {
    const int i = base + tid;
    const int64_t j = i < a.M ? m0[i] : -1;
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f), q = p;
    if (j >= 0 && j < a.N) {
      const float* x = a.pts0 + ((long)b * a.M + i) * 3;
      const float* y = a.pts1 + ((long)b * a.N + j) * 3;
      p = make_float4(x[0], x[1], x[2], 0.f);
      q = make_float4(y[0], y[1], y[2], 0.f);
    }
    const bool valid = j >= 0 && j < a.N && isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(q.x) &&
                       isfinite(q.y) && isfinite(q.z);
    const int k = block_scan_step(valid, tid, warp_sums, &carry);
    if (valid) {
      a.w.p[(long)b * a.M + k] = p;
      a.w.q[(long)b * a.M + k] = q;
      a.w.idx[(long)b * a.M + k] = i;
    }
  }
  if (tid == 0) {
    RigidPair& P = a.w.pair[b];
    P.best = 0;
    P.n = carry;
    P.ok = carry >= S;
    P.stop = !P.ok;
    P.drawn = 0;
  }
}

}  // namespace

extern "C" size_t geo_rigid_workspace_bytes(int32_t B, int32_t M, int32_t) {
  if (B < 0 || M < 0) return 0;
  RigidWs w;
  return carve(nullptr, B, M, &w) + 256;
}

extern "C" int geo_estimate_rigid(const GeoConfig* cfg, const GeoInputs* in, GeoRigidOutputs* out, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  const char* entry = "geo_estimate_rigid";
  int rc = geo_check_config(entry, cfg, in, out, INT_MAX, [&] {
    return cfg->model != GEO_RIGID_3D && cfg->model != GEO_SIMILARITY_3D ? "unknown model" : nullptr;
  }, geo_no_check);
  if (rc == GEO_RUN)
    rc = geo_check_buffers(entry, in, {out->R, out->t, out->scale, out->num_inliers, out->success,
                                       out->best_hypothesis, out->num_hypotheses}, {out->inliers}, {}, in->kpts1,
                           workspace, workspace_bytes, geo_rigid_workspace_bytes(in->B, in->M, cfg->max_iters));
  if (rc != GEO_RUN) return rc;
  RigidArgs a{};
  carve(geo_workspace_base(workspace), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.kind = cfg->model;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.thr2 = (float)(cfg->threshold * cfg->threshold);
  a.confidence = cfg->confidence;
  a.pts0 = in->kpts0; a.pts1 = in->kpts1; a.matches0 = in->matches0;
  a.out = *out;
  return geo_launch<RigidRansac>(a, rigid_prepare_kernel, (cudaStream_t)stream_);
}
