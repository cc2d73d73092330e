// The H/F RANSAC's shared pieces (include/geometry_b200.h, steps 1-5): the workspace, the compaction and Hartley
// normalisation kernel, the sampler and minimal solvers, and the fp32 error.  Included by geo_api.cu (RANSAC, steps
// 1-7) and lo_hf_api.cu (LO-RANSAC homography and fundamental matrix, LH1-LH8 and LF1-LF8), both compiled with
// -fmad=false.
#pragma once
#include <stdint.h>

#include "block_scan.cuh"
#include "geo_common.cuh"
#include "ws_bump.h"

namespace {

constexpr int TILE = 1024;  // points per shared-memory tile of the score kernel

struct GeoPair {
  double cx0, cy0, s0, cx1, cy1, s1;  // Hartley normalisation of image 0 and image 1
  unsigned long long best;            // (count + 1) << 32 | ~(h * 16) of the best hypothesis so far; 0: none
  int n;                              // valid matches
  int ok;                             // n >= sample size and the normalisation succeeded
  int stop;                           // no further hypotheses are drawn
  int drawn;                          // hypotheses drawn so far
};

struct GeoWs {
  GeoPair* pair;  // [B]
  float4* pts;    // [B, M] compacted (x0, y0, x1, y1)
  int* idx;       // [B, M] row of matches0 of each compacted match
  float* hyp;     // [B, GEO_CHUNK, 9] the current chunk's models, fp32
  int* count;     // [B, GEO_CHUNK] their inlier counts; -1: degenerate or not drawn
};

size_t carve(char* base, int B, int M, GeoWs* w) {
  WsBump b{base, 0};
  w->pair = b.take<GeoPair>(B);
  w->pts = b.take<float4>((size_t)B * M);
  w->idx = b.take<int>((size_t)B * M);
  w->hyp = b.take<float>((size_t)B * GEO_CHUNK * 9);
  w->count = b.take<int>((size_t)B * GEO_CHUNK);
  return b.bytes();
}

// geo_fold's and geo_score_kernel's valid models of chunk slot `slot`: one, unless degenerate or not drawn
__device__ __forceinline__ int geo_models(const GeoWs& w, long slot) { return w.count[slot] >= 0; }
__device__ __forceinline__ void geo_set_models(const GeoWs& w, long slot, int ns) { w.count[slot] = ns ? 0 : -1; }

struct GeoArgs {
  int B, M, N, kind, s, max_iters, chunks;
  unsigned seed;
  float thr2;
  int refine_iters;  // the affine refinement's LM steps
  double confidence;
  const float* kpts0;
  const float* kpts1;
  const int64_t* matches0;
  GeoWs w;
  GeoOutputs out;
};

// (A B)_ij = (A_i0 B_0j + A_i1 B_1j) + A_i2 B_2j, row-major 3x3
__device__ void mm3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = (A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j]) + A[i * 3 + 2] * B[6 + j];
}

// Rank 2 by one-sided Jacobi on the columns (header step 4), in place on a row-major 3x3.
__device__ void rank2(double* F) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) A[i] = F[i];
  jacobi_columns3(A, V);
  int m = 0;
  double nm = 0.0;
  for (int j = 0; j < 3; ++j) {
    double nj = 0.0;
    for (int i = 0; i < 3; ++i) nj = nj + A[i * 3 + j] * A[i * 3 + j];
    if (j == 0 || nj < nm) { nm = nj; m = j; }
  }
  for (int i = 0; i < 3; ++i) A[i * 3 + m] = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      F[i * 3 + j] = (A[i * 3] * V[j * 3] + A[i * 3 + 1] * V[j * 3 + 1]) + A[i * 3 + 2] * V[j * 3 + 2];
}

// A normalised model v (row-major) -> pixel coordinates, then the output scale (header step 4).
__device__ void denormalise(int kind, const GeoPair& P, const double* v, double* out) {
  const double T0[9] = {P.s0, 0.0, -(P.s0 * P.cx0), 0.0, P.s0, -(P.s0 * P.cy0), 0.0, 0.0, 1.0};
  double L[9];
  if (kind == GEO_HOMOGRAPHY) {
    const double r = 1.0 / P.s1;
    const double Li[9] = {r, 0.0, P.cx1, 0.0, r, P.cy1, 0.0, 0.0, 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Li[i];
  } else {
    const double Lt[9] = {P.s1, 0.0, 0.0, 0.0, P.s1, 0.0, -(P.s1 * P.cx1), -(P.s1 * P.cy1), 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Lt[i];
  }
  double tmp[9];
  mm3(L, v, tmp);
  mm3(tmp, T0, out);
  double f = 0.0;
  for (int i = 0; i < 9; ++i) f = f + out[i] * out[i];
  f = sqrt(f);
  if (kind == GEO_HOMOGRAPHY) {
    const double d = fabs(out[8]) >= 1e-12 * f ? out[8] : f;
    for (int i = 0; i < 9; ++i) out[i] = out[i] / d;
  } else {
    int k = 0;
    for (int i = 0; i < 9; ++i) {
      out[i] = out[i] / f;
      if (fabs(out[i]) > fabs(out[k])) k = i;
    }
    if (out[k] < 0.0)
      for (int i = 0; i < 9; ++i) out[i] = -out[i];
  }
}

// OpenCV's orientation test and collinearity check on the 4 points of an H sample (header step 4).
__device__ bool h_sample_ok(const double* x0, const double* y0, const double* x1, const double* y1) {
  const int TT[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {0, 1, 3}};
  int negative = 0;
  for (int q = 0; q < 4; ++q) {
    double D[2];
    for (int img = 0; img < 2; ++img) {
      const double* X = img ? x1 : x0;
      const double* Y = img ? y1 : y0;
      const int i = TT[q][0], j = TT[q][1], k = TT[q][2];
      const double dxj = X[j] - X[i], dyj = Y[j] - Y[i], dxk = X[k] - X[i], dyk = Y[k] - Y[i];
      D[img] = dxj * dyk - dxk * dyj;
      if (fabs(D[img]) <= GEO_FLT_EPS * (((fabs(dxj) + fabs(dyj)) + fabs(dxk)) + fabs(dyk))) return false;
    }
    negative += D[0] * D[1] < 0.0;
  }
  return negative == 0 || negative == 4;
}

// Null vector of an 8x9 system by Gaussian elimination with partial pivoting; false when rank-deficient.
__device__ bool null_vector(double (*A)[9], double* v) {
  for (int k = 0; k < 8; ++k) {
    int p = k;
    double best = fabs(A[k][k]);
    for (int r = k + 1; r < 8; ++r)
      if (fabs(A[r][k]) > best) { best = fabs(A[r][k]); p = r; }
    if (!(best > GEO_PIVOT_EPS)) return false;
    if (p != k)
      for (int c = k; c < 9; ++c) { const double t = A[k][c]; A[k][c] = A[p][c]; A[p][c] = t; }
    for (int r = k + 1; r < 8; ++r) {
      const double f = A[r][k] / A[k][k];
      for (int c = k + 1; c < 9; ++c) A[r][c] = A[r][c] - f * A[k][c];
    }
  }
  v[8] = 1.0;
  for (int k = 7; k >= 0; --k) {
    double acc = A[k][8];
    for (int c = k + 1; c < 8; ++c) acc = acc + A[k][c] * v[c];
    v[k] = -acc / A[k][k];
  }
  return true;
}

// Hypothesis h of a pair: its sample (header step 3) and minimal solve (step 4).  False for a degenerate sample.
__device__ bool geo_hypothesis(const GeoArgs& a, const GeoPair& P, const float4* pts, unsigned h, double* model) {
  int id[8];
  int k = 0;
  const unsigned x = geo_mix(geo_mix(a.seed ^ 0x9e3779b9u) ^ h);
  for (unsigned t = 0; t < GEO_MAX_DRAWS && k < a.s; ++t) {
    const int j = (int)(((unsigned long long)geo_mix(x + t) * (unsigned)P.n) >> 32);
    bool dup = false;
    for (int q = 0; q < k; ++q) dup = dup || id[q] == j;
    if (!dup) id[k++] = j;
  }
  if (k < a.s) return false;
  double x0[8], y0[8], x1[8], y1[8];
  for (int q = 0; q < a.s; ++q) {
    const float4 p = pts[id[q]];
    x0[q] = ((double)p.x - P.cx0) * P.s0;
    y0[q] = ((double)p.y - P.cy0) * P.s0;
    x1[q] = ((double)p.z - P.cx1) * P.s1;
    y1[q] = ((double)p.w - P.cy1) * P.s1;
  }
  double A[8][9];
  if (a.kind == GEO_HOMOGRAPHY) {
    if (!h_sample_ok(x0, y0, x1, y1)) return false;
    for (int q = 0; q < 4; ++q) {
      const double x = x0[q], y = y0[q], u = x1[q], v = y1[q];
      const double ra[9] = {x, y, 1.0, 0.0, 0.0, 0.0, -u * x, -u * y, -u};
      const double rb[9] = {0.0, 0.0, 0.0, x, y, 1.0, -v * x, -v * y, -v};
      for (int c = 0; c < 9; ++c) { A[2 * q][c] = ra[c]; A[2 * q + 1][c] = rb[c]; }
    }
  } else {
    for (int q = 0; q < 8; ++q) {
      const double x = x0[q], y = y0[q], u = x1[q], v = y1[q];
      const double r[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
      for (int c = 0; c < 9; ++c) A[q][c] = r[c];
    }
  }
  double v[9];
  if (!null_vector(A, v)) return false;
  if (a.kind == GEO_FUNDAMENTAL) rank2(v);
  denormalise(a.kind, P, v, model);
  return true;
}

// geo_hyp_kernel's solver of H or F (a.kind and a.s pick it): one pixel model per sample
struct HfSolver {
  static constexpr int SOLS = 1, NX = 9, NF = 9;
  static __device__ int s(const GeoArgs& a) { return a.s; }
  static __device__ int solve(const GeoArgs& a, int b, unsigned h, double (*x)[NX]) {
    return geo_hypothesis(a, a.w.pair[b], a.w.pts + (long)b * a.M, h, x[0]);
  }
  static __device__ void pixels(const GeoArgs&, int, const double* x, double* px) {
    for (int i = 0; i < NF; ++i) px[i] = x[i];
  }
};

// fp32 error of one correspondence (header step 5)
__device__ __forceinline__ float geo_err(int kind, const float* h, float4 p) {
  if (kind == GEO_HOMOGRAPHY) {
    const float w = 1.f / ((h[6] * p.x + h[7] * p.y) + h[8]);
    const float dx = p.z - ((h[0] * p.x + h[1] * p.y) + h[2]) * w;
    const float dy = p.w - ((h[3] * p.x + h[4] * p.y) + h[5]) * w;
    return dx * dx + dy * dy;
  }
  float a = (h[0] * p.x + h[1] * p.y) + h[2], b = (h[3] * p.x + h[4] * p.y) + h[5], c = (h[6] * p.x + h[7] * p.y) + h[8];
  const float d2 = (p.z * a + p.w * b) + c, s2 = 1.f / (a * a + b * b);
  a = (h[0] * p.z + h[3] * p.w) + h[6];
  b = (h[1] * p.z + h[4] * p.w) + h[7];
  c = (h[2] * p.z + h[5] * p.w) + h[8];
  const float d1 = (p.x * a + p.y * b) + c, s1 = 1.f / (a * a + b * b);
  return fmaxf(d1 * d1 * s1, d2 * d2 * s2);
}

// Step 1's compaction and step 2's normalisation of pair blockIdx.x, by a CTA of 1024 threads
__device__ __forceinline__ void geo_prepare(GeoArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  __shared__ double red[RED];
  if (tid == 0) carry = 0;
  __syncthreads();
  const int64_t* m0 = a.matches0 + (long)b * a.M;
  float4* pts = a.w.pts + (long)b * a.M;
  for (int base = 0; base < a.M; base += 1024) {
    const int i = base + tid;
    const int64_t j = i < a.M ? m0[i] : -1;
    float2 p0 = make_float2(0.f, 0.f), p1 = p0;
    if (j >= 0 && j < a.N) {
      p0 = reinterpret_cast<const float2*>(a.kpts0)[(long)b * a.M + i];
      p1 = reinterpret_cast<const float2*>(a.kpts1)[(long)b * a.N + j];
    }
    const bool valid = j >= 0 && j < a.N && finite2(p0) && finite2(p1);
    const int slot = block_scan_step(valid, tid, warp_sums, &carry);
    if (valid) {
      pts[slot] = make_float4(p0.x, p0.y, p1.x, p1.y);
      a.w.idx[(long)b * a.M + slot] = i;
    }
  }
  const int n = carry;
  __syncthreads();
  double c[4], d[2];
  for (int q = 0; q < 4; ++q) {
    double p = 0.0;
    for (int k = tid; tid < RED && k < n; k += RED) {
      const float4 v = pts[k];
      p = p + (double)(q == 0 ? v.x : q == 1 ? v.y : q == 2 ? v.z : v.w);
    }
    c[q] = tree_sum(p, red, tid) / (double)n;
  }
  for (int img = 0; img < 2; ++img) {
    double p = 0.0;
    for (int k = tid; tid < RED && k < n; k += RED) {
      const float4 v = pts[k];
      const double dx = (double)(img ? v.z : v.x) - c[2 * img], dy = (double)(img ? v.w : v.y) - c[2 * img + 1];
      p = p + sqrt(dx * dx + dy * dy);
    }
    d[img] = tree_sum(p, red, tid) / (double)n;
  }
  if (tid == 0) {
    GeoPair& P = a.w.pair[b];
    P.cx0 = c[0]; P.cy0 = c[1]; P.s0 = M_SQRT2 / d[0];
    P.cx1 = c[2]; P.cy1 = c[3]; P.s1 = M_SQRT2 / d[1];
    P.best = 0;
    P.n = n;
    P.ok = n >= a.s && d[0] > 0.0 && d[1] > 0.0;
    P.stop = !P.ok;
    P.drawn = 0;
  }
}

__global__ void __launch_bounds__(1024) geo_prepare_kernel(GeoArgs a) { geo_prepare(a); }

}  // namespace
