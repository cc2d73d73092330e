// Batched RANSAC on the matcher's output (include/geometry_b200.h, which states the algorithm step by step).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  one 1024-thread CTA per pair: ordered compaction of the valid matches, Hartley normalisation
//   per chunk of GEO_CHUNK hypotheses:
//     hyp    one CTA per pair: folds the previous chunk's counts into the pair's best (packed (count + 1, ~h), atomic
//            max), decides the adaptive stop, then one thread per hypothesis draws and solves its sample in double
//     score  (splits, B) CTAs: each streams a slice of the pair's points through shared memory against the chunk's
//            fp32 models, one thread per hypothesis, and adds its inlier counts
//   refit    one CTA per pair: folds the last chunk, least-squares refit on the best hypothesis's inliers, recount,
//            outputs
// A stopped pair's CTAs return at once.  This file is compiled with -fmad=false: every multiply and add rounds on its
// own, as numpy's do in oracle/geometry_oracle.py.
#include "block_scan.cuh"
#include "geo_common.cuh"
#include "lg_internal.h"
#include "ws_bump.h"

namespace {

constexpr int TILE = 1024;  // points per shared-memory tile of the score kernel

struct GeoPair {
  double cx0, cy0, s0, cx1, cy1, s1;  // Hartley normalisation of image 0 and image 1
  unsigned long long best;            // (count + 1) << 32 | ~h of the best hypothesis so far; 0: none
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

struct GeoArgs {
  int B, M, N, kind, s, max_iters, chunks;
  unsigned seed;
  float thr2;
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

// Folds chunk c's counts into the pair's best and decides whether the pair stops.  Called by every thread of a
// GEO_CHUNK-thread CTA; thread t owns hypothesis c * GEO_CHUNK + t.
__device__ void geo_fold(const GeoArgs& a, int b, int c) {
  __shared__ unsigned long long best;
  GeoPair* P = a.w.pair + b;
  const int t = threadIdx.x;
  const bool live = P->stop == 0;
  if (t == 0) best = P->best;
  __syncthreads();
  const int k = a.w.count[(long)b * GEO_CHUNK + t];
  if (live && k >= 0) atomicMax(&best, ((unsigned long long)(k + 1) << 32) | (unsigned)~(unsigned)(c * GEO_CHUNK + t));
  __syncthreads();
  if (t == 0 && live) {
    const int drawn = min((c + 1) * GEO_CHUNK, a.max_iters);
    const int cnt = best ? (int)(best >> 32) - 1 : 0;
    P->best = best;
    P->drawn = drawn;
    P->stop = drawn >= a.max_iters || drawn >= update_num_iters(a.confidence, 1.0 - (double)cnt / P->n, a.s, a.max_iters);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(1024) geo_prepare_kernel(GeoArgs a) {
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
    const bool valid = j >= 0 && j < a.N;
    const int slot = block_scan_step(valid, tid, warp_sums, &carry);
    if (valid) {
      const float2 p0 = reinterpret_cast<const float2*>(a.kpts0)[(long)b * a.M + i];
      const float2 p1 = reinterpret_cast<const float2*>(a.kpts1)[(long)b * a.N + j];
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

__global__ void __launch_bounds__(GEO_CHUNK, 1) geo_hyp_kernel(GeoArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c > 0) geo_fold(a, b, c - 1);
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

__global__ void __launch_bounds__(GEO_CHUNK) geo_score_kernel(GeoArgs a) {
  const int b = blockIdx.y, split = blockIdx.x, t = threadIdx.x;
  const GeoPair& P = a.w.pair[b];
  if (P.stop) return;
  const int lo = (int)((long)P.n * split / gridDim.x), hi = (int)((long)P.n * (split + 1) / gridDim.x);
  int* cnt = a.w.count + (long)b * GEO_CHUNK + t;
  const bool valid = *cnt >= 0;
  float h[9];
  for (int i = 0; i < 9; ++i) h[i] = valid ? a.w.hyp[((long)b * GEO_CHUNK + t) * 9 + i] : 0.f;
  const float4* pts = a.w.pts + (long)b * a.M;
  __shared__ float4 tile[TILE];
  int k = 0;
  for (int base = lo; base < hi; base += TILE) {
    const int m = min(TILE, hi - base);
    __syncthreads();
    for (int i = t; i < m; i += GEO_CHUNK) tile[i] = pts[base + i];
    __syncthreads();
    if (valid)
      for (int i = 0; i < m; ++i) k += geo_err(a.kind, h, tile[i]) < a.thr2;
  }
  if (k) atomicAdd(cnt, k);
}

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
  geo_fold(a, b, a.chunks - 1);
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
  const unsigned hb = ~(unsigned)(key & 0xffffffffu);
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
  if (!cfg || !in || !out) return lg_set_error("geo_estimate: null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return lg_set_error("geo_estimate: ABI version mismatch");
  if (cfg->model != GEO_HOMOGRAPHY && cfg->model != GEO_FUNDAMENTAL) return lg_set_error("geo_estimate: unknown model");
  if (cfg->max_iters < 1 || cfg->max_iters > GEO_MAX_ITERS) return lg_set_error("geo_estimate: max_iters outside [1, 2^24]");
  if (!(cfg->threshold > 0.0) || !isfinite(cfg->threshold)) return lg_set_error("geo_estimate: threshold must be positive");
  if (!(cfg->confidence >= 0.0 && cfg->confidence <= 1.0)) return lg_set_error("geo_estimate: confidence outside [0, 1]");
  if (in->B < 0 || in->M < 0 || in->N < 0) return lg_set_error("geo_estimate: negative size");
  if (in->B == 0) return 0;
  if (!out->model || !out->inliers || !out->num_inliers || !out->success || !out->best_hypothesis || !out->num_hypotheses)
    return lg_set_error("geo_estimate: null output");
  if (in->M > 0 && (!in->kpts0 || !in->matches0 || (in->N > 0 && !in->kpts1))) return lg_set_error("geo_estimate: null input");
  if (!workspace || workspace_bytes < geo_workspace_bytes(in->B, in->M, cfg->max_iters))
    return lg_set_error("geo_estimate: workspace too small");
  GeoArgs a{};
  carve((char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.kind = cfg->model;
  a.s = cfg->model == GEO_HOMOGRAPHY ? 4 : 8;
  a.max_iters = cfg->max_iters;
  a.chunks = (cfg->max_iters + GEO_CHUNK - 1) / GEO_CHUNK;
  a.seed = cfg->seed;
  a.thr2 = (float)(cfg->threshold * cfg->threshold);
  a.confidence = cfg->confidence;
  a.kpts0 = in->kpts0; a.kpts1 = in->kpts1; a.matches0 = in->matches0;
  a.out = *out;
  // enough score CTAs to cover the SMs twice, with at least 128 points per slice
  const int want = (2 * lg_num_sms() + a.B - 1) / a.B;
  int splits = (a.M + 127) / 128;
  if (splits > want) splits = want;
  if (splits < 1) splits = 1;
  const cudaStream_t stream = (cudaStream_t)stream_;
  geo_prepare_kernel<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    geo_hyp_kernel<<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    geo_score_kernel<<<dim3(splits, a.B), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  geo_refit_kernel<<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
