// Batched relative pose on the matcher's output: five-point RANSAC for E, then recoverPose's cheirality test
// (include/geometry_b200.h, steps P1-P8).
//
// Launches, all fixed by (B, M, max_iters):
//   prepare  one 1024-thread CTA per pair: ordered compaction of the valid matches, calibrated coordinates, K checks
//   per chunk of GEO_CHUNK samples:
//     hyp    one CTA per pair: folds the previous chunk's counts into the pair's best (packed (count + 1, ~(h*16 + r)),
//            atomic max), decides the adaptive stop, then one thread per sample solves it: up to 10 fp32 models
//     score  (splits, B) CTAs: each streams a slice of the pair's points through shared memory against every solution
//            of the chunk, one thread per sample, and adds the inlier counts
//   refit    one CTA per pair: folds the last chunk, least-squares refit projected on the essential manifold, recount,
//            E and the inliers
//   pose     one CTA per pair: the four (R, t) of E, linear triangulation of every inlier, the cheirality test
// A stopped pair's CTAs return at once.  Compiled with -fmad=false, like geo_api.cu: oracle/pose_oracle.py takes the same
// steps in numpy.
#include <stdint.h>

#include "block_scan.cuh"
#include "geo_common.cuh"
#include "lg_internal.h"
#include "ws_bump.h"

namespace {

constexpr int S = 5;                  // points per sample
constexpr int SOLS = GEO_MAX_SOLUTIONS;
constexpr int TILE = 1024;            // points per shared-memory tile of the score kernel
constexpr int POSE_THREADS = 256;

struct PosePair {
  double E[9];               // the pair's final E (refit -> pose)
  unsigned long long best;   // (count + 1) << 32 | ~(h * 16 + r) of the best solution so far; 0: none
  float thr2;                // (threshold / mean focal)^2
  int n;                     // valid matches
  int ok;                    // n >= 5 and both K valid
  int stop;                  // no further samples are drawn
  int drawn;                 // samples drawn so far
  int success;               // set by the refit kernel
};

struct PoseWs {
  PosePair* pair;  // [B]
  float4* pts;     // [B, M] compacted calibrated (x0, y0, x1, y1)
  int* idx;        // [B, M] row of matches0 of each compacted match
  float* hyp;      // [B, GEO_CHUNK, SOLS, 9] the current chunk's solutions, fp32
  int* nsol;       // [B, GEO_CHUNK] their number; 0: degenerate or not drawn
  int* count;      // [B, GEO_CHUNK, SOLS] their inlier counts
  uint8_t* flags;  // [B, M] bit c: the point passes candidate c's cheirality test
};

size_t carve(char* base, int B, int M, PoseWs* w) {
  WsBump b{base, 0};
  w->pair = b.take<PosePair>(B);
  w->pts = b.take<float4>((size_t)B * M);
  w->idx = b.take<int>((size_t)B * M);
  w->hyp = b.take<float>((size_t)B * GEO_CHUNK * SOLS * 9);
  w->nsol = b.take<int>((size_t)B * GEO_CHUNK);
  w->count = b.take<int>((size_t)B * GEO_CHUNK * SOLS);
  w->flags = b.take<uint8_t>((size_t)B * M);
  return b.bytes();
}

struct PoseArgs {
  int B, M, N, max_iters, chunks;
  unsigned seed;
  double threshold, confidence, distance;
  const float* kpts0;
  const float* kpts1;
  const int64_t* matches0;
  const double* K0;
  const double* K1;
  PoseWs w;
  GeoPoseOutputs out;
};

// ---- five-point solver (header step P3) ----

// graded monomials x^a y^b z^c of degree <= 3: 1 | x y z | xx xy xz yy yz zz | xxx xxy xxz xyy xyz xzz yyy yyz yzz zzz
__device__ constexpr int MX[20] = {0, 1, 0, 0, 2, 1, 1, 0, 0, 0, 3, 2, 2, 1, 1, 1, 0, 0, 0, 0};
__device__ constexpr int MY[20] = {0, 0, 1, 0, 0, 1, 0, 2, 1, 0, 0, 1, 0, 2, 1, 0, 3, 2, 1, 0};
__device__ constexpr int MZ[20] = {0, 0, 0, 1, 0, 0, 1, 0, 1, 2, 0, 0, 1, 0, 1, 2, 0, 1, 2, 3};
// the ten monomials Gauss-Jordan eliminates, then x*(zz z 1), y*(zz z 1), zzz zz z 1
__device__ constexpr int COLUMNS[20] = {10, 16, 11, 13, 12, 4, 17, 7, 14, 5, 15, 6, 1, 18, 8, 2, 19, 9, 3, 0};

__device__ constexpr int mono_mul(int i, int j) {
  const int a = MX[i] + MX[j], b = MY[i] + MY[j], c = MZ[i] + MZ[j];
  for (int k = 0; k < 20; ++k)
    if (MX[k] == a && MY[k] == b && MZ[k] == c) return k;
  return -1;
}

// out = a * b over the graded monomials (NA, NB, NO slots), terms added in ascending (i, j) from 0
template <int NA, int NB, int NO>
__device__ __forceinline__ void pmul(const double* a, const double* b, double* out) {
#pragma unroll
  for (int k = 0; k < NO; ++k) out[k] = 0.0;
#pragma unroll
  for (int i = 0; i < NA; ++i)
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int k = mono_mul(i, j);
      out[k] = out[k] + a[i] * b[j];
    }
}

// univariate product, ascending powers, terms added in ascending (i, j) from 0
template <int NA, int NB>
__device__ __forceinline__ void umul(const double* a, const double* b, double* out) {
#pragma unroll
  for (int k = 0; k < NA + NB - 1; ++k) out[k] = 0.0;
#pragma unroll
  for (int i = 0; i < NA; ++i)
#pragma unroll
    for (int j = 0; j < NB; ++j) out[i + j] = out[i + j] + a[i] * b[j];
}

__device__ __forceinline__ double horner(const double* p, int deg, double z) {
  double v = p[deg];
  for (int i = deg - 1; i >= 0; --i) v = v * z + p[i];
  return v;
}

__device__ __forceinline__ int sgn3(double v) { return (v > 0.0) - (v < 0.0); }

// Sign changes of the first L members of the Sturm sequence at z (sg: signs given instead of z when non-null)
__device__ int sign_changes(const double (*seq)[11], int L, double z, const int* sg) {
  int prev = 0, v = 0;
  for (int k = 0; k < L; ++k) {
    const int s = sg ? sg[k] : sgn3(horner(seq[k], 10 - k, z));
    if (s != 0 && prev != 0 && s != prev) ++v;
    if (s != 0) prev = s;
  }
  return v;
}

// Unit Frobenius norm (row-major running sum), first largest-magnitude entry positive
__device__ void unit_scale(double* E) {
  double f = 0.0;
  for (int i = 0; i < 9; ++i) f = f + E[i] * E[i];
  f = sqrt(f);
  int k = 0;
  for (int i = 0; i < 9; ++i) {
    E[i] = E[i] / f;
    if (fabs(E[i]) > fabs(E[k])) k = i;
  }
  if (E[k] < 0.0)
    for (int i = 0; i < 9; ++i) E[i] = -E[i];
}

// Real roots of the degree-10 p (ascending), in ascending order; returns their number (header step P3)
__device__ int real_roots(const double* p, double* roots) {
  double amax = 0.0;
  bool finite = true;
  for (int i = 0; i < 11; ++i) {
    finite = finite && isfinite(p[i]);
    amax = fmax(amax, fabs(p[i]));
  }
  if (!finite || !(fabs(p[10]) > GEO_LEAD_EPS * amax)) return 0;
  double seq[11][11];
  for (int i = 0; i < 11; ++i) seq[0][i] = p[i] / p[10];
  double rb = 0.0;
  for (int i = 0; i < 10; ++i) rb = fmax(rb, fabs(seq[0][i]));
  rb = 1.0 + rb;
  for (int i = 0; i < 10; ++i) seq[1][i] = (i + 1.0) * seq[0][i + 1];
  int L = 2;
  for (int k = 2; k < 11; ++k, ++L) {
    const double* a = seq[k - 2];
    const double* b = seq[k - 1];
    const int da = 12 - k, db = 11 - k;
    const double qh = a[da] / b[db];
    double r[10];
    r[0] = a[0];
    for (int i = 1; i < da; ++i) r[i] = a[i] - qh * b[i - 1];
    const double ql = r[da - 1] / b[db];
    bool ok = true;
    double m = 0.0;
    for (int i = 0; i < db; ++i) {
      r[i] = r[i] - ql * b[i];
      ok = ok && isfinite(r[i]);
      m = fmax(m, fabs(r[i]));
    }
    if (!ok || r[db - 1] == 0.0) break;
    for (int i = 0; i < db; ++i) seq[k][i] = -r[i] / m;
  }
  int lneg[11], lpos[11];
  for (int k = 0; k < L; ++k) {
    lpos[k] = sgn3(seq[k][10 - k]);
    lneg[k] = k % 2 == 0 ? lpos[k] : -lpos[k];
  }
  const int vneg = sign_changes(seq, L, 0.0, lneg);
  const int n = max(vneg - sign_changes(seq, L, 0.0, lpos), 0);
  for (int k = 1; k <= n; ++k) {
    double lo = -rb, hi = rb;
    for (int s = 0; s < GEO_STURM_STEPS; ++s) {
      const double mid = 0.5 * (lo + hi);
      if (vneg - sign_changes(seq, L, mid, nullptr) >= k) hi = mid; else lo = mid;
    }
    double z = 0.5 * (lo + hi);
    for (int s = 0; s < GEO_NEWTON_STEPS; ++s) {
      double v = seq[0][10], d = 0.0;
      for (int i = 9; i >= 0; --i) {
        d = d * z + v;
        v = v * z + seq[0][i];
      }
      const double zn = z - v / d;
      if (isfinite(zn)) z = zn;
    }
    roots[k - 1] = z;
  }
  return n;
}

// The solutions of the sample id (unit scale, ascending root); returns their number, 0 for a degenerate sample
__device__ __noinline__ int five_point(const float4* pts, const int* id, double (*sol)[9]) {
  double A[S][9];
  for (int q = 0; q < S; ++q) {
    const float4 p = pts[id[q]];
    const double x = p.x, y = p.y, u = p.z, v = p.w;
    const double r[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
    for (int c = 0; c < 9; ++c) A[q][c] = r[c];
  }
  for (int k = 0; k < S; ++k) {
    int p = k;
    double best = fabs(A[k][k]);
    for (int r = k + 1; r < S; ++r)
      if (fabs(A[r][k]) > best) { best = fabs(A[r][k]); p = r; }
    if (!(best > GEO_PIVOT_EPS)) return 0;
    if (p != k)
      for (int c = k; c < 9; ++c) { const double t = A[k][c]; A[k][c] = A[p][c]; A[p][c] = t; }
    for (int r = k + 1; r < S; ++r) {
      const double f = A[r][k] / A[k][k];
      for (int c = k + 1; c < 9; ++c) A[r][c] = A[r][c] - f * A[k][c];
    }
  }
  double bs[4][9];  // X, Y, Z, W: free column 5, 6, 7, 8 set to 1
  for (int f = 0; f < 4; ++f) {
    for (int c = 0; c < 9; ++c) bs[f][c] = c == 5 + f ? 1.0 : 0.0;
    for (int k = S - 1; k >= 0; --k) {
      double acc = A[k][5 + f];
      for (int c = k + 1; c < S; ++c) acc = acc + A[k][c] * bs[f][c];
      bs[f][k] = -acc / A[k][k];
    }
  }
  for (int i = 0; i < 4; ++i) {  // modified Gram-Schmidt
    for (int j = 0; j < i; ++j) {
      double d = 0.0;
      for (int e = 0; e < 9; ++e) d = d + bs[i][e] * bs[j][e];
      for (int e = 0; e < 9; ++e) bs[i][e] = bs[i][e] - d * bs[j][e];
    }
    double nn = 0.0;
    for (int e = 0; e < 9; ++e) nn = nn + bs[i][e] * bs[i][e];
    nn = sqrt(nn);
    for (int e = 0; e < 9; ++e) bs[i][e] = bs[i][e] / nn;
  }
  double E[9][4];  // E_e = W + x X + y Y + z Z over the monomials 1, x, y, z
  for (int e = 0; e < 9; ++e) { E[e][0] = bs[3][e]; E[e][1] = bs[0][e]; E[e][2] = bs[1][e]; E[e][3] = bs[2][e]; }
  double G[10][20];
  {
    double d[3][10], t0[10], t1[10], a[20], b[20], c[20];
    const int DI[3][4] = {{4, 8, 5, 7}, {3, 8, 5, 6}, {3, 7, 4, 6}};
    for (int r = 0; r < 3; ++r) {
      pmul<4, 4, 10>(E[DI[r][0]], E[DI[r][1]], t0);
      pmul<4, 4, 10>(E[DI[r][2]], E[DI[r][3]], t1);
      for (int k = 0; k < 10; ++k) d[r][k] = t0[k] - t1[k];
    }
    pmul<4, 10, 20>(E[0], d[0], a);
    pmul<4, 10, 20>(E[1], d[1], b);
    pmul<4, 10, 20>(E[2], d[2], c);
    for (int k = 0; k < 20; ++k) a[k] = (a[k] - b[k]) + c[k];
    for (int k = 0; k < 20; ++k) G[0][k] = a[COLUMNS[k]];
  }
  {
    double EE[3][3][10], tr[10], t0[10], t1[10], t2[10], a[20], b[20], c[20];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        pmul<4, 4, 10>(E[3 * i], E[3 * j], t0);
        pmul<4, 4, 10>(E[3 * i + 1], E[3 * j + 1], t1);
        pmul<4, 4, 10>(E[3 * i + 2], E[3 * j + 2], t2);
        for (int k = 0; k < 10; ++k) EE[i][j][k] = (t0[k] + t1[k]) + t2[k];
      }
    for (int k = 0; k < 10; ++k) tr[k] = (EE[0][0][k] + EE[1][1][k]) + EE[2][2][k];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        pmul<10, 4, 20>(EE[i][0], E[j], a);
        pmul<10, 4, 20>(EE[i][1], E[3 + j], b);
        pmul<10, 4, 20>(EE[i][2], E[6 + j], c);
        for (int k = 0; k < 20; ++k) a[k] = (a[k] + b[k]) + c[k];
        pmul<10, 4, 20>(tr, E[3 * i + j], b);
        for (int k = 0; k < 20; ++k) c[k] = 2.0 * a[k] - b[k];
        for (int k = 0; k < 20; ++k) G[1 + 3 * i + j][k] = c[COLUMNS[k]];
      }
  }
  double amax = 0.0;
  bool finite = true;
  for (int r = 0; r < 10; ++r)
    for (int c = 0; c < 20; ++c) {
      finite = finite && isfinite(G[r][c]);
      amax = fmax(amax, fabs(G[r][c]));
    }
  if (!finite) return 0;
  for (int k = 0; k < 10; ++k) {  // Gauss-Jordan with partial pivoting
    int p = k;
    double best = fabs(G[k][k]);
    for (int r = k + 1; r < 10; ++r)
      if (fabs(G[r][k]) > best) { best = fabs(G[r][k]); p = r; }
    if (!(best > GEO_PIVOT_EPS * amax)) return 0;
    if (p != k)
      for (int c = k; c < 20; ++c) { const double t = G[k][c]; G[k][c] = G[p][c]; G[p][c] = t; }
    const double piv = G[k][k];
    for (int c = k + 1; c < 20; ++c) G[k][c] = G[k][c] / piv;
    for (int r = 0; r < 10; ++r) {
      if (r == k) continue;
      const double f = G[r][k];
      for (int c = k + 1; c < 20; ++c) G[r][c] = G[r][c] - f * G[k][c];
    }
  }
  // rows 4 - z*5, 6 - z*7, 8 - z*9: x*px(z) + y*py(z) + p1(z) = 0, the hidden-variable 3x3
  double px[3][4], py[3][4], p1[3][5];
  for (int h = 0; h < 3; ++h) {
    const double* a = G[4 + 2 * h] + 10;
    const double* b = G[5 + 2 * h] + 10;
    const double X4[4] = {a[2], a[1] - b[2], a[0] - b[1], -b[0]};
    const double Y4[4] = {a[5], a[4] - b[5], a[3] - b[4], -b[3]};
    const double O5[5] = {a[9], a[8] - b[9], a[7] - b[8], a[6] - b[7], -b[6]};
    for (int i = 0; i < 4; ++i) { px[h][i] = X4[i]; py[h][i] = Y4[i]; }
    for (int i = 0; i < 5; ++i) p1[h][i] = O5[i];
  }
  double c0[8], c1[8], c2[7], det[11];
  {
    double t0[8], t1[8];
    umul<4, 5>(py[1], p1[2], t0);
    umul<5, 4>(p1[1], py[2], t1);
    for (int i = 0; i < 8; ++i) c0[i] = t0[i] - t1[i];
    umul<4, 5>(px[1], p1[2], t0);
    umul<5, 4>(p1[1], px[2], t1);
    for (int i = 0; i < 8; ++i) c1[i] = t0[i] - t1[i];
    umul<4, 4>(px[1], py[2], t0);
    umul<4, 4>(py[1], px[2], t1);
    for (int i = 0; i < 7; ++i) c2[i] = t0[i] - t1[i];
    double a[11], b[11], c[11];
    umul<4, 8>(px[0], c0, a);
    umul<4, 8>(py[0], c1, b);
    umul<5, 7>(p1[0], c2, c);
    for (int i = 0; i < 11; ++i) det[i] = (a[i] - b[i]) + c[i];
  }
  double roots[10];
  const int nr = real_roots(det, roots);
  int ns = 0;
  for (int k = 0; k < nr; ++k) {
    const double z = roots[k];
    double Bm[3][3];
    for (int h = 0; h < 3; ++h) {
      Bm[h][0] = horner(px[h], 3, z);
      Bm[h][1] = horner(py[h], 3, z);
      Bm[h][2] = horner(p1[h], 4, z);
    }
    const int PR[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    double cb[3];
    for (int w = 0; w < 3; ++w) {
      const double* a = Bm[PR[w][0]];
      const double* b = Bm[PR[w][1]];
      const double cr[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
      if (w == 0 || fabs(cr[2]) > fabs(cb[2]))
        for (int i = 0; i < 3; ++i) cb[i] = cr[i];
    }
    const double xs = cb[0] / cb[2], ys = cb[1] / cb[2];
    double* e = sol[ns];
    double f = 0.0;
    for (int i = 0; i < 9; ++i) {
      e[i] = ((xs * bs[0][i] + ys * bs[1][i]) + z * bs[2][i]) + bs[3][i];
      f = f + e[i] * e[i];
    }
    if (!(isfinite(f) && f > 0.0)) continue;
    unit_scale(e);
    ++ns;
  }
  return ns;
}

// fp32 squared Sampson error of one correspondence (header step P4)
__device__ __forceinline__ float sampson(const float* g, float4 p) {
  const float a0 = (g[0] * p.x + g[1] * p.y) + g[2], a1 = (g[3] * p.x + g[4] * p.y) + g[5];
  const float a2 = (g[6] * p.x + g[7] * p.y) + g[8];
  const float d = (p.z * a0 + p.w * a1) + a2;
  const float b0 = (g[0] * p.z + g[3] * p.w) + g[6], b1 = (g[1] * p.z + g[4] * p.w) + g[7];
  return (d * d) / (((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1);
}

__device__ bool k_valid(const double* K) {
  bool finite = true;
  for (int i = 0; i < 9; ++i) finite = finite && isfinite(K[i]);
  return finite && K[0] > 0.0 && K[4] > 0.0 && K[6] == 0.0 && K[7] == 0.0 && K[8] == 1.0;
}

// Folds chunk c's counts into the pair's best and decides whether the pair stops.  Called by every thread of a
// GEO_CHUNK-thread CTA; thread t owns sample c * GEO_CHUNK + t.
__device__ void pose_fold(const PoseArgs& a, int b, int c) {
  __shared__ unsigned long long best;
  PosePair* P = a.w.pair + b;
  const int t = threadIdx.x;
  const bool live = P->stop == 0;
  if (t == 0) best = P->best;
  __syncthreads();
  const int ns = a.w.nsol[(long)b * GEO_CHUNK + t];
  const unsigned h = c * GEO_CHUNK + t;
  for (int r = 0; live && r < ns; ++r) {
    const int k = a.w.count[((long)b * GEO_CHUNK + t) * SOLS + r];
    atomicMax(&best, ((unsigned long long)(k + 1) << 32) | (unsigned)~(h * 16u + (unsigned)r));
  }
  __syncthreads();
  if (t == 0 && live) {
    const int drawn = min((c + 1) * GEO_CHUNK, a.max_iters);
    const int cnt = best ? (int)(best >> 32) - 1 : 0;
    P->best = best;
    P->drawn = drawn;
    P->stop = drawn >= a.max_iters || drawn >= update_num_iters(a.confidence, 1.0 - (double)cnt / P->n, S, a.max_iters);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(1024) pose_prepare_kernel(PoseArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  const double* K0 = a.K0 + (long)b * 9;
  const double* K1 = a.K1 + (long)b * 9;
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
      const double y0 = ((double)p0.y - K0[5]) / K0[4], x0 = (((double)p0.x - K0[2]) - K0[1] * y0) / K0[0];
      const double y1 = ((double)p1.y - K1[5]) / K1[4], x1 = (((double)p1.x - K1[2]) - K1[1] * y1) / K1[0];
      pts[slot] = make_float4((float)x0, (float)y0, (float)x1, (float)y1);
      a.w.idx[(long)b * a.M + slot] = i;
    }
  }
  __syncthreads();
  if (tid == 0) {
    PosePair& P = a.w.pair[b];
    const double f = (((K0[0] + K0[4]) + K1[0]) + K1[4]) / 4.0;
    const double t = a.threshold / f;
    P.thr2 = (float)(t * t);
    P.best = 0;
    P.n = carry;
    P.ok = carry >= S && k_valid(K0) && k_valid(K1);
    P.stop = !P.ok;
    P.drawn = 0;
    P.success = 0;
  }
}

__global__ void __launch_bounds__(GEO_CHUNK, 1) pose_hyp_kernel(PoseArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c > 0) pose_fold(a, b, c - 1);
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

__global__ void __launch_bounds__(GEO_CHUNK) pose_score_kernel(PoseArgs a) {
  const int b = blockIdx.y, split = blockIdx.x, t = threadIdx.x;
  const PosePair& P = a.w.pair[b];
  if (P.stop) return;
  const int lo = (int)((long)P.n * split / gridDim.x), hi = (int)((long)P.n * (split + 1) / gridDim.x);
  const int ns = a.w.nsol[(long)b * GEO_CHUNK + t];
  const float* hm = a.w.hyp + ((long)b * GEO_CHUNK + t) * SOLS * 9;
  const float thr2 = P.thr2;
  float g[SOLS][9];
  int k[SOLS];
#pragma unroll
  for (int r = 0; r < SOLS; ++r) {
    k[r] = 0;
#pragma unroll
    for (int i = 0; i < 9; ++i) g[r][i] = r < ns ? hm[r * 9 + i] : 0.f;
  }
  const float4* pts = a.w.pts + (long)b * a.M;
  __shared__ float4 tile[TILE];
  for (int base = lo; base < hi; base += TILE) {
    const int m = min(TILE, hi - base);
    __syncthreads();
    for (int i = t; i < m; i += GEO_CHUNK) tile[i] = pts[base + i];
    __syncthreads();
    for (int i = 0; i < m; ++i) {
      const float4 p = tile[i];
#pragma unroll
      for (int r = 0; r < SOLS; ++r)
        if (r < ns) k[r] += sampson(g[r], p) < thr2;
    }
  }
#pragma unroll
  for (int r = 0; r < SOLS; ++r)
    if (r < ns && k[r]) atomicAdd(a.w.count + ((long)b * GEO_CHUNK + t) * SOLS + r, k[r]);
}

// One-sided Jacobi of a row-major 3x3 E: unit u1, u2 of its two larger columns (ascending index) and v1, v2
__device__ void svd2(const double* E, double* u1, double* u2, double* v1, double* v2) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) A[i] = E[i];
  jacobi_columns3(A, V);
  double nrm[3];
  for (int j = 0; j < 3; ++j) {
    double nj = 0.0;
    for (int i = 0; i < 3; ++i) nj = nj + A[i * 3 + j] * A[i * 3 + j];
    nrm[j] = nj;
  }
  int m = 0;
  for (int j = 1; j < 3; ++j)
    if (nrm[j] < nrm[m]) m = j;
  const int i0 = m == 0 ? 1 : 0, j0 = m == 2 ? 1 : 2;
  const double si = sqrt(nrm[i0]), sj = sqrt(nrm[j0]);
  for (int r = 0; r < 3; ++r) {
    u1[r] = A[r * 3 + i0] / si;
    u2[r] = A[r * 3 + j0] / sj;
    v1[r] = V[r * 3 + i0];
    v2[r] = V[r * 3 + j0];
  }
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

__global__ void __launch_bounds__(RED, 1) pose_refit_kernel(PoseArgs a) {
  const int b = blockIdx.x, t = threadIdx.x;
  pose_fold(a, b, a.chunks - 1);
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
  if (t == 0) {
    double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
    svd2(P.E, u1, u2, v1, v2);
    cross3(u1, u2, u3);
    cross3(v1, v2, v3);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        Rs[0][r * 3 + c] = (u2[r] * v1[c] - u1[r] * v2[c]) + u3[r] * v3[c];
        Rs[1][r * 3 + c] = (u1[r] * v2[c] - u2[r] * v1[c]) + u3[r] * v3[c];
      }
    for (int r = 0; r < 3; ++r) ts[r] = u3[r];
  }
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
  if (!cfg || !in || !out) return lg_set_error("geo_relative_pose: null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return lg_set_error("geo_relative_pose: ABI version mismatch");
  if (cfg->max_iters < 1 || cfg->max_iters > GEO_MAX_ITERS)
    return lg_set_error("geo_relative_pose: max_iters outside [1, 2^24]");
  if (!(cfg->threshold > 0.0) || !isfinite(cfg->threshold))
    return lg_set_error("geo_relative_pose: threshold must be positive");
  if (!(cfg->confidence >= 0.0 && cfg->confidence <= 1.0))
    return lg_set_error("geo_relative_pose: confidence outside [0, 1]");
  if (!(cfg->distance_threshold > 0.0) || !isfinite(cfg->distance_threshold))
    return lg_set_error("geo_relative_pose: distance_threshold must be positive");
  if (in->B < 0 || in->M < 0 || in->N < 0) return lg_set_error("geo_relative_pose: negative size");
  if (in->B == 0) return 0;
  if (!out->E || !out->R || !out->t || !out->inliers || !out->num_inliers || !out->pose_inliers ||
      !out->num_pose_inliers || !out->success || !out->best_hypothesis || !out->best_solution || !out->num_hypotheses)
    return lg_set_error("geo_relative_pose: null output");
  if (!in->K0 || !in->K1) return lg_set_error("geo_relative_pose: null intrinsics");
  if (in->M > 0 && (!in->kpts0 || !in->matches0 || (in->N > 0 && !in->kpts1)))
    return lg_set_error("geo_relative_pose: null input");
  if (!workspace || workspace_bytes < geo_pose_workspace_bytes(in->B, in->M, cfg->max_iters))
    return lg_set_error("geo_relative_pose: workspace too small");
  PoseArgs a{};
  carve((char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255), in->B, in->M, &a.w);
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.max_iters = cfg->max_iters;
  a.chunks = (cfg->max_iters + GEO_CHUNK - 1) / GEO_CHUNK;
  a.seed = cfg->seed;
  a.threshold = cfg->threshold;
  a.confidence = cfg->confidence;
  a.distance = cfg->distance_threshold;
  a.kpts0 = in->kpts0; a.kpts1 = in->kpts1; a.matches0 = in->matches0;
  a.K0 = in->K0; a.K1 = in->K1;
  a.out = *out;
  // enough score CTAs to cover the SMs twice, with at least 128 points per slice
  const int want = (2 * lg_num_sms() + a.B - 1) / a.B;
  int splits = (a.M + 127) / 128;
  if (splits > want) splits = want;
  if (splits < 1) splits = 1;
  const cudaStream_t stream = (cudaStream_t)stream_;
  pose_prepare_kernel<<<a.B, 1024, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  for (int c = 0; c < a.chunks; ++c) {
    pose_hyp_kernel<<<a.B, GEO_CHUNK, 0, stream>>>(a, c);
    LG_CHECK_LAUNCH();
    pose_score_kernel<<<dim3(splits, a.B), GEO_CHUNK, 0, stream>>>(a);
    LG_CHECK_LAUNCH();
  }
  pose_refit_kernel<<<a.B, RED, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  pose_kernel<<<a.B, POSE_THREADS, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
