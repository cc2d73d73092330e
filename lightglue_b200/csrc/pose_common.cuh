// The relative pose's shared pieces (include/geometry_b200.h, steps P1-P7): the workspace, the five-point solver, the
// fp32 Sampson error, the K check, the pose candidates of an E and the compaction kernel.  Included by pose_api.cu
// (RANSAC, P1-P8) and lo_pose_api.cu (LO-RANSAC, L1-L8), both compiled with -fmad=false.
#pragma once
#include <stdint.h>

#include "block_scan.cuh"
#include "geo_common.cuh"
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

// geo_hyp_kernel's solver of the relative pose: sample h's five-point solutions E
struct PoseSolver {
  static constexpr int SOLS = ::SOLS, NX = 9, NF = 9;
  static __device__ int s(const PoseArgs&) { return S; }
  static __device__ int solve(const PoseArgs& a, int b, unsigned h, double (*x)[NX]) {
    int id[S];
    if (geo_sample(a.seed, h, a.w.pair[b].n, S, id) < S) return 0;
    return five_point(a.w.pts + (long)b * a.M, id, x);
  }
  static __device__ void pixels(const PoseArgs&, int, const double* x, double* px) {
    for (int i = 0; i < NF; ++i) px[i] = x[i];
  }
};

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

// The two rotations R1, R2 and the translation u3 of E's four pose candidates (header step P7)
__device__ __forceinline__ void pose_candidates(const double* E, double (*Rs)[9], double* ts) {
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
  svd2(E, u1, u2, v1, v2);
  cross3(u1, u2, u3);
  cross3(v1, v2, v3);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      Rs[0][r * 3 + c] = (u2[r] * v1[c] - u1[r] * v2[c]) + u3[r] * v3[c];
      Rs[1][r * 3 + c] = (u1[r] * v2[c] - u2[r] * v1[c]) + u3[r] * v3[c];
    }
  for (int r = 0; r < 3; ++r) ts[r] = u3[r];
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
    float2 p0 = make_float2(0.f, 0.f), p1 = p0;
    if (j >= 0 && j < a.N) {
      p0 = reinterpret_cast<const float2*>(a.kpts0)[(long)b * a.M + i];
      p1 = reinterpret_cast<const float2*>(a.kpts1)[(long)b * a.N + j];
    }
    const bool valid = j >= 0 && j < a.N && finite2(p0) && finite2(p1);
    const int slot = block_scan_step(valid, tid, warp_sums, &carry);
    if (valid) {
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

}  // namespace
