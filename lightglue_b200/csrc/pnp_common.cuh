// The absolute-pose pieces shared by the plain (pnp_api.cu, header steps A1-A8) and the LO-RANSAC estimator
// (lo_pnp_api.cu, LA1-LA8), both compiled with -fmad=false: the workspace, the Lambda Twist solver, the projection,
// the fp32 reprojection test, the residuals and pose update of the Levenberg-Marquardt steps, and their counterparts
// with lens distortion (AD1-AD4) or the fisheye lens (AE1-AE4); then the three camera policies, Pinhole, Distorted and
// Fisheye, that route to one or the other, and the solver and compaction kernel templated on them.
#pragma once
#include <stdint.h>

#include "block_scan.cuh"
#include "camera_common.cuh"
#include "geo_common.cuh"
#include "geo_lm.cuh"
#include "lg_internal.h"
#include "ws_bump.h"

namespace {

constexpr int S = 3;                   // points per sample
constexpr int SOLS = GEO_PNP_MAX_SOLUTIONS;
constexpr int TILE = 512;              // points per shared-memory tile of the score kernel

struct PnpPair {
  float P[12];               // the final K0 [R | t], fp32 (final -> mask)
  unsigned long long best;   // (count + 1) << 32 | ~(h * 16 + r) of the best solution so far; 0: none
  float thr2;                // threshold^2
  int n;                     // valid matches
  int ok;                    // n >= 3 and K0 valid
  int stop;                  // no further samples are drawn
  int drawn;                 // samples drawn so far
  int success;               // set by the final kernel
};

struct PnpWs {
  PnpPair* pair;   // [B]
  float4* pts;     // [B, M] compacted (u, v, x, y): pixel and calibrated coordinates
  float4* wld;     // [B, M] compacted world point (X, Y, Z, 0)
  int* slot;       // [B, M] compacted slot of each row of matches0, -1 for an invalid match
  float* hyp;      // [B, GEO_CHUNK, SOLS, 12] the current chunk's projections, fp32
  int* nsol;       // [B, GEO_CHUNK] their number; 0: degenerate or not drawn
  int* count;      // [B, GEO_CHUNK, SOLS] their inlier counts
};

size_t carve(char* base, int B, int M, PnpWs* w) {
  WsBump b{base, 0};
  w->pair = b.take<PnpPair>(B);
  w->pts = b.take<float4>((size_t)B * M);
  w->wld = b.take<float4>((size_t)B * M);
  w->slot = b.take<int>((size_t)B * M);
  w->hyp = b.take<float>((size_t)B * GEO_CHUNK * SOLS * 12);
  w->nsol = b.take<int>((size_t)B * GEO_CHUNK);
  w->count = b.take<int>((size_t)B * GEO_CHUNK * SOLS);
  return b.bytes();
}

struct PnpArgs {
  int B, M, N, max_iters, chunks;
  unsigned seed;
  double threshold, confidence;
  const float* kpts0;
  const float* points3d1;
  const int64_t* matches0;
  const double* K0;
  PnpWs w;
  GeoPnpOutputs out;
  const double* dist0;  // [B, nd]: the coefficients, read by the Distorted camera only
  int nd;
};

__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Both roots of z^2 + b z + c, the larger-magnitude one first; a negative discriminant counts as 0 (header step A4)
__device__ __forceinline__ void root2(double b, double c, double* r1, double* r2) {
  const double y = sqrt(fmax(b * b - 4.0 * c, 0.0));
  const double q = -0.5 * (b + (b >= 0.0 ? y : -y));
  *r1 = q;
  *r2 = c / q;
}

__device__ __forceinline__ double cubic(double g, double cb, double cc, double cd) { return ((g + cb) * g + cc) * g + cd; }

// Lambda Twist P3P on the calibrated (x, y) in pts[id[k]].z/w and the world points wlds[id[k]] (header step A4).
// Writes the kept solutions' R (row-major, 0-8) and t (9-11) in the solver's order; returns their number.
__device__ __noinline__ int p3p(const float4* pts, const float4* wlds, const int* id, double (*sol)[12]) {
  double y[3][3], X[3][3];
  for (int k = 0; k < 3; ++k) {
    const float4 p = pts[id[k]], q = wlds[id[k]];
    const double xx = p.z, yy = p.w;
    const double n = sqrt(xx * xx + yy * yy + 1.0);
    y[k][0] = xx / n;
    y[k][1] = yy / n;
    y[k][2] = 1.0 / n;
    X[k][0] = q.x;
    X[k][1] = q.y;
    X[k][2] = q.z;
  }
  const double b12 = -2.0 * dot3(y[0], y[1]), b13 = -2.0 * dot3(y[0], y[2]), b23 = -2.0 * dot3(y[1], y[2]);
  double d12[3], d13[3], d23[3], nrm[3];
  for (int i = 0; i < 3; ++i) {
    d12[i] = X[0][i] - X[1][i];
    d13[i] = X[0][i] - X[2][i];
    d23[i] = X[1][i] - X[2][i];
  }
  const double a12 = dot3(d12, d12), a13 = dot3(d13, d13), a23 = dot3(d23, d23);
  cross3(d12, d13, nrm);
  if (!(dot3(nrm, nrm) > GEO_PNP_COLLINEAR_EPS * (a12 * a13))) return 0;
  const double c31 = -0.5 * b13, c23 = -0.5 * b23, c12 = -0.5 * b12;
  const double blob = c12 * c23 * c31 - 1.0;
  const double s31 = 1.0 - c31 * c31, s23 = 1.0 - c23 * c23, s12 = 1.0 - c12 * c12;
  const double p3 = a13 * (a23 * s31 - a13 * s23);
  const double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31;
  const double p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23);
  const double p0 = a12 * (a12 * s23 - a23 * s12);
  const double cb = p2 / p3, cc = p1 / p3, cd = p0 / p3;
  if (!(isfinite(cb) && isfinite(cc) && isfinite(cd))) return 0;
  // one real root of the monic cubic: bisection on a bracket holding exactly one root, then Newton
  const double rb = 1.0 + fmax(fmax(fabs(cb), fabs(cc)), fabs(cd));
  double lo = -rb, hi = rb;
  const double disc = cb * cb - 3.0 * cc;
  if (disc >= 0.0) {
    const double v = sqrt(fmax(disc, 0.0));
    const double t1 = (-cb - v) / 3.0;
    if (cubic(t1, cb, cc, cd) > 0.0) hi = t1; else lo = (-cb + v) / 3.0;
  }
  for (int s = 0; s < GEO_PNP_BISECT_STEPS; ++s) {
    const double mid = 0.5 * (lo + hi);
    if (cubic(mid, cb, cc, cd) > 0.0) hi = mid; else lo = mid;
  }
  double g = 0.5 * (lo + hi);
  for (int s = 0; s < GEO_PNP_NEWTON_STEPS; ++s) {
    const double gn = g - cubic(g, cb, cc, cd) / ((3.0 * g + 2.0 * cb) * g + cc);
    if (isfinite(gn)) g = gn;
  }
  // the degenerate conic A = D1 + g D2 and its two eigenvectors of nonzero eigenvalue
  const double A00 = a23 * (1.0 - g);
  const double A01 = a23 * b12 * 0.5;
  const double A02 = a23 * b13 * g * -0.5;
  const double A11 = a23 - a12 + a13 * g;
  const double A12 = b23 * (a13 * g - a12) * 0.5;
  const double A22 = g * (a13 - a23) - a12;
  double e1, e2;
  root2(-A00 - A11 - A22, -(A01 * A01) - A02 * A02 - A12 * A12 + A00 * (A11 + A22) + A11 * A22, &e1, &e2);
  if (fabs(e1) < fabs(e2)) { const double tmp = e1; e1 = e2; e2 = tmp; }
  const double mx = -(A00 * A11);
  const double pr0 = A01 * A12 - A02 * A11;
  const double pr1 = A01 * A02 - A00 * A12;
  double V[2][3];
  for (int k = 0; k < 2; ++k) {
    const double e = k == 0 ? e1 : e2;
    const double tmp = 1.0 / (e * (A00 + A11) + mx - e * e + A01 * A01);
    const double a1 = -(e * A02 + pr0) * tmp;
    const double a2 = -(e * A12 + pr1) * tmp;
    const double rn = 1.0 / sqrt(a1 * a1 + a2 * a2 + 1.0);
    V[k][0] = a1 * rn;
    V[k][1] = a2 * rn;
    V[k][2] = rn;
  }
  const double sv = sqrt(fmax(0.0, -e2 / e1));
  // the inverse of X = [d12 d13 d12 x d13] by cofactors
  const double x[3][3] = {{d12[0], d13[0], nrm[0]}, {d12[1], d13[1], nrm[1]}, {d12[2], d13[2], nrm[2]}};
  const double C[3][3] = {
      {x[1][1] * x[2][2] - x[1][2] * x[2][1], x[1][2] * x[2][0] - x[1][0] * x[2][2], x[1][0] * x[2][1] - x[1][1] * x[2][0]},
      {x[0][2] * x[2][1] - x[0][1] * x[2][2], x[0][0] * x[2][2] - x[0][2] * x[2][0], x[0][1] * x[2][0] - x[0][0] * x[2][1]},
      {x[0][1] * x[1][2] - x[0][2] * x[1][1], x[0][2] * x[1][0] - x[0][0] * x[1][2], x[0][0] * x[1][1] - x[0][1] * x[1][0]}};
  const double det = x[0][0] * C[0][0] + x[0][1] * C[0][1] + x[0][2] * C[0][2];
  double Xi[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Xi[i][j] = C[j][i] / det;
  int ns = 0;
  for (int sg = 0; sg < 2; ++sg) {
    const double s = sg == 0 ? sv : -sv;
    const double w2 = 1.0 / (s * V[1][0] - V[0][0]);
    const double w0 = (V[0][1] - s * V[1][1]) * w2;
    const double w1 = (V[0][2] - s * V[1][2]) * w2;
    const double ia = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
    const double qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * ia;
    const double qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * ia;
    if (!(qb * qb - 4.0 * qc >= 0.0)) continue;
    double taus[2];
    root2(qb, qc, &taus[0], &taus[1]);
    for (int k = 0; k < 2; ++k) {
      const double tau = taus[k];
      if (!(tau > 0.0)) continue;
      const double d = a23 / (tau * (b23 + tau) + 1.0);
      if (!(d > 0.0)) continue;
      double l2 = sqrt(d);
      double l3 = tau * l2;
      double l1 = w0 * l2 + w1 * l3;
      if (!(l1 >= 0.0)) continue;
      for (int it = 0; it < GEO_PNP_GN_STEPS; ++it) {
        const double r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12;
        const double r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13;
        const double r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23;
        const double v0 = 2.0 * l1 + b12 * l2, v1 = 2.0 * l2 + b12 * l1;
        const double v3 = 2.0 * l1 + b13 * l3, v5 = 2.0 * l3 + b13 * l1;
        const double v7 = 2.0 * l2 + b23 * l3, v8 = 2.0 * l3 + b23 * l2;
        const double dt = -(v0 * v5 * v7) - v1 * v3 * v8;
        const double j0 = -(v5 * v7) * r1 - v1 * v8 * r2 + v1 * v5 * r3;
        const double j1 = -(v3 * v8) * r1 + v0 * v8 * r2 - v0 * v5 * r3;
        const double j2 = v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3;
        const double n1 = l1 - j0 / dt, n2 = l2 - j1 / dt, n3 = l3 - j2 / dt;
        if (isfinite(n1) && isfinite(n2) && isfinite(n3)) { l1 = n1; l2 = n2; l3 = n3; }
      }
      const double lam[3] = {l1, l2, l3};
      double ry[3][3];
      for (int q = 0; q < 3; ++q)
        for (int i = 0; i < 3; ++i) ry[q][i] = y[q][i] * lam[q];
      double yd1[3], yd2[3], yc[3];
      for (int i = 0; i < 3; ++i) {
        yd1[i] = ry[0][i] - ry[1][i];
        yd2[i] = ry[0][i] - ry[2][i];
      }
      cross3(yd1, yd2, yc);
      double* R = sol[ns];
      double* t = sol[ns] + 9;
      bool fin = true;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
          R[i * 3 + j] = yd1[i] * Xi[0][j] + yd2[i] * Xi[1][j] + yc[i] * Xi[2][j];
          fin = fin && isfinite(R[i * 3 + j]);
        }
      for (int i = 0; i < 3; ++i) {
        t[i] = ry[0][i] - (R[i * 3] * X[0][0] + R[i * 3 + 1] * X[0][1] + R[i * 3 + 2] * X[0][2]);
        fin = fin && isfinite(t[i]);
      }
      if (fin) ++ns;
    }
  }
  return ns;
}

// P = K [R | t] (header step A5), P_ij = (K_i0*M_0j + K_i1*M_1j) + K_i2*M_2j
__device__ __forceinline__ void projection(const double* K, const double* R, const double* t, double* P) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) {
      const double m0 = j < 3 ? R[j] : t[0], m1 = j < 3 ? R[3 + j] : t[1], m2 = j < 3 ? R[6 + j] : t[2];
      P[i * 4 + j] = K[3 * i] * m0 + K[3 * i + 1] * m1 + K[3 * i + 2] * m2;
    }
}

// fp32 inlier test of one point (header step A5): depth w > 0 and squared reprojection error below thr2
__device__ __forceinline__ bool reproj_inlier(const float* g, float4 p, float4 q, float thr2) {
  const float w = g[8] * q.x + g[9] * q.y + g[10] * q.z + g[11];
  const float iw = 1.f / w;
  const float du = p.x - (g[0] * q.x + g[1] * q.y + g[2] * q.z + g[3]) * iw;
  const float dv = p.y - (g[4] * q.x + g[5] * q.y + g[6] * q.z + g[7]) * iw;
  return w > 0.f && du * du + dv * dv < thr2;
}

// The same point's fp32 error for the MSAC score (header step LA3): du * du + dv * dv in front of the camera, +inf
// behind it, so that lo_term counts it as an outlier.  e < thr2 exactly when reproj_inlier holds.
__device__ __forceinline__ float reproj_err(const float* g, float4 p, float4 q) {
  const float w = g[8] * q.x + g[9] * q.y + g[10] * q.z + g[11];
  const float iw = 1.f / w;
  const float du = p.x - (g[0] * q.x + g[1] * q.y + g[2] * q.z + g[3]) * iw;
  const float dv = p.y - (g[4] * q.x + g[5] * q.y + g[6] * q.z + g[7]) * iw;
  return w > 0.f ? du * du + dv * dv : INFINITY;
}

// The reprojection residual (ru, rv) of world point q at pixel p (u, v) under K [R | t], and what its Jacobian needs
struct PnpResidual {
  double Xc[3];  // the camera-frame point; Xc[2] is its depth
  double iz, pu, bx, ru, rv;
};

__device__ __forceinline__ PnpResidual pnp_residual(const double* K, const double* R, const double* t, float4 p,
                                                    float4 q) {
  const double fx = K[0], sk = K[1], cx = K[2], fy = K[4], cy = K[5];
  const double u = p.x, v = p.y, W[3] = {q.x, q.y, q.z};
  PnpResidual e;
  for (int i = 0; i < 3; ++i) e.Xc[i] = R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i];
  e.iz = 1.0 / e.Xc[2];
  const double ax = e.Xc[0] * e.iz;
  e.bx = e.Xc[1] * e.iz;
  e.pu = fx * ax + sk * e.bx;
  e.ru = e.pu + cx - u;
  e.rv = fy * e.bx + cy - v;
  return e;
}

// Adds a point's J^T J upper triangle (acc[0..20]) and J^T r (acc[21..26]) in A7's parameters, from its camera-frame
// point Xc, the gradients gu, gv of its residuals (ru, rv) with respect to Xc, and the residuals (header step A7)
__device__ __forceinline__ void pnp_add_rows(const double* Xc, const double* gu, const double* gv, double ru, double rv,
                                             double* acc) {
  const double ju[6] = {gu[2] * Xc[1] - gu[1] * Xc[2], gu[0] * Xc[2] - gu[2] * Xc[0], gu[1] * Xc[0] - gu[0] * Xc[1],
                        gu[0], gu[1], gu[2]};
  const double jv[6] = {gv[2] * Xc[1] - gv[1] * Xc[2], gv[0] * Xc[2] - gv[2] * Xc[0], gv[1] * Xc[0] - gv[0] * Xc[1],
                        gv[0], gv[1], gv[2]};
  int k = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j, ++k) acc[k] = acc[k] + (ju[i] * ju[j] + jv[i] * jv[j]);
#pragma unroll
  for (int i = 0; i < 6; ++i) acc[21 + i] = acc[21 + i] + (ju[i] * ru + jv[i] * rv);
}

// The same sums of a pinhole residual (header step A7)
__device__ __forceinline__ void pnp_add_normal(const double* K, const PnpResidual& e, double* acc) {
  const double fx = K[0], sk = K[1], fy = K[4];
  const double gu[3] = {fx * e.iz, sk * e.iz, -(e.pu * e.iz)};
  const double gv[3] = {0.0, fy * e.iz, -(fy * e.bx * e.iz)};
  pnp_add_rows(e.Xc, gu, gv, e.ru, e.rv, acc);
}

// R' = Q R, t' = Q t + d[3..5], Q of the unit quaternion (1, d[0..2] / 2) / norm
__device__ void lm_update(const double* R, const double* t, const double* d, double* Rn, double* tn) {
  double Q[9];
  quat_rotation(d, Q);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rn[3 * i + j] = Q[3 * i] * R[j] + Q[3 * i + 1] * R[3 + j] + Q[3 * i + 2] * R[6 + j];
    tn[i] = Q[3 * i] * t[0] + Q[3 * i + 1] * t[1] + Q[3 * i + 2] * t[2] + d[3 + i];
  }
}

// The kernel arguments of an entry point's configuration, inputs and coefficients (none for the pinhole camera); the
// caller carves the workspace and sets out
inline PnpArgs pnp_args(const GeoPnpConfig* cfg, const GeoPnpInputs* in, const double* dist0, int nd) {
  PnpArgs a{};
  a.B = in->B; a.M = in->M; a.N = in->N;
  a.max_iters = cfg->max_iters;
  a.chunks = geo_chunks(cfg->max_iters);
  a.seed = cfg->seed;
  a.threshold = cfg->threshold;
  a.confidence = cfg->confidence;
  a.kpts0 = in->kpts0; a.points3d1 = in->points3d1; a.matches0 = in->matches0;
  a.K0 = in->K0;
  a.dist0 = dist0;
  a.nd = nd;
  return a;
}

// ---- the lens distortion primitives (header steps AD1-AD4) ----

constexpr int PNP_UNDISTORT_ITERS = 5;  // AD1: cv2.solvePnP's undistortion

__device__ __forceinline__ const double* pair_dist(const PnpArgs& a, int b) { return a.dist0 + (long)b * a.nd; }

// Pair b's K0 and coefficients in T: double for the LM, float for AD2's test
template <class T>
__device__ __forceinline__ Camera<T> pair_camera(const PnpArgs& a, int b) {
  return load_camera<T>(a.K0 + (long)b * 9, pair_dist(a, b), a.nd);
}

// M = [R | t] as a row-major 3x4, the model AD2 rounds to float
__device__ __forceinline__ void rt_matrix(const double* x, double* M) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) M[i * 4 + j] = x[i * 3 + j];
    M[i * 4 + 3] = x[9 + i];
  }
}

// AD2's (AE2's) fp32 error of one point under the float [R | t] g: du * du + dv * dv in distorted pixels of Lens in
// front of the camera, +inf behind it (so that an inlier has err < thr2 and lo_term counts the others as outliers)
template <class Lens>
__device__ __forceinline__ float dist_reproj_err(const float* g, const Camera<float>& c, float4 p, float4 q) {
  const float X0 = g[0] * q.x + g[1] * q.y + g[2] * q.z + g[3];
  const float X1 = g[4] * q.x + g[5] * q.y + g[6] * q.z + g[7];
  const float w = g[8] * q.x + g[9] * q.y + g[10] * q.z + g[11];
  float xd, yd;
  Lens::distort(c.d, X0 / w, X1 / w, &xd, &yd);
  const float du = p.x - (c.fx * xd + c.s * yd + c.cx), dv = p.y - (c.fy * yd + c.cy);
  return w > 0.f ? du * du + dv * dv : INFINITY;
}

// AD3's (AE3's) residual (ru, rv) of world point q at pixel p, in distorted pixels of Lens, and what its Jacobian needs
struct PnpDistResidual {
  double Xc[3];  // the camera-frame point; Xc[2] is its depth
  double iz, a, b, ru, rv;
};

template <class Lens>
__device__ __forceinline__ PnpDistResidual pnp_dist_residual(const Camera<double>& c, const double* R, const double* t,
                                                             float4 p, float4 q) {
  const double W[3] = {q.x, q.y, q.z};
  PnpDistResidual e;
  for (int i = 0; i < 3; ++i) e.Xc[i] = R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i];
  e.iz = 1.0 / e.Xc[2];
  e.a = e.Xc[0] * e.iz;
  e.b = e.Xc[1] * e.iz;
  double xd, yd;
  Lens::distort(c.d, e.a, e.b, &xd, &yd);
  e.ru = c.fx * xd + c.s * yd + c.cx - (double)p.x;
  e.rv = c.fy * yd + c.cy - (double)p.y;
  return e;
}

// AD3's (AE3's) J^T J and J^T r terms of one point: A7's rows through D1's (FE2's) Jacobian
template <class Lens>
__device__ __forceinline__ void pnp_dist_add_normal(const Camera<double>& c, const PnpDistResidual& e, double* acc) {
  double J[4];
  Lens::jacobian(c.d, e.a, e.b, J);
  const double ua = c.fx * J[0] + c.s * J[2], ub = c.fx * J[1] + c.s * J[3], va = c.fy * J[2], vb = c.fy * J[3];
  const double gu[3] = {ua * e.iz, ub * e.iz, -((ua * e.a + ub * e.b) * e.iz)};
  const double gv[3] = {va * e.iz, vb * e.iz, -((va * e.a + vb * e.b) * e.iz)};
  pnp_add_rows(e.Xc, gu, gv, e.ru, e.rv, acc);
}

// The entry points' check of the coefficient count, at geo_check_config's distance() place
inline const char* dist_count_check(int nd) {
  return nd == 4 || nd == 5 || nd == 8 || nd == 12 ? nullptr : "num_dist must be 4, 5, 8 or 12";
}

// ---- the camera policies ----
//
// Everything that differs between the pinhole absolute pose (A1-A8, LA1-LA8) and the ones with lens distortion
// (AD1-AD4) or a fisheye lens (AE1-AE4) is one of these three policies, on which every kernel and entry point below is
// a template:
//   COEFFS, whether the entry point takes coefficients, and count_check(nd), its check of their number (host);
//   BEARING_FAILS, whether bearing can fail a match (AE1): then it runs before the compaction and returns false;
//   Consts and consts(a, b), pair b's constants of the LM and the scored model; Test and test(a, b), those of the fp32
//   test;
//   valid(K, dist, nd), whether K (and the coefficients) let the pair run;
//   bearing(K, dist, nd, p, x, y), the calibrated (x, y) of pixel p that P3P reads;
//   model(c, x, px), the 12-float model of x = (R, t) that is rounded to float and scored;
//   inlier(c, g, p, q, thr2) and err(c, g, p, q), the fp32 test and error of a point against the float model g;
//   residual(c, x, p, q) and add_normal(c, e, acc), a point's double residual and its J^T J and J^T r terms.

// The pinhole camera: K0^-1 (A2), K0 [R | t] (A5), the fp32 test in pixels (A5, LA3) and A7's residual
struct Pinhole {
  static constexpr bool COEFFS = false, BEARING_FAILS = false;
  static const char* count_check(int) { return nullptr; }
  using Consts = const double*;  // K0
  struct Test {};

  static __device__ __forceinline__ Consts consts(const PnpArgs& a, int b) { return a.K0 + (long)b * 9; }
  static __device__ __forceinline__ Test test(const PnpArgs&, int) { return {}; }
  static __device__ __forceinline__ bool valid(const double* K, const double*, int) { return k_valid(K); }
  static __device__ __forceinline__ void bearing(const double* K, const double*, int, float2 p, double* x, double* y) {
    const double yy = ((double)p.y - K[5]) / K[4], xx = (((double)p.x - K[2]) - K[1] * yy) / K[0];
    *x = xx;
    *y = yy;
  }
  static __device__ __forceinline__ void model(const double* K, const double* x, double* px) {
    projection(K, x, x + 9, px);
  }
  static __device__ __forceinline__ bool inlier(Test, const float* g, float4 p, float4 q, float thr2) {
    return reproj_inlier(g, p, q, thr2);
  }
  static __device__ __forceinline__ float err(Test, const float* g, float4 p, float4 q) { return reproj_err(g, p, q); }
  static __device__ __forceinline__ PnpResidual residual(const double* K, const double* x, float4 p, float4 q) {
    return pnp_residual(K, x, x + 9, p, q);
  }
  static __device__ __forceinline__ void add_normal(const double* K, const PnpResidual& e, double* acc) {
    pnp_add_normal(K, e, acc);
  }
};

// The camera with lens distortion: D2's undistortion (AD1), [R | t] and the fp32 test in distorted pixels (AD2) and
// AD3's residual; invalid coefficients fail the pair as an invalid K0
struct Distorted {
  static constexpr bool COEFFS = true, BEARING_FAILS = false;
  static const char* count_check(int nd) { return dist_count_check(nd); }
  using Consts = Camera<double>;
  using Test = Camera<float>;

  static __device__ __forceinline__ Consts consts(const PnpArgs& a, int b) { return pair_camera<double>(a, b); }
  static __device__ __forceinline__ Test test(const PnpArgs& a, int b) { return pair_camera<float>(a, b); }
  static __device__ __forceinline__ bool valid(const double* K, const double* dist, int nd) {
    return k_valid(K) && dist_valid(dist, nd);
  }
  static __device__ __forceinline__ void bearing(const double* K, const double* dist, int nd, float2 p, double* x,
                                                 double* y) {
    undistort(load_camera<double>(K, dist, nd), p.x, p.y, PNP_UNDISTORT_ITERS, 0.0, x, y);
  }
  static __device__ __forceinline__ void model(const Consts&, const double* x, double* px) { rt_matrix(x, px); }
  static __device__ __forceinline__ bool inlier(const Test& c, const float* g, float4 p, float4 q, float thr2) {
    return dist_reproj_err<BrownLens>(g, c, p, q) < thr2;
  }
  static __device__ __forceinline__ float err(const Test& c, const float* g, float4 p, float4 q) {
    return dist_reproj_err<BrownLens>(g, c, p, q);
  }
  static __device__ __forceinline__ PnpDistResidual residual(const Consts& c, const double* x, float4 p, float4 q) {
    return pnp_dist_residual<BrownLens>(c, x, x + 9, p, q);
  }
  static __device__ __forceinline__ void add_normal(const Consts& c, const PnpDistResidual& e, double* acc) {
    pnp_dist_add_normal<BrownLens>(c, e, acc);
  }
};

// The fisheye camera: FE3's bearing at cv2.fisheye's default criteria, which drops its match when it fails (AE1),
// [R | t] and the fp32 test in fisheye pixels (AE2) and AE3's residual; coefficients that fail FE4 fail the pair as an
// invalid K0
struct Fisheye {
  static constexpr bool COEFFS = true, BEARING_FAILS = true;
  static const char* count_check(int nd) { return nd == 4 ? nullptr : "num_dist must be 4"; }
  using Consts = Camera<double>;
  using Test = Camera<float>;

  static __device__ __forceinline__ Consts consts(const PnpArgs& a, int b) { return pair_camera<double>(a, b); }
  static __device__ __forceinline__ Test test(const PnpArgs& a, int b) { return pair_camera<float>(a, b); }
  static __device__ __forceinline__ bool valid(const double* K, const double* dist, int) {
    return k_valid(K) && fisheye_valid(dist);
  }
  static __device__ __forceinline__ bool bearing(const double* K, const double* dist, int nd, float2 p, double* x,
                                                 double* y) {
    return fisheye_undistort(load_camera<double>(K, dist, nd), p.x, p.y, GEO_FISHEYE_ITERS, GEO_FISHEYE_EPS, x, y);
  }
  static __device__ __forceinline__ void model(const Consts&, const double* x, double* px) { rt_matrix(x, px); }
  static __device__ __forceinline__ bool inlier(const Test& c, const float* g, float4 p, float4 q, float thr2) {
    return dist_reproj_err<FisheyeLens>(g, c, p, q) < thr2;
  }
  static __device__ __forceinline__ float err(const Test& c, const float* g, float4 p, float4 q) {
    return dist_reproj_err<FisheyeLens>(g, c, p, q);
  }
  static __device__ __forceinline__ PnpDistResidual residual(const Consts& c, const double* x, float4 p, float4 q) {
    return pnp_dist_residual<FisheyeLens>(c, x, x + 9, p, q);
  }
  static __device__ __forceinline__ void add_normal(const Consts& c, const PnpDistResidual& e, double* acc) {
    pnp_dist_add_normal<FisheyeLens>(c, e, acc);
  }
};

// geo_hyp_kernel's solver of the absolute pose: sample h's P3P solutions (R, t), scored as Cam's model
template <class Cam>
struct PnpSolver {
  static constexpr int SOLS = ::SOLS, NX = 12, NF = 12;
  static __device__ int s(const PnpArgs&) { return S; }
  static __device__ int solve(const PnpArgs& a, int b, unsigned h, double (*x)[NX]) {
    int id[S];
    if (geo_sample(a.seed, h, a.w.pair[b].n, S, id) < S) return 0;
    return p3p(a.w.pts + (long)b * a.M, a.w.wld + (long)b * a.M, id, x);
  }
  static __device__ void pixels(const PnpArgs& a, int b, const double* x, double* px) {
    Cam::model(Cam::consts(a, b), x, px);
  }
};

// A1 (and AD1, AE1): ordered compaction of the valid matches with Cam's calibrated coordinates, and the camera check
template <class Cam>
__global__ void __launch_bounds__(1024) pnp_prepare_kernel(PnpArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  const double* K = a.K0 + (long)b * 9;
  const double* dist = pair_dist(a, b);
  const int64_t* m0 = a.matches0 + (long)b * a.M;
  float4* pts = a.w.pts + (long)b * a.M;
  float4* wld = a.w.wld + (long)b * a.M;
  int* slot = a.w.slot + (long)b * a.M;
  for (int base = 0; base < a.M; base += 1024) {
    const int i = base + tid;
    const int64_t j = i < a.M ? m0[i] : -1;
    float X = 0.f, Y = 0.f, Z = 0.f;
    float2 p = make_float2(0.f, 0.f);
    if (j >= 0 && j < a.N) {
      const float* q = a.points3d1 + ((long)b * a.N + j) * 3;
      X = q[0];
      Y = q[1];
      Z = q[2];
      p = reinterpret_cast<const float2*>(a.kpts0)[(long)b * a.M + i];
    }
    bool valid = j >= 0 && j < a.N && isfinite(X) && isfinite(Y) && isfinite(Z) && finite2(p);
    double xx, yy;
    if constexpr (Cam::BEARING_FAILS) valid = valid && Cam::bearing(K, dist, a.nd, p, &xx, &yy);
    const int k = block_scan_step(valid, tid, warp_sums, &carry);
    if (i < a.M) slot[i] = valid ? k : -1;
    if (valid) {
      if constexpr (!Cam::BEARING_FAILS) Cam::bearing(K, dist, a.nd, p, &xx, &yy);
      pts[k] = make_float4(p.x, p.y, (float)xx, (float)yy);
      wld[k] = make_float4(X, Y, Z, 0.f);
    }
  }
  __syncthreads();
  if (tid == 0) {
    PnpPair& P = a.w.pair[b];
    P.thr2 = (float)(a.threshold * a.threshold);
    P.best = 0;
    P.n = carry;
    P.ok = carry >= S && Cam::valid(K, dist, a.nd);
    P.stop = !P.ok;
    P.drawn = 0;
    P.success = 0;
  }
}

}  // namespace
