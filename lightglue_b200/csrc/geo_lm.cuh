// Levenberg-Marquardt pieces shared by the absolute pose (pnp_api.cu, header step A7) and the LO-RANSAC relative pose,
// homography and fundamental matrix (lo_pose_api.cu and lo_hf_api.cu through lo_common.cuh, header steps L7,
// LH7 and LF7), all compiled with -fmad=false.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace {

// delta of (J^T J, its diagonal times (1 + lam)) delta = -J^T r by Cholesky; false on a pivot <= 0 or a non-finite
// delta.  Hu is the row-major upper triangle of J^T J, g = J^T r.
template <int N>
__device__ bool lm_solve(const double* Hu, const double* g, double lam, double* x) {
  double A[N][N], L[N][N], yv[N];
  for (int i = 0, e = 0; i < N; ++i)
    for (int j = i; j < N; ++j, ++e) A[i][j] = A[j][i] = Hu[e];
  for (int i = 0; i < N; ++i) A[i][i] = A[i][i] * (1.0 + lam);
  for (int j = 0; j < N; ++j) {
    double d = A[j][j];
    for (int k = 0; k < j; ++k) d = d - L[j][k] * L[j][k];
    if (!(d > 0.0)) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < N; ++i) {
      double e = A[i][j];
      for (int k = 0; k < j; ++k) e = e - L[i][k] * L[j][k];
      L[i][j] = e / L[j][j];
    }
  }
  for (int i = 0; i < N; ++i) {
    double e = -g[i];
    for (int k = 0; k < i; ++k) e = e - L[i][k] * yv[k];
    yv[i] = e / L[i][i];
  }
  bool fin = true;
  for (int i = N - 1; i >= 0; --i) {
    double e = yv[i];
    for (int k = i + 1; k < N; ++k) e = e - L[k][i] * x[k];
    x[i] = e / L[i][i];
    fin = fin && isfinite(x[i]);
  }
  return fin;
}

// Row-major rotation Q of the unit quaternion (1, d[0..2] / 2) / norm
__device__ __forceinline__ void quat_rotation(const double* d, double* Q) {
  double qw = 1.0, qx = d[0] * 0.5, qy = d[1] * 0.5, qz = d[2] * 0.5;
  const double n = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
  qw = qw / n;
  qx = qx / n;
  qy = qy / n;
  qz = qz / n;
  Q[0] = 1.0 - 2.0 * (qy * qy + qz * qz);
  Q[1] = 2.0 * (qx * qy - qw * qz);
  Q[2] = 2.0 * (qx * qz + qw * qy);
  Q[3] = 2.0 * (qx * qy + qw * qz);
  Q[4] = 1.0 - 2.0 * (qx * qx + qz * qz);
  Q[5] = 2.0 * (qy * qz - qw * qx);
  Q[6] = 2.0 * (qx * qz - qw * qy);
  Q[7] = 2.0 * (qy * qz + qw * qx);
  Q[8] = 1.0 - 2.0 * (qx * qx + qy * qy);
}

}  // namespace
