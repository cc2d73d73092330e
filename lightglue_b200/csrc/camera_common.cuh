// OpenCV's lens distortion model (include/geometry_b200.h, steps D1-D3), shared by the batched undistortion
// (camera_api.cu) and the distortion-aware absolute pose (pnp_api.cu, lo_pnp_api.cu), all compiled with -fmad=false:
// oracle/camera_oracle.py restates every step in numpy.
#pragma once
#include <float.h>
#include <math.h>

namespace {

// OpenCV's coefficient order: k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 (missing trailing ones are zero)
constexpr int CAM_COEFFS = 12;

// A K is valid as header step P1 states it: finite, fx > 0, fy > 0, bottom row (0, 0, 1)
__device__ bool k_valid(const double* K) {
  bool finite = true;
  for (int i = 0; i < 9; ++i) finite = finite && isfinite(K[i]);
  return finite && K[0] > 0.0 && K[4] > 0.0 && K[6] == 0.0 && K[7] == 0.0 && K[8] == 1.0;
}

// A pair's K and its coefficients padded to 12, in T (double, or float for the fp32 inlier test of step AD2)
template <class T>
struct Camera {
  T fx, s, cx, fy, cy;
  T d[CAM_COEFFS];
};

template <class T>
__device__ __forceinline__ Camera<T> load_camera(const double* K, const double* dist, int nd) {
  Camera<T> c;
  c.fx = (T)K[0]; c.s = (T)K[1]; c.cx = (T)K[2]; c.fy = (T)K[4]; c.cy = (T)K[5];
#pragma unroll
  for (int i = 0; i < CAM_COEFFS; ++i) c.d[i] = i < nd ? (T)dist[i] : (T)0;
  return c;
}

// D3: the coefficients are valid when all are finite
__device__ __forceinline__ bool dist_valid(const double* dist, int nd) {
  bool finite = true;
  for (int i = 0; i < nd; ++i) finite = finite && isfinite(dist[i]);
  return finite;
}

// D1: the distorted normalised point of (x, y), cv2.projectPoints' formula in T
template <class T>
__device__ __forceinline__ void distort(const T* d, T x, T y, T* xd, T* yd) {
  const T r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
  const T a1 = (T)2 * x * y, a2 = r2 + (T)2 * x * x, a3 = r2 + (T)2 * y * y;
  const T cdist = (T)1 + d[0] * r2 + d[1] * r4 + d[4] * r6;
  const T icdist2 = (T)1 / ((T)1 + d[5] * r2 + d[6] * r4 + d[7] * r6);
  *xd = x * cdist * icdist2 + d[2] * a1 + d[3] * a2 + d[8] * r2 + d[9] * r4;
  *yd = y * cdist * icdist2 + d[2] * a3 + d[3] * a1 + d[10] * r2 + d[11] * r4;
}

// D1's Jacobian d(xd, yd) / d(x, y), row-major (header step AD3)
__device__ __forceinline__ void distort_jacobian(const double* d, double x, double y, double* J) {
  const double r2 = x * x + y * y, r4 = r2 * r2;
  const double id = 1.0 / (1.0 + d[5] * r2 + d[6] * r4 + d[7] * r2 * r4);
  const double c = (1.0 + d[0] * r2 + d[1] * r4 + d[4] * r2 * r4) * id;
  const double dc = (d[0] + 2.0 * d[1] * r2 + 3.0 * d[4] * r4 - c * (d[5] + 2.0 * d[6] * r2 + 3.0 * d[7] * r4)) * id;
  const double gx = d[8] + 2.0 * d[9] * r2, gy = d[10] + 2.0 * d[11] * r2;
  J[0] = c + 2.0 * x * (x * dc + gx) + 2.0 * d[2] * y + 6.0 * d[3] * x;
  J[1] = 2.0 * y * (x * dc + d[3] + gx) + 2.0 * d[2] * x;
  J[2] = 2.0 * x * (y * dc + d[2] + gy) + 2.0 * d[3] * y;
  J[3] = c + 2.0 * y * (y * dc + gy) + 6.0 * d[2] * y + 2.0 * d[3] * x;
}

// D2: OpenCV's fixed-point undistortion of pixel (u, v) into the normalised (x, y), at most iters iterations; with
// eps > 0 it stops before an iteration once the previous iterate reprojects within eps pixels
__device__ __forceinline__ void undistort(const Camera<double>& c, double u, double v, int iters, double eps,
                                          double* xo, double* yo) {
  const double* d = c.d;
  const double y0 = (v - c.cy) / c.fy, x0 = ((u - c.cx) - c.s * y0) / c.fx;
  double x = x0, y = y0, err = DBL_MAX;
  for (int j = 0; j < iters; ++j) {
    if (err < eps) break;
    const double r2 = x * x + y * y;
    const double icdist = (1.0 + ((d[7] * r2 + d[6]) * r2 + d[5]) * r2) / (1.0 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2);
    if (icdist < 0.0) {
      x = x0;
      y = y0;
      break;
    }
    const double dx = 2.0 * d[2] * x * y + d[3] * (r2 + 2.0 * x * x) + d[8] * r2 + d[9] * r2 * r2;
    const double dy = d[2] * (r2 + 2.0 * y * y) + 2.0 * d[3] * x * y + d[10] * r2 + d[11] * r2 * r2;
    x = (x0 - dx) * icdist;
    y = (y0 - dy) * icdist;
    if (eps > 0.0) {
      double xd, yd;
      distort(d, x, y, &xd, &yd);
      const double du = c.fx * xd + c.s * yd + c.cx - u, dv = c.fy * yd + c.cy - v;
      err = sqrt(du * du + dv * dv);
    }
  }
  *xo = x;
  *yo = y;
}

}  // namespace
