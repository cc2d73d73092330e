// OpenCV's lens distortion model (include/geometry_b200.h, steps D1-D3) and its fisheye model (FE1-FE4), shared by
// the batched undistortion (camera_api.cu) and the distortion-aware absolute pose (pnp_api.cu, lo_pnp_api.cu), all
// compiled with -fmad=false: oracle/camera_oracle.py and oracle/fisheye_oracle.py restate every step in numpy.
#pragma once
#include <float.h>
#include <math.h>

#include "fisheye_poly.h"

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

// ---- the fisheye model (header steps FE1-FE4) ----

// FE1: t + t*(z*Q(z)), z = t*t, Q by Horner from its last coefficient
template <class T, int N>
__device__ __forceinline__ T fe_poly(T t, const T (&q)[N]) {
  const T z = t * t;
  T acc = q[N - 1];
#pragma unroll
  for (int i = N - 2; i >= 0; --i) acc = acc * z + q[i];
  return t + t * (z * acc);
}

// FE1's atan in double: |r| to |t| <= tan(pi/8) in three intervals, the odd polynomial, r's sign
__device__ __forceinline__ double fe_atan(double r) {
  const double a = fabs(r);
  double res;
  if (a > FE_TAN_3PI_8) res = FE_PI_2_HI + (FE_PI_2_LO + fe_poly(-1.0 / a, FE_ATAN_D));
  else if (a > FE_TAN_PI_8) res = FE_PI_4_HI + (FE_PI_4_LO + fe_poly((a - 1.0) / (a + 1.0), FE_ATAN_D));
  else res = fe_poly(a, FE_ATAN_D);
  return r < 0.0 ? -res : res;
}

// FE1's atan in float (AE2's test): |r| to |t| <= 1 in two intervals
__device__ __forceinline__ float fe_atan(float r) {
  const float a = fabsf(r);
  const float res = a > 1.f ? FE_PI_2_HI_F + (FE_PI_2_LO_F + fe_poly(-1.f / a, FE_ATAN_F)) : fe_poly(a, FE_ATAN_F);
  return r < 0.f ? -res : res;
}

// FE1's tan in double: x less n*pi/2 in three parts, n = rint(x * 2/pi), the odd polynomial p, -1/p for odd n
__device__ __forceinline__ double fe_tan(double x) {
  const double n = rint(x * FE_2_PI);
  const double y = ((x - n * FE_PIO2_1) - n * FE_PIO2_2) - n * FE_PIO2_3;
  const double p = fe_poly(y, FE_TAN_D);
  return floor(n * 0.5) != n * 0.5 ? -1.0 / p : p;
}

// FE2's theta_d of theta and its powers t2, t4, t6, t8 = t4*t4
template <class T>
__device__ __forceinline__ T fe_theta_d(const T* d, T th, T* t2, T* t4, T* t6, T* t8) {
  *t2 = th * th;
  *t4 = *t2 * *t2;
  *t6 = *t4 * *t2;
  *t8 = *t4 * *t4;
  return th * ((T)1 + d[0] * *t2 + d[1] * *t4 + d[2] * *t6 + d[3] * *t8);
}

// FE2: the distorted normalised point of (x, y), cv2.fisheye.distortPoints' model in T
template <class T>
__device__ __forceinline__ void fisheye_distort(const T* d, T x, T y, T* xd, T* yd) {
  const T r = sqrt(x * x + y * y);
  T t2, t4, t6, t8;
  const T thd = fe_theta_d(d, fe_atan(r), &t2, &t4, &t6, &t8);
  const T cdist = r > (T)1e-8 ? thd / r : (T)1;
  *xd = cdist * x;
  *yd = cdist * y;
}

// FE2's Jacobian d(xd, yd) / d(x, y), row-major (header step AE3): c*I + (dc/dr)/r [x y]^T [x y]
__device__ __forceinline__ void fisheye_jacobian(const double* d, double x, double y, double* J) {
  const double r2 = x * x + y * y, r = sqrt(r2);
  double t2, t4, t6, t8;
  const double thd = fe_theta_d(d, fe_atan(r), &t2, &t4, &t6, &t8);
  double c = 1.0, g = 0.0;
  if (r > 1e-8) {
    c = thd / r;
    const double dd = 1.0 + 3.0 * d[0] * t2 + 5.0 * d[1] * t4 + 7.0 * d[2] * t6 + 9.0 * d[3] * t8;
    g = ((dd / (1.0 + r2) - c) / r) / r;
  }
  const double gx = g * x, gy = g * y;
  J[0] = c + gx * x;
  J[1] = gx * y;
  J[2] = gy * x;
  J[3] = c + gy * y;
}

// FE3: cv2.fisheye.undistortPoints' Newton on theta for pixel (u, v), at most iters steps; with eps > 0 a step below
// eps converges the point and |theta_d| <= eps skips the steps.  Returns false where FE3 fails (theta flipped sign, or
// eps > 0 and no convergence).
__device__ __forceinline__ bool fisheye_undistort(const Camera<double>& c, double u, double v, int iters, double eps,
                                                  double* xo, double* yo) {
  const double* d = c.d;
  const double y0 = (v - c.cy) / c.fy, x0 = ((u - c.cx) - c.s * y0) / c.fx;
  double thd = sqrt(x0 * x0 + y0 * y0);
  if (thd < -FE_PI_2_HI) thd = -FE_PI_2_HI;
  if (thd > FE_PI_2_HI) thd = FE_PI_2_HI;
  double th = thd, scale = 0.0;
  bool converged = false;
  if (eps > 0.0 && fabs(thd) <= eps) {
    converged = true;
  } else {
    for (int j = 0; j < iters; ++j) {
      const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t6 * t2;
      const double a2 = d[0] * t2, a4 = d[1] * t4, a6 = d[2] * t6, a8 = d[3] * t8;
      const double fix = (th * (1.0 + a2 + a4 + a6 + a8) - thd) / (1.0 + 3.0 * a2 + 5.0 * a4 + 7.0 * a6 + 9.0 * a8);
      th = th - fix;
      if (eps > 0.0 && fabs(fix) < eps) {
        converged = true;
        break;
      }
    }
    scale = fe_tan(th) / thd;
  }
  const bool flipped = (thd < 0.0 && th > 0.0) || (thd > 0.0 && th < 0.0);
  *xo = scale * x0;
  *yo = scale * y0;
  return (converged || eps == 0.0) && !flipped;
}

// FE4: exactly 4 finite coefficients (the count is checked on the host)
__device__ __forceinline__ bool fisheye_valid(const double* dist) {
  return isfinite(dist[0]) && isfinite(dist[1]) && isfinite(dist[2]) && isfinite(dist[3]);
}

// The two lens models as camera_kernel and the absolute pose read them: validity of the coefficients, the pixel
// undistortion (false: the point fails), the distortion of a normalised point in T and its double Jacobian
struct BrownLens {
  static __device__ __forceinline__ bool valid(const double* dist, int nd) { return dist_valid(dist, nd); }
  static __device__ __forceinline__ bool undistort(const Camera<double>& c, double u, double v, int iters, double eps,
                                                   double* x, double* y) {
    ::undistort(c, u, v, iters, eps, x, y);
    return true;
  }
  template <class T>
  static __device__ __forceinline__ void distort(const T* d, T x, T y, T* xd, T* yd) { ::distort(d, x, y, xd, yd); }
  static __device__ __forceinline__ void jacobian(const double* d, double x, double y, double* J) {
    distort_jacobian(d, x, y, J);
  }
};

struct FisheyeLens {
  static __device__ __forceinline__ bool valid(const double* dist, int) { return fisheye_valid(dist); }
  static __device__ __forceinline__ bool undistort(const Camera<double>& c, double u, double v, int iters, double eps,
                                                   double* x, double* y) {
    return fisheye_undistort(c, u, v, iters, eps, x, y);
  }
  template <class T>
  static __device__ __forceinline__ void distort(const T* d, T x, T y, T* xd, T* yd) {
    fisheye_distort(d, x, y, xd, yd);
  }
  static __device__ __forceinline__ void jacobian(const double* d, double x, double y, double* J) {
    fisheye_jacobian(d, x, y, J);
  }
};

}  // namespace
