// Batched undistortion and distortion of keypoints under OpenCV's lens model (include/geometry_b200.h, steps D1-D3)
// and its fisheye model (FE1-FE4): one thread per point, computed in double from float or double pixels.  One launch
// per call, fixed by (B, N), with no host synchronisation.  Compiled with -fmad=false: oracle/camera_oracle.py and
// oracle/fisheye_oracle.py take the same steps.
#include <stdint.h>

#include <type_traits>

#include "camera_common.cuh"
#include "geo_common.cuh"

namespace {

constexpr int CAM_THREADS = 256;

struct CamArgs {
  int B, N, nd, max_iters;
  double eps;
  const void* in;
  const double* K;     // [B, 9]
  const double* dist;  // [B, nd]
  void* out;
};

// D2 or FE3 (undistort) or D1 or FE2 through K (distort) of point i of pair b, as Lens is BrownLens or FisheyeLens;
// NaN for an invalid K or coefficients, a non-finite input pixel or a point FE3 fails on
template <class T, class Lens, bool UNDISTORT>
__global__ void __launch_bounds__(CAM_THREADS) camera_kernel(CamArgs a) {
  const int b = blockIdx.y, i = blockIdx.x * CAM_THREADS + threadIdx.x;
  if (i >= a.N) return;
  const double* K = a.K + (long)b * 9;
  const double* dist = a.dist + (long)b * a.nd;
  const long o = ((long)b * a.N + i) * 2;
  const double u = (double)((const T*)a.in)[o], v = (double)((const T*)a.in)[o + 1];
  double pu = NAN, pv = NAN;
  if (k_valid(K) && Lens::valid(dist, a.nd) && isfinite(u) && isfinite(v)) {
    const Camera<double> c = load_camera<double>(K, dist, a.nd);
    double x, y;
    bool ok = true;
    if (UNDISTORT) {
      ok = Lens::undistort(c, u, v, a.max_iters, a.eps, &x, &y);
    } else {
      const double y0 = (v - c.cy) / c.fy, x0 = ((u - c.cx) - c.s * y0) / c.fx;
      Lens::distort(c.d, x0, y0, &x, &y);
    }
    if (ok) {
      pu = c.fx * x + c.s * y + c.cx;
      pv = c.fy * y + c.cy;
    }
  }
  ((T*)a.out)[o] = (T)pu;
  ((T*)a.out)[o + 1] = (T)pv;
}

template <class Lens>
int camera_run(const char* entry, bool undist, const GeoCameraConfig* cfg, const GeoCameraInputs* in,
               GeoCameraOutputs* out, void* stream) {
  constexpr bool FISHEYE = std::is_same<Lens, FisheyeLens>::value;
  if (!cfg || !in || !out) return geo_error(entry, "null argument");
  if (cfg->abi_version != GEO_ABI_VERSION) return geo_error(entry, "ABI version mismatch");
  if (cfg->dtype != GEO_CAMERA_FLOAT32 && cfg->dtype != GEO_CAMERA_FLOAT64) return geo_error(entry, "unknown dtype");
  const int nd = cfg->num_dist;
  if (FISHEYE && nd != 4) return geo_error(entry, "num_dist must be 4");
  if (!FISHEYE && nd != 4 && nd != 5 && nd != 8 && nd != 12) return geo_error(entry, "num_dist must be 4, 5, 8 or 12");
  if (undist && (cfg->max_iters < 0 || cfg->max_iters > GEO_UNDISTORT_MAX_ITERS))
    return geo_error(entry, "max_iters outside [0, GEO_UNDISTORT_MAX_ITERS]");
  if (undist && !(cfg->eps >= 0.0 && isfinite(cfg->eps))) return geo_error(entry, "eps must be finite and >= 0");
  if (in->B < 0 || in->N < 0) return geo_error(entry, "negative size");
  if ((long)in->N * 2 > INT_MAX) return geo_error(entry, "N too large");
  if (in->B == 0 || in->N == 0) return 0;
  if (!in->pts || !in->K || !in->dist || !out->pts) return geo_error(entry, "null input or output");
  if (in->B > 65535) return geo_error(entry, "B above 65535");
  const CamArgs a{in->B, in->N, nd, cfg->max_iters, cfg->eps, in->pts, in->K, in->dist, out->pts};
  const dim3 grid((in->N + CAM_THREADS - 1) / CAM_THREADS, in->B);
  const cudaStream_t s = (cudaStream_t)stream;
  const bool f64 = cfg->dtype == GEO_CAMERA_FLOAT64;
  if (undist) {
    if (f64) camera_kernel<double, Lens, true><<<grid, CAM_THREADS, 0, s>>>(a);
    else camera_kernel<float, Lens, true><<<grid, CAM_THREADS, 0, s>>>(a);
  } else {
    if (f64) camera_kernel<double, Lens, false><<<grid, CAM_THREADS, 0, s>>>(a);
    else camera_kernel<float, Lens, false><<<grid, CAM_THREADS, 0, s>>>(a);
  }
  LG_CHECK_LAUNCH();
  return 0;
}

}  // namespace

extern "C" int geo_undistort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                    void* stream) {
  return camera_run<BrownLens>("geo_undistort_points", true, cfg, in, out, stream);
}

extern "C" int geo_distort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                  void* stream) {
  return camera_run<BrownLens>("geo_distort_points", false, cfg, in, out, stream);
}

extern "C" int geo_fisheye_undistort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in,
                                            GeoCameraOutputs* out, void* stream) {
  return camera_run<FisheyeLens>("geo_fisheye_undistort_points", true, cfg, in, out, stream);
}

extern "C" int geo_fisheye_distort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                          void* stream) {
  return camera_run<FisheyeLens>("geo_fisheye_distort_points", false, cfg, in, out, stream);
}
