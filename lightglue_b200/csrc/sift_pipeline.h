// SIFT extractor forward (include/sift_b200.h; reference lightglue/sift.py, backend "opencv"): OpenCV's SIFT
// (detectAndCompute with the first octave upsampled) followed by the reference's post-processing.
//
// As in sp_pipeline.h, every stage is a functor whose `operator()(i, scratch)` is the work of ONE logical thread, and
// the whole per-image forward is one template `sift_run(Exec&, ...)`.  The CUDA build (sift_api.cu) runs each functor
// with one thread per index (scratch = a per-thread slice of shared memory); the test-only host build
// (oracle/sift_emul.cpp, g++ -ffp-contract=off) runs THE SAME functors and orchestration in host loops.  Functors that
// append to a list use an atomic counter, so list order is not deterministic; every later stage orders its inputs by a
// total key before it depends on order.
//
// Arithmetic is written out the way OpenCV's float SIFT does it (operation order, float vs double, cvRound as
// round-half-even).  Both builds must round the same: sift_api.cu is compiled with -fmad=false and the host build with
// -ffp-contract=off; where OpenCV's SIMD code fuses a multiply-add, fmaf() says so explicitly.
//
// Per image: the crop (h, w) is turned into the 8-bit gray image the reference hands to OpenCV, upsampled 2x, blurred
// to sigma 1.6, and nOct octaves of L+3 Gaussians and L+2 DoG layers are built (L = nOctaveLayers).  Extrema of the
// DoG layers 1..L are refined and tested (candidates), each candidate gets an orientation histogram and one keypoint
// per peak (raw keypoints), the raw list is sorted and filtered (OpenCV's dedupe and retainBest, the reference's
// filter_dog_point and top-k), and the survivors get descriptors.
#pragma once
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "ws_bump.h"

#if defined(__CUDACC__)
#define SIFT_HD __host__ __device__ __forceinline__
#else
#define SIFT_HD inline
#endif

#define SIFT_IMG_BORDER 5
#define SIFT_MAX_INTERP_STEPS 5
#define SIFT_ORI_HIST_BINS 36
#define SIFT_ORI_SIG_FCTR 1.5f
#define SIFT_ORI_RADIUS 4.5f
#define SIFT_ORI_PEAK_RATIO 0.8f
#define SIFT_DESCR_WIDTH 4
#define SIFT_DESCR_HIST_BINS 8
#define SIFT_DESCR_SCL_FCTR 3.f
#define SIFT_DESCR_MAG_THR 0.2f
#define SIFT_INT_DESCR_FCTR 512.f
#define SIFT_DESC 128
#define SIFT_MAX_KSIZE 127     // Gaussian taps (ksize = round(8 sigma + 1) | 1); 89 for nOctaveLayers = 1
#define SIFT_MAX_LAYERS 8      // nOctaveLayers
#define SIFT_MAX_OCTAVES 16    // 2^17 pixels on the shorter side
#define SIFT_DESC_HIST ((SIFT_DESCR_WIDTH + 2) * (SIFT_DESCR_WIDTH + 2) * (SIFT_DESCR_HIST_BINS + 2))  // 360

SIFT_HD int sift_round(float v) { return (int)rintf(v); }  // cvRound: half to even
SIFT_HD int sift_floor(float v) { return (int)floorf(v); }

SIFT_HD int sift_atomic_add(int* p, int v) {
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  return __atomic_fetch_add(p, v, __ATOMIC_RELAXED);
#endif
}

// cv::borderInterpolate(p, len, BORDER_REFLECT_101), including repeated reflection for kernels wider than the image.
SIFT_HD int sift_reflect101(int p, int len) {
  if ((unsigned)p < (unsigned)len) return p;
  if (len == 1) return 0;
  do {
    if (p < 0) p = -p;
    else p = len - 1 - (p - len) - 1;
  } while ((unsigned)p >= (unsigned)len);
  return p;
}

// cv::fastAtan2 in degrees, [0, 360).  The polynomial of OpenCV's vectorised version (v_atan_f32), which fuses the
// Horner steps, is what its orientation and descriptor loops run.
SIFT_HD float sift_fast_atan2(float y, float x) {
  const float p1 = 0.9997878412794807f * (float)(180 / M_PI), p3 = -0.3258083974640975f * (float)(180 / M_PI);
  const float p5 = 0.1555786518463281f * (float)(180 / M_PI), p7 = -0.04432655554792128f * (float)(180 / M_PI);
  const float ax = fabsf(x), ay = fabsf(y);
  const float c = fminf(ax, ay) / (fmaxf(ax, ay) + (float)DBL_EPSILON);
  const float cc = c * c;
  float a = fmaf(fmaf(fmaf(cc, p7, p5), cc, p3), cc, p1) * c;
  if (!(ax >= ay)) a = 90.f - a;
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

SIFT_HD float sift_magnitude(float x, float y) { return sqrtf(fmaf(x, x, y * y)); }

// ---------------------------------------------------------------------------------------------------------------------
// pyramid
// ---------------------------------------------------------------------------------------------------------------------
struct SiftGray {  // crop -> kornia rgb_to_grayscale -> (uint8)(v * 255) as float
  const float* image; float* out;
  int C, H, W, h, w;  // image [C, H, W], crop [:h, :w]
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return (long)h * w; }
  SIFT_HD void operator()(long i, float*) const {
    const int y = (int)(i / w), x = (int)(i % w);
    const long p = (long)y * W + x, plane = (long)H * W;
    float g = image[p];
    if (C == 3) g = 0.299f * image[p] + 0.587f * image[p + plane] + 0.114f * image[p + 2 * plane];
    out[i] = (float)(uint8_t)(int)(g * 255.0f);
  }
};

struct SiftUpsample {  // cv::resize(2x, INTER_LINEAR); exact in float for 8-bit inputs
  const float* in; float* out;
  int h, w;  // input size; output 2h x 2w
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return 4L * h * w; }
  SIFT_HD static void tap(int d, int n, int& s0, int& s1, float& a0, float& a1) {
    // src = (d + 0.5) / 2 - 0.5: even d -> (k - 1, k) with 1/4, 3/4; odd d -> (k, k + 1) with 3/4, 1/4; clamped ends
    const int k = d >> 1;
    if (d & 1) { s0 = k; s1 = k + 1; a0 = 0.75f; a1 = 0.25f; }
    else { s0 = k - 1; s1 = k; a0 = 0.25f; a1 = 0.75f; }
    if (s0 < 0) { s0 = 0; s1 = 0; a0 = 1.f; a1 = 0.f; }
    if (s1 > n - 1) { s0 = n - 1; s1 = n - 1; a0 = 1.f; a1 = 0.f; }
  }
  SIFT_HD void operator()(long i, float*) const {
    const int W2 = 2 * w, Y = (int)(i / W2), X = (int)(i % W2);
    int x0, x1, y0, y1; float ax0, ax1, ay0, ay1;
    tap(X, w, x0, x1, ax0, ax1);
    tap(Y, h, y0, y1, ay0, ay1);
    const float r0 = in[(long)y0 * w + x0] * ax0 + in[(long)y0 * w + x1] * ax1;
    const float r1 = in[(long)y1 * w + x0] * ax0 + in[(long)y1 * w + x1] * ax1;
    out[i] = r0 * ay0 + r1 * ay1;
  }
};

struct SiftKernel {  // one Gaussian: ksize taps, k[0..ksize) in OpenCV's order
  int ksize;
  float k[SIFT_MAX_KSIZE];
};

struct SiftRowBlur {  // row pass of cv::GaussianBlur (RowFilter, taps in order, fused multiply-add)
  const float* in; float* out;
  int h, w;
  SiftKernel kr;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return (long)h * w; }
  SIFT_HD void operator()(long i, float*) const {
    const int y = (int)(i / w), x = (int)(i % w), r = kr.ksize / 2;
    const float* row = in + (long)y * w;
    float s = 0.f;
    if (x >= r && x + r < w) {
      for (int t = 0; t < kr.ksize; ++t) s = fmaf(row[x - r + t], kr.k[t], s);
    } else {
      for (int t = 0; t < kr.ksize; ++t) s = fmaf(row[sift_reflect101(x - r + t, w)], kr.k[t], s);
    }
    out[i] = s;
  }
};

struct SiftColBlur {  // column pass (SymmColumnFilter: centre tap, then pairs k, -k), plus DoG = out - prev
  const float* in; float* out; const float* prev; float* dog;  // prev/dog null: no DoG
  int h, w;
  SiftKernel kr;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return (long)h * w; }
  SIFT_HD void operator()(long i, float*) const {
    const int y = (int)(i / w), x = (int)(i % w), r = kr.ksize / 2;
    float s = kr.k[r] * in[i];
    for (int t = 1; t <= r; ++t) {
      const int ya = sift_reflect101(y + t, h), yb = sift_reflect101(y - t, h);
      s = fmaf(in[(long)ya * w + x] + in[(long)yb * w + x], kr.k[r + t], s);
    }
    out[i] = s;
    if (dog) dog[i] = s - prev[i];
  }
};

struct SiftDecimate {  // next octave's base: cv::resize(INTER_NEAREST) to half size = every other pixel
  const float* in; float* out;
  int w_in, h, w;  // output size
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return (long)h * w; }
  SIFT_HD void operator()(long i, float*) const {
    const int y = (int)(i / w), x = (int)(i % w);
    out[i] = in[(long)(2 * y) * w_in + 2 * x];
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// detection
// ---------------------------------------------------------------------------------------------------------------------
struct SiftOctave {  // one octave of the pyramid
  const float* gauss[SIFT_MAX_LAYERS + 3];
  const float* dog[SIFT_MAX_LAYERS + 2];
  int h, w;
};

struct SiftTables {  // every octave's Gaussian layers and sizes, passed by value
  const float* gauss[SIFT_MAX_OCTAVES * (SIFT_MAX_LAYERS + 3)];  // [o * (L + 3) + i]
  int dims[SIFT_MAX_OCTAVES * 2];                                // (h, w) of octave o
};

struct SiftCand {  // a refined extremum (adjustLocalExtrema's output), octave coordinates of the upsampled image
  float x, y, size, response;  // as cv::KeyPoint before the first-octave halving
  int r, c, layer, octave_packed;
};

struct SiftKpt {  // a raw keypoint in final (halved) coordinates
  float x, y, size, angle, response;
  int octave_packed;  // after the first-octave adjustment
  int o, layer;       // pyramid octave (0 = upsampled) and layer of the descriptor
};

struct SiftParams {
  int L;                    // nOctaveLayers (the reference's num_octaves)
  float contrast, edge;     // contrastThreshold, edgeThreshold (as float in adjustLocalExtrema)
  float sigma;              // 1.6
  int threshold;            // cvFloor(0.5 * contrast / L * 255)
  int nfeatures;            // retainBest (max_num_keypoints)
  int nms_radius;           // < 0: filter_dog_point off
  int max_kpts;             // top-k after filter_dog_point (max_num_keypoints)
  int rootsift;
};

// The parameters of a conf (include/sift_b200.h SiftConfig): L = num_octaves, contrast = detection_threshold,
// edge = edge_threshold, max_kpts = max_num_keypoints (> 0), nms_radius (-1 = None), rootsift.
inline SiftParams sift_params(int L, double contrast, double edge, int nms_radius, int max_kpts, int rootsift) {
  SiftParams p{};
  p.L = L;
  p.contrast = (float)contrast;
  p.edge = (float)edge;
  p.sigma = 1.6f;
  p.threshold = (int)floor(0.5 * contrast / L * 255);
  p.nfeatures = max_kpts;
  p.nms_radius = nms_radius;
  p.max_kpts = max_kpts;
  p.rootsift = rootsift;
  return p;
}

// adjustLocalExtrema: up to five Newton steps on the DoG cube, then the contrast and edge tests.
SIFT_HD bool sift_adjust(const SiftOctave& oc, int o, const SiftParams& p, int& layer, int& r, int& c, SiftCand& out) {
  const float img_scale = 1.f / 255.f, deriv_scale = img_scale * 0.5f, second_deriv_scale = img_scale,
              cross_deriv_scale = img_scale * 0.25f;
  float xi = 0, xr = 0, xc = 0, contr = 0;
  const int w = oc.w;
  int i = 0;
  for (; i < SIFT_MAX_INTERP_STEPS; i++) {
    const float* img = oc.dog[layer];
    const float* prv = oc.dog[layer - 1];
    const float* nxt = oc.dog[layer + 1];
#define AT(m, yy, xx) (m)[(long)(yy) * w + (xx)]
    const float dD[3] = {(AT(img, r, c + 1) - AT(img, r, c - 1)) * deriv_scale, (AT(img, r + 1, c) - AT(img, r - 1, c)) * deriv_scale,
                   (AT(nxt, r, c) - AT(prv, r, c)) * deriv_scale};
    const float v2 = AT(img, r, c) * 2;
    const float dxx = (AT(img, r, c + 1) + AT(img, r, c - 1) - v2) * second_deriv_scale;
    const float dyy = (AT(img, r + 1, c) + AT(img, r - 1, c) - v2) * second_deriv_scale;
    const float dss = (AT(nxt, r, c) + AT(prv, r, c) - v2) * second_deriv_scale;
    const float dxy = (AT(img, r + 1, c + 1) - AT(img, r + 1, c - 1) - AT(img, r - 1, c + 1) + AT(img, r - 1, c - 1)) * cross_deriv_scale;
    const float dxs = (AT(nxt, r, c + 1) - AT(nxt, r, c - 1) - AT(prv, r, c + 1) + AT(prv, r, c - 1)) * cross_deriv_scale;
    const float dys = (AT(nxt, r + 1, c) - AT(nxt, r - 1, c) - AT(prv, r + 1, c) + AT(prv, r - 1, c)) * cross_deriv_scale;
    // cv::Matx33f::solve: Cramer's rule (Matx_FastSolveOp<float, 3, 3, 1>), all in float; singular -> X = 0
    const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
    const float b0 = dD[0], b1 = dD[1], b2 = dD[2];
    float X[3] = {0.f, 0.f, 0.f};
    float det = a00 * (a11 * a22 - a21 * a12) - a01 * (a10 * a22 - a20 * a12) + a02 * (a10 * a21 - a20 * a11);
    if (det != 0) {
      det = 1 / det;
      X[0] = det * (b0 * (a11 * a22 - a12 * a21) - a01 * (b1 * a22 - a12 * b2) + a02 * (b1 * a21 - a11 * b2));
      X[1] = det * (a00 * (b1 * a22 - a12 * b2) - b0 * (a10 * a22 - a12 * a20) + a02 * (a10 * b2 - b1 * a20));
      X[2] = det * (a00 * (a11 * b2 - b1 * a21) - a01 * (a10 * b2 - b1 * a20) + b0 * (a10 * a21 - a11 * a20));
    }
    xi = -X[2]; xr = -X[1]; xc = -X[0];
    if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
    if (fabsf(xi) > (float)(INT32_MAX / 3) || fabsf(xr) > (float)(INT32_MAX / 3) || fabsf(xc) > (float)(INT32_MAX / 3)) return false;
    c += sift_round(xc);
    r += sift_round(xr);
    layer += sift_round(xi);
    if (layer < 1 || layer > p.L || c < SIFT_IMG_BORDER || c >= oc.w - SIFT_IMG_BORDER || r < SIFT_IMG_BORDER ||
        r >= oc.h - SIFT_IMG_BORDER)
      return false;
  }
  if (i >= SIFT_MAX_INTERP_STEPS) return false;
  {
    const float* img = oc.dog[layer];
    const float* prv = oc.dog[layer - 1];
    const float* nxt = oc.dog[layer + 1];
    const float dD0 = (AT(img, r, c + 1) - AT(img, r, c - 1)) * deriv_scale;
    const float dD1 = (AT(img, r + 1, c) - AT(img, r - 1, c)) * deriv_scale;
    const float dD2 = (AT(nxt, r, c) - AT(prv, r, c)) * deriv_scale;
    const float t = dD0 * xc + dD1 * xr + dD2 * xi;
    contr = AT(img, r, c) * img_scale + t * 0.5f;
    if (fabsf(contr) * p.L < p.contrast) return false;
    const float v2 = AT(img, r, c) * 2.f;
    const float dxx = (AT(img, r, c + 1) + AT(img, r, c - 1) - v2) * second_deriv_scale;
    const float dyy = (AT(img, r + 1, c) + AT(img, r - 1, c) - v2) * second_deriv_scale;
    const float dxy = (AT(img, r + 1, c + 1) - AT(img, r + 1, c - 1) - AT(img, r - 1, c + 1) + AT(img, r - 1, c - 1)) * cross_deriv_scale;
    const float tr = dxx + dyy, det = dxx * dyy - dxy * dxy;
    if (det <= 0 || tr * tr * p.edge >= (p.edge + 1) * (p.edge + 1) * det) return false;
#undef AT
  }
  out.x = (c + xc) * (float)(1 << o);
  out.y = (r + xr) * (float)(1 << o);
  out.octave_packed = o + (layer << 8) + ((int)rint((xi + 0.5) * 255) << 16);
  out.size = p.sigma * powf(2.f, (layer + xi) / p.L) * (float)(1 << o) * 2;
  out.response = fabsf(contr);
  out.r = r; out.c = c; out.layer = layer;
  return true;
}

struct SiftDetect {  // 3x3x3 extremum test of DoG layer `layer` (1..L) + refinement; appends to cand
  SiftOctave oc; SiftParams p;
  int o, layer;
  SiftCand* cand; int* n_cand; int cand_cap;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const {
    const int hh = oc.h - 2 * SIFT_IMG_BORDER, ww = oc.w - 2 * SIFT_IMG_BORDER;
    return (hh > 0 && ww > 0) ? (long)hh * ww : 0;
  }
  SIFT_HD void operator()(long i, float*) const {
    const int ww = oc.w - 2 * SIFT_IMG_BORDER, w = oc.w;
    const int r = (int)(i / ww) + SIFT_IMG_BORDER, c = (int)(i % ww) + SIFT_IMG_BORDER;
    const float* cur = oc.dog[layer] + (long)r * w + c;
    const float val = *cur;
    if (!(fabsf(val) > (float)p.threshold)) return;
    const float* prv = oc.dog[layer - 1] + (long)r * w + c;
    const float* nxt = oc.dog[layer + 1] + (long)r * w + c;
    bool ext = true;
    if (val > 0) {
      for (int dy = -1; dy <= 1 && ext; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const long q = (long)dy * w + dx;
          if (!(val >= cur[q] && val >= prv[q] && val >= nxt[q])) { ext = false; break; }
        }
    } else {
      for (int dy = -1; dy <= 1 && ext; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const long q = (long)dy * w + dx;
          if (!(val <= cur[q] && val <= prv[q] && val <= nxt[q])) { ext = false; break; }
        }
    }
    if (!ext) return;
    int r1 = r, c1 = c, l1 = layer;
    SiftCand k;
    if (!sift_adjust(oc, o, p, l1, r1, c1, k)) return;
    const int slot = sift_atomic_add(n_cand, 1);
    if (slot < cand_cap) cand[slot] = k;
  }
};

// calcOrientationHist + the peak loop of findScaleSpaceExtrema; appends one raw keypoint per peak.
struct SiftOrient {
  SiftTables t;
  int L;
  const SiftCand* cand; const int* n_cand; int cand_cap;
  SiftKpt* kpt; int* n_kpt; int kpt_cap;
  static constexpr int SCRATCH = SIFT_ORI_HIST_BINS + 4;
  SIFT_HD long count() const { return cand_cap; }
  SIFT_HD void operator()(long i, float* temp) const {
    const int nc = *n_cand;
    if (i >= (nc < cand_cap ? nc : cand_cap)) return;
    const SiftCand k = cand[i];
    const int o = k.octave_packed & 255, n = SIFT_ORI_HIST_BINS;
    const float* img = t.gauss[o * (L + 3) + k.layer];
    const int rows = t.dims[2 * o], cols = t.dims[2 * o + 1];
    const float scl_octv = k.size * 0.5f / (float)(1 << o);
    const int radius = sift_round(SIFT_ORI_RADIUS * scl_octv);
    const float sigma = SIFT_ORI_SIG_FCTR * scl_octv;
    const float expf_scale = -1.f / (2.f * sigma * sigma);
    float* th = temp + 2;  // temphist[-2 .. n+1]
    for (int b = 0; b < n; ++b) th[b] = 0.f;
    for (int a = -radius; a <= radius; a++) {
      const int y = k.r + a;
      if (y <= 0 || y >= rows - 1) continue;
      for (int j = -radius; j <= radius; j++) {
        const int x = k.c + j;
        if (x <= 0 || x >= cols - 1) continue;
        const float dx = img[(long)y * cols + x + 1] - img[(long)y * cols + x - 1];
        const float dy = img[(long)(y - 1) * cols + x] - img[(long)(y + 1) * cols + x];
        const float wt = expf((float)(a * a + j * j) * expf_scale);
        const float ori = sift_fast_atan2(dy, dx), mag = sift_magnitude(dx, dy);
        int bin = sift_round((n / 360.f) * ori);
        if (bin >= n) bin -= n;
        if (bin < 0) bin += n;
        th[bin] += wt * mag;
      }
    }
    th[-1] = th[n - 1]; th[-2] = th[n - 2]; th[n] = th[0]; th[n + 1] = th[1];
    float hist[SIFT_ORI_HIST_BINS];
    float omax = 0.f;
    for (int b = 0; b < n; b++) {
      hist[b] = (th[b - 2] + th[b + 2]) * (1.f / 16.f) + (th[b - 1] + th[b + 1]) * (4.f / 16.f) + th[b] * (6.f / 16.f);
      omax = b == 0 ? hist[0] : fmaxf(omax, hist[b]);
    }
    const float mag_thr = omax * SIFT_ORI_PEAK_RATIO;
    for (int j = 0; j < n; j++) {
      const int l = j > 0 ? j - 1 : n - 1, r2 = j < n - 1 ? j + 1 : 0;
      if (hist[j] > hist[l] && hist[j] > hist[r2] && hist[j] >= mag_thr) {
        float bin = j + 0.5f * (hist[l] - hist[r2]) / (hist[l] - 2 * hist[j] + hist[r2]);
        bin = bin < 0 ? n + bin : bin >= n ? bin - n : bin;
        float angle = 360.f - (360.f / n) * bin;
        if (fabsf(angle - 360.f) < FLT_EPSILON) angle = 0.f;
        SiftKpt q;
        // detectAndCompute's first-octave adjustment (firstOctave = -1): coordinates and size halved, octave - 1
        q.x = k.x * 0.5f; q.y = k.y * 0.5f; q.size = k.size * 0.5f;
        q.angle = angle; q.response = k.response;
        q.octave_packed = (k.octave_packed & ~255) | ((k.octave_packed - 1) & 255);
        q.o = o; q.layer = k.layer;
        const int slot = sift_atomic_add(n_kpt, 1);
        if (slot < kpt_cap) kpt[slot] = q;
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// ordering and filtering of the raw keypoints: every stage counts over all raw keypoints (n is at most a few
// thousand per image), which gives a deterministic total order without a sort
// ---------------------------------------------------------------------------------------------------------------------
// KeyPoint_LessThan: x, y ascending, size descending, angle ascending, response descending, octave descending; full
// ties by list index (such keypoints are identical in every output).
SIFT_HD bool sift_lex_less(const SiftKpt& a, int ia, const SiftKpt& b, int ib) {
  if (a.x != b.x) return a.x < b.x;
  if (a.y != b.y) return a.y < b.y;
  if (a.size != b.size) return a.size > b.size;
  if (a.angle != b.angle) return a.angle < b.angle;
  if (a.response != b.response) return a.response > b.response;
  if (a.octave_packed != b.octave_packed) return a.octave_packed > b.octave_packed;
  return ia < ib;
}

SIFT_HD float sift_deg2rad(float a) { return a * ((float)M_PI / 180.0f); }  // np.deg2rad on float32

struct SiftPost {  // per-image state of the filtering passes, indexed by lexicographic position
  const SiftKpt* kpt; const int* n_kpt; int cap;
  int* order;   // [cap] position -> raw index
  int* flags;   // [cap] bit 0 unique, 1 retained, 2 filter_dog_point, 3 NMS
  int* pix;     // [cap] filter_dog_point pixel (i * w + j) of the position
  int* counters;  // [0] n_raw (clamped) [1] capped [2] n_out [3] overflow
  int w;
};

struct SiftSortLex {  // order[rank] = i
  SiftPost s;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return s.cap; }
  SIFT_HD void operator()(long i, float*) const {
    const int n = *s.n_kpt < s.cap ? *s.n_kpt : s.cap;
    if (i == 0) { s.counters[0] = n; s.counters[3] = *s.n_kpt > s.cap || s.counters[4] > s.cap; }
    if (i >= n) return;
    const SiftKpt a = s.kpt[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += sift_lex_less(s.kpt[j], j, a, (int)i);
    s.order[rank] = (int)i;
  }
};

struct SiftRetain {  // removeDuplicatedSorted, then retainBest(nfeatures): keep responses >= the nfeatures-th largest
  SiftPost s; SiftParams p;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return s.cap; }
  SIFT_HD static bool same(const SiftKpt& a, const SiftKpt& b) {
    return a.x == b.x && a.y == b.y && a.size == b.size && a.angle == b.angle;
  }
  SIFT_HD void operator()(long i, float*) const {
    const int n = s.counters[0];
    if (i >= n) return;
    const SiftKpt a = s.kpt[s.order[i]];
    const bool uniq = i == 0 || !same(s.kpt[s.order[i - 1]], a);
    int n_uniq = 0, greater = 0;
    for (int j = 0; j < n; ++j) {
      const SiftKpt b = s.kpt[s.order[j]];
      if (j > 0 && same(s.kpt[s.order[j - 1]], b)) continue;
      ++n_uniq;
      greater += b.response > a.response;
    }
    const bool cut = p.nfeatures > 0 && n_uniq > p.nfeatures;
    const bool keep = uniq && (!cut || greater < p.nfeatures);
    // filter_dog_point's pixel: np.round(pt - 0.5) (half to even), as (row, column)
    const int pj = (int)rintf(a.x - 0.5f), pi = (int)rintf(a.y - 0.5f);
    s.pix[i] = pi * s.w + pj;
    s.flags[i] = (uniq ? 1 : 0) | (keep ? 2 : 0);
    if (i == 0) s.counters[1] = cut;
  }
};

struct SiftDogFilter {  // filter_dog_point, duplicates: highest score per pixel, then lowest |angle|, ties kept
  SiftPost s; SiftParams p;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return s.cap; }
  SIFT_HD void operator()(long i, float*) const {
    const int n = s.counters[0];
    if (i >= n) return;
    int f = s.flags[i];
    if ((f & 2) && p.nms_radius >= 0) {
      const SiftKpt a = s.kpt[s.order[i]];
      const float oa = fabsf(sift_deg2rad(a.angle));
      bool keep = true;
      for (int j = 0; j < n && keep; ++j) {
        if (!(s.flags[j] & 2) || s.pix[j] != s.pix[i]) continue;
        const SiftKpt b = s.kpt[s.order[j]];
        if (b.response > a.response) keep = false;
        else if (b.response == a.response && fabsf(sift_deg2rad(b.angle)) < oa) keep = false;
      }
      if (keep) f |= 4;
    } else if (f & 2) {
      f |= 4;
    }
    s.flags[i] = f;
  }
};

struct SiftNms {  // filter_dog_point with nms_radius > 0: max-pool NMS over the surviving pixels' scores
  SiftPost s; SiftParams p;
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return s.cap; }
  SIFT_HD void operator()(long i, float*) const {
    const int n = s.counters[0];
    if (i >= n) return;
    int f = s.flags[i];
    if ((f & 4) && p.nms_radius > 0) {
      const SiftKpt a = s.kpt[s.order[i]];
      const int ai = s.pix[i] / s.w, aj = s.pix[i] % s.w;
      bool keep = true;
      for (int j = 0; j < n && keep; ++j) {
        if (!(s.flags[j] & 4)) continue;
        const int bi = s.pix[j] / s.w, bj = s.pix[j] % s.w;
        if (abs(bi - ai) > p.nms_radius || abs(bj - aj) > p.nms_radius) continue;
        if (s.kpt[s.order[j]].response > a.response) keep = false;
      }
      if (keep) f |= 8;
    } else if (f & 4) {
      f |= 8;
    }
    s.flags[i] = f;
  }
};

struct SiftSelect {  // top-k by score; output slot of every survivor: lexicographic order, or by score when capped
  SiftPost s; SiftParams p;
  int* out_src;  // [max_kpts] slot -> lexicographic position
  static constexpr int SCRATCH = 0;
  SIFT_HD long count() const { return s.cap; }
  SIFT_HD void operator()(long i, float*) const {
    const int n = s.counters[0];
    if (i >= n) {
      if (n == 0 && i == 0) s.counters[2] = 0;
      return;
    }
    const bool alive = s.flags[i] & 8;
    if (!alive && i != 0) return;
    const float sa = s.kpt[s.order[i]].response;
    int n_alive = 0, before_lex = 0, before_score = 0;
    for (int j = 0; j < n; ++j) {
      if (!(s.flags[j] & 8)) continue;
      ++n_alive;
      before_lex += j < i;
      const float sb = s.kpt[s.order[j]].response;
      before_score += sb > sa || (sb == sa && j < i);
    }
    const bool topk = p.max_kpts > 0 && n_alive > p.max_kpts;
    const int n_out = topk ? p.max_kpts : n_alive;
    if (i == 0) s.counters[2] = n_out;
    if (!alive) return;
    const bool by_score = topk || s.counters[1];
    const int slot = by_score ? before_score : before_lex;
    if (slot < n_out) out_src[slot] = (int)i;
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// descriptors (calcSIFTDescriptor) and outputs
// ---------------------------------------------------------------------------------------------------------------------
struct SiftDescribe {
  SiftTables t; int L;
  SiftPost s; SiftParams p;
  const int* out_src;
  int cap_out;
  float* kpts; float* scales; float* oris; float* scores; float* desc;  // this image's rows; desc null: no descriptors
  static constexpr int SCRATCH = SIFT_DESC_HIST;
  SIFT_HD long count() const { return cap_out; }
  SIFT_HD void operator()(long slot, float* hist) const {
    const int n_out = s.counters[2];
    if (slot >= n_out) {
      kpts[2 * slot] = kpts[2 * slot + 1] = 0.f;
      scales[slot] = oris[slot] = scores[slot] = 0.f;
      for (int k = 0; desc && k < SIFT_DESC; ++k) desc[slot * SIFT_DESC + k] = 0.f;
      return;
    }
    const SiftKpt kp = s.kpt[s.order[out_src[slot]]];
    kpts[2 * slot] = kp.x; kpts[2 * slot + 1] = kp.y;
    scales[slot] = kp.size; oris[slot] = sift_deg2rad(kp.angle); scores[slot] = kp.response;
    if (!desc) return;
    float* dst = desc + slot * SIFT_DESC;

    // unpackOctave: scale = 1 / 2^octave (2 for octave -1)
    const int octave = kp.o - 1;
    const float scale = octave >= 0 ? 1.f / (float)(1 << octave) : (float)(1 << -octave);
    const float size = kp.size * scale, ptx = kp.x * scale, pty = kp.y * scale;
    const float* img = t.gauss[kp.o * (L + 3) + kp.layer];
    const int rows = t.dims[2 * kp.o], cols = t.dims[2 * kp.o + 1];
    float angle = 360.f - kp.angle;
    if (fabsf(angle - 360.f) < FLT_EPSILON) angle = 0.f;
    const float ori = angle, scl = size * 0.5f;

    const int d = SIFT_DESCR_WIDTH, n = SIFT_DESCR_HIST_BINS;
    const int px = sift_round(ptx), py = sift_round(pty);
    float cos_t = cosf(ori * (float)(M_PI / 180)), sin_t = sinf(ori * (float)(M_PI / 180));
    const float bins_per_rad = n / 360.f, exp_scale = -1.f / (d * d * 0.5f), hist_width = SIFT_DESCR_SCL_FCTR * scl;
    int radius = sift_round(hist_width * 1.4142135623730951f * (d + 1) * 0.5f);
    const int diag = (int)sqrt((double)cols * cols + (double)rows * rows);
    radius = radius < diag ? radius : diag;
    cos_t /= hist_width;
    sin_t /= hist_width;
    for (int k = 0; k < SIFT_DESC_HIST; ++k) hist[k] = 0.f;
    for (int i = -radius; i <= radius; i++)
      for (int j = -radius; j <= radius; j++) {
        const float c_rot = j * cos_t - i * sin_t, r_rot = j * sin_t + i * cos_t;
        float rbin = r_rot + d / 2 - 0.5f, cbin = c_rot + d / 2 - 0.5f;
        const int r = py + i, c = px + j;
        if (!(rbin > -1 && rbin < d && cbin > -1 && cbin < d && r > 0 && r < rows - 1 && c > 0 && c < cols - 1)) continue;
        const float dx = img[(long)r * cols + c + 1] - img[(long)r * cols + c - 1];
        const float dy = img[(long)(r - 1) * cols + c] - img[(long)(r + 1) * cols + c];
        const float wexp = (c_rot * c_rot + r_rot * r_rot) * exp_scale;
        const float o_k = sift_fast_atan2(dy, dx), m_k = sift_magnitude(dx, dy), w_k = expf(wexp);
        float obin = (o_k - ori) * bins_per_rad;
        const float mag = m_k * w_k;
        const int r0 = sift_floor(rbin), c0 = sift_floor(cbin);
        int o0 = sift_floor(obin);
        rbin -= r0; cbin -= c0; obin -= o0;
        if (o0 < 0) o0 += n;
        if (o0 >= n) o0 -= n;
        const float v_r1 = mag * rbin, v_r0 = mag - v_r1;
        const float v_rc11 = v_r1 * cbin, v_rc10 = v_r1 - v_rc11;
        const float v_rc01 = v_r0 * cbin, v_rc00 = v_r0 - v_rc01;
        const float v_rco111 = v_rc11 * obin, v_rco110 = v_rc11 - v_rco111;
        const float v_rco101 = v_rc10 * obin, v_rco100 = v_rc10 - v_rco101;
        const float v_rco011 = v_rc01 * obin, v_rco010 = v_rc01 - v_rco011;
        const float v_rco001 = v_rc00 * obin, v_rco000 = v_rc00 - v_rco001;
        const int idx = ((r0 + 1) * (d + 2) + c0 + 1) * (n + 2) + o0;
        hist[idx] += v_rco000;
        hist[idx + 1] += v_rco001;
        hist[idx + (n + 2)] += v_rco010;
        hist[idx + (n + 3)] += v_rco011;
        hist[idx + (d + 2) * (n + 2)] += v_rco100;
        hist[idx + (d + 2) * (n + 2) + 1] += v_rco101;
        hist[idx + (d + 3) * (n + 2)] += v_rco110;
        hist[idx + (d + 3) * (n + 2) + 1] += v_rco111;
      }
    // circular orientation bins, then the 128 values (written to dst first, as OpenCV does)
    for (int i = 0; i < d; i++)
      for (int j = 0; j < d; j++) {
        const int idx = ((i + 1) * (d + 2) + (j + 1)) * (n + 2);
        hist[idx] += hist[idx + n];
        hist[idx + 1] += hist[idx + n + 1];
        for (int k = 0; k < n; k++) dst[(i * d + j) * n + k] = hist[idx + k];
      }
    float nrm2 = 0;
    for (int k = 0; k < SIFT_DESC; k++) nrm2 += dst[k] * dst[k];
    const float thr = sqrtf(nrm2) * SIFT_DESCR_MAG_THR;
    nrm2 = 0;
    for (int k = 0; k < SIFT_DESC; k++) {
      const float v = fminf(dst[k], thr);
      dst[k] = v;
      nrm2 += v * v;
    }
    nrm2 = SIFT_INT_DESCR_FCTR / fmaxf(sqrtf(nrm2), FLT_EPSILON);
    float l1 = 0.f;
    for (int k = 0; k < SIFT_DESC; k++) {  // saturate_cast<uchar>
      int q = sift_round(dst[k] * nrm2);
      q = q < 0 ? 0 : q > 255 ? 255 : q;
      dst[k] = (float)q;
      l1 += (float)q;  // exact: integers
    }
    if (!p.rootsift) return;
    // sift_to_rootsift: L1 normalise (eps 1e-6), clip at 1e-6, sqrt, L2 normalise (eps 1e-6)
    const float eps = 1e-6f, n1 = fmaxf(l1, eps);
    float l2 = 0.f;
    for (int k = 0; k < SIFT_DESC; k++) {
      const float v = sqrtf(fmaxf(dst[k] / n1, eps));
      dst[k] = v;
      l2 += v * v;
    }
    const float n2 = fmaxf(sqrtf(l2), eps);
    for (int k = 0; k < SIFT_DESC; k++) dst[k] = dst[k] / n2;
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// sizes and orchestration
// ---------------------------------------------------------------------------------------------------------------------
// Octave count for an h x w image: cvRound(log2(min side of the upsampled base) - 2) + 1.
inline int sift_num_octaves(int h, int w) {
  const int m = 2 * (h < w ? h : w);
  int n = (int)lrint(log((double)m) / log(2.) - 2) + 1;
  return n < 1 ? 1 : n > SIFT_MAX_OCTAVES ? SIFT_MAX_OCTAVES : n;
}

// Capacity of the candidate and raw keypoint lists per image (an image that overflows is reported, not truncated).
inline int sift_raw_cap(int H, int W) {
  const long c = (long)H * W / 4 + 4096;
  return (int)(c < (1L << 24) ? c : (1L << 24));
}

// cv::getGaussianKernel(ksize = round(8 sigma + 1) | 1, sigma) in double, rounded to float.
inline SiftKernel sift_kernel(double sigma) {
  SiftKernel k{};
  int ks = (int)lrint(sigma * 4 * 2 + 1) | 1;
  if (ks > SIFT_MAX_KSIZE) ks = SIFT_MAX_KSIZE;
  k.ksize = ks;
  double t[SIFT_MAX_KSIZE], sum = 0;
  const double scale2X = -0.5 / (sigma * sigma);
  for (int i = 0; i < ks; i++) {
    const double x = i - (ks - 1) * 0.5;
    t[i] = exp(scale2X * x * x);
    sum += t[i];
  }
  for (int i = 0; i < ks; i++) k.k[i] = (float)(t[i] / sum);
  return k;
}

struct SiftWs {  // workspace carve for one image at most H x W (images are processed one after the other)
  float* q;                 // [H * W] 8-bit gray
  float* tmp;               // [4 H W] row-pass output
  float* pyr;               // all Gaussians and DoGs, octave after octave
  SiftCand* cand;
  SiftKpt* kpt;
  int *order, *flags, *pix, *out_src, *counters;  // counters: [0..3] SiftPost, [4] n_cand, [5] n_kpt
  int raw_cap;
  size_t bytes;
};

inline size_t sift_pyr_floats(int H, int W, int L) {
  size_t f = 0;
  int h = 2 * H, w = 2 * W;
  for (int o = 0; o < sift_num_octaves(H, W); ++o) {
    f += (size_t)(2 * L + 5) * h * w;
    h /= 2; w /= 2;
  }
  return f;
}

inline void sift_carve(char* base, int H, int W, int L, int max_kpts, SiftWs* w) {
  WsBump b{base, 0};
  w->raw_cap = sift_raw_cap(H, W);
  w->counters = b.take<int>(8);
  w->q = b.take<float>((size_t)H * W);
  w->tmp = b.take<float>((size_t)4 * H * W);
  w->pyr = b.take<float>(sift_pyr_floats(H, W, L));
  w->cand = b.take<SiftCand>(w->raw_cap);
  w->kpt = b.take<SiftKpt>(w->raw_cap);
  w->order = b.take<int>(w->raw_cap);
  w->flags = b.take<int>(w->raw_cap);
  w->pix = b.take<int>(w->raw_cap);
  w->out_src = b.take<int>(max_kpts > 0 ? max_kpts : 1);
  w->bytes = b.bytes();
}

// Host-side layout of one image's pyramid inside w.pyr: gauss[o][i] and dog[o][i] pointers and octave sizes.
struct SiftPyr {
  int n_oct, L;
  int h[SIFT_MAX_OCTAVES], w[SIFT_MAX_OCTAVES];
  float* gauss[SIFT_MAX_OCTAVES][SIFT_MAX_LAYERS + 3];
  float* dog[SIFT_MAX_OCTAVES][SIFT_MAX_LAYERS + 2];
};

inline void sift_layout(const SiftWs& ws, int h, int w, int L, SiftPyr* P) {
  P->n_oct = sift_num_octaves(h, w);
  P->L = L;
  float* f = ws.pyr;
  int hh = 2 * h, ww = 2 * w;
  for (int o = 0; o < P->n_oct; ++o) {
    P->h[o] = hh; P->w[o] = ww;
    for (int i = 0; i < L + 3; ++i) { P->gauss[o][i] = f; f += (size_t)hh * ww; }
    for (int i = 0; i < L + 2; ++i) { P->dog[o][i] = f; f += (size_t)hh * ww; }
    hh /= 2; ww /= 2;
  }
}

// One image: image [C, H, W] (device), crop (h, w); writes cap_out rows of outputs and counters[2] (n_out), [3]
// (overflow).  `Exec` provides run(functor), which runs the functor over its count() indices in stream order, and
// zero(ptr, n_ints).
template <class Exec>
int sift_run(Exec& ex, const SiftParams& p, const float* image, int C, int H, int W, int h, int w, const SiftWs& ws,
             int cap_out, float* kpts, float* scales, float* oris, float* scores, float* desc) {
  SiftPyr P;
  sift_layout(ws, h, w, p.L, &P);
  const int L = p.L;
  int rc = 0;
  rc |= ex.zero(ws.counters, 8);
  rc |= ex.run(SiftGray{image, ws.q, C, H, W, h, w});
  // initial image: 2x linear upsample, blur by sqrt(sigma^2 - (2 * 0.5)^2) (createInitialImage, float sigma)
  rc |= ex.run(SiftUpsample{ws.q, P.gauss[0][1], h, w});
  const float sig_diff = sqrtf(fmaxf(p.sigma * p.sigma - 0.5f * 0.5f * 4, 0.01f));
  {
    const SiftKernel k = sift_kernel(sig_diff);
    rc |= ex.run(SiftRowBlur{P.gauss[0][1], ws.tmp, P.h[0], P.w[0], k});
    rc |= ex.run(SiftColBlur{ws.tmp, P.gauss[0][0], nullptr, nullptr, P.h[0], P.w[0], k});
  }
  // buildGaussianPyramid: incremental sigmas (double), DoG in the column pass
  double sig[SIFT_MAX_LAYERS + 3];
  sig[0] = p.sigma;
  const double kk = pow(2., 1. / L);
  for (int i = 1; i < L + 3; i++) {
    const double sig_prev = pow(kk, (double)(i - 1)) * p.sigma, sig_total = sig_prev * kk;
    sig[i] = sqrt(sig_total * sig_total - sig_prev * sig_prev);
  }
  for (int o = 0; o < P.n_oct; ++o) {
    if (o > 0) rc |= ex.run(SiftDecimate{P.gauss[o - 1][L], P.gauss[o][0], P.w[o - 1], P.h[o], P.w[o]});
    for (int i = 1; i < L + 3; ++i) {
      const SiftKernel k = sift_kernel(sig[i]);
      rc |= ex.run(SiftRowBlur{P.gauss[o][i - 1], ws.tmp, P.h[o], P.w[o], k});
      rc |= ex.run(SiftColBlur{ws.tmp, P.gauss[o][i], P.gauss[o][i - 1], P.dog[o][i - 1], P.h[o], P.w[o], k});
    }
  }
  SiftTables tab{};  // for the stages that look up any octave
  for (int o = 0; o < P.n_oct; ++o) {
    for (int i = 0; i < L + 3; ++i) tab.gauss[o * (L + 3) + i] = P.gauss[o][i];
    tab.dims[2 * o] = P.h[o]; tab.dims[2 * o + 1] = P.w[o];
  }
  // findScaleSpaceExtrema
  int* n_cand = ws.counters + 4;
  int* n_kpt = ws.counters + 5;
  for (int o = 0; o < P.n_oct; ++o) {
    SiftOctave oc{};
    for (int i = 0; i < L + 3; ++i) oc.gauss[i] = P.gauss[o][i];
    for (int i = 0; i < L + 2; ++i) oc.dog[i] = P.dog[o][i];
    oc.h = P.h[o]; oc.w = P.w[o];
    for (int i = 1; i <= L; ++i) rc |= ex.run(SiftDetect{oc, p, o, i, ws.cand, n_cand, ws.raw_cap});
  }
  rc |= ex.run(SiftOrient{tab, L, ws.cand, n_cand, ws.raw_cap, ws.kpt, n_kpt, ws.raw_cap});
  // ordering, OpenCV's dedupe / retainBest, filter_dog_point, top-k
  const SiftPost s{ws.kpt, n_kpt, ws.raw_cap, ws.order, ws.flags, ws.pix, ws.counters, w};
  rc |= ex.run(SiftSortLex{s});
  rc |= ex.run(SiftRetain{s, p});
  rc |= ex.run(SiftDogFilter{s, p});
  rc |= ex.run(SiftNms{s, p});
  rc |= ex.run(SiftSelect{s, p, ws.out_src});
  rc |= ex.run(SiftDescribe{tab, L, s, p, ws.out_src, cap_out, kpts, scales, oris, scores, desc});
  return rc;
}
