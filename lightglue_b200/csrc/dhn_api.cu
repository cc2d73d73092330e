// C ABI of the DoG-HardNet extractor (include/doghardnet_b200.h): lightglue/dog_hardnet.py, i.e. the SIFT extractor's
// keypoints and kornia's LAFDescriptor(HardNet(pretrained)) on the LAFs laf_from_center_scale_ori(kpts, 6 scales,
// rad2deg(oris)).
//
// Per image, in stream order, in one set of workspace buffers:
//   SIFT's detection (sift_api.cu: sift_detect_image, the functors of sift_pipeline.h without the descriptor histograms)
//   the float gray crop and its pyrdown pyramid (5x5 binomial blur with reflect borders, then bilinear resize to
//   (int(h / 2), w // 2)), up to and including the first level whose shorter side is < 32 (kornia's
//   extract_patches_from_pyramid; keypoints whose level is never reached keep an all-zero patch)
//   per chunk of NP keypoints:
//     dhn_patch_kernel: level and affine grid of each keypoint, bilinear 32x32 patch (border clamp), mean / unbiased
//     std normalisation, conv 0 (1 -> 32, K = 9, fp32, folded BatchNorm + ReLU) -> padded NHWC bf16 hi / lo, 34 x 34
//     per patch, 32 channels zero-padded to 64
//     conv 1 (3x3) / conv 3 (3x3) / conv 5 (3x3) on the tensor cores (tc_conv); conv 2 and conv 4 (stride 2) as
//     tc_conv by phase split over the four polyphase images of their padded input (dhn_phase_kernel), each held in the
//     output's padded frame (18 x 18, 10 x 10)
//     dhn_gather_kernel: the 8 x 8 x 128 output of conv 5 of every keypoint -> one [8192] row
//   conv 6 (8 x 8, K = 8192) as one tensor-core GEMM over the image's gathered rows (fp32 out), then F.normalize.
// Every BatchNorm (eval, affine=False) is folded into its convolution's weights and a bias at dhn_create, in double
// (tc_conv_weights_create).
// GEMM rows past the device-side keypoint count are skipped through SeqState.len: nothing is read back to the host.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <math.h>
#include <new>

#include "../../include/doghardnet_b200.h"
#include "../../include/sift_b200.h"
#include "lg_internal.h"
#include "lg_tc.h"
#include "ws_bump.h"

size_t sift_detect_workspace_bytes(const SiftConfig& c, int H, int W);
int sift_detect_image(const SiftConfig& c, const float* image, int channels, int H, int W, int h, int w, void* workspace,
                      int64_t cap, float* keypoints, float* scales, float* oris, float* scores, int32_t* count,
                      cudaStream_t stream);

namespace {

constexpr int PS = 32;           // patch side
constexpr int NP = 256;          // patches per chunk
constexpr int DESC = 128;
constexpr int RA = 34 * 34, RB = 18 * 18, RC = 10 * 10;  // padded rows per patch at 32 x 32, 16 x 16, 8 x 8
constexpr int K6 = 64 * 128;     // conv 6: 8 x 8 taps x 128 channels
constexpr int MAXLV = 24;        // pyramid levels (2^17-pixel sides need 13)
constexpr int NL = 7;
struct HLayer { int cin, cout, k; };
constexpr HLayer HL[NL] = {{1, 32, 3}, {32, 32, 3}, {32, 64, 3}, {64, 64, 3}, {64, 128, 3}, {128, 128, 3}, {128, 128, 8}};

size_t layer_blob_off(int l) {  // weight [cout, cin, k, k], running_mean [cout], running_var [cout]
  size_t o = 0;
  for (int i = 0; i < l; ++i) o += (size_t)HL[i].cout * HL[i].cin * HL[i].k * HL[i].k + 2 * HL[i].cout;
  return o;
}

struct PyrTab {  // levels of one image's pyramid: float offset in the pyramid buffer, height, width
  int n;
  long off[MAXLV];
  int h[MAXLV], w[MAXLV];
};
PyrTab pyr_tab(int h, int w) {
  PyrTab t{};
  long off = 0;
  for (t.n = 0; t.n < MAXLV;) {
    t.off[t.n] = off; t.h[t.n] = h; t.w[t.n] = w;
    off += (long)h * w;
    ++t.n;
    if (std::min(h, w) < PS) break;  // kornia samples this level, then stops
    h = (int)((float)h / 2.f); w = w / 2;
  }
  return t;
}
long pyr_floats(int h, int w) {
  const PyrTab t = pyr_tab(h, w);
  return t.off[t.n - 1] + (long)t.h[t.n - 1] * t.w[t.n - 1];
}

struct Geo {
  int cap;  // keypoints per image (max_num_keypoints)
  int nchunk;
  TcRows A, B, C, D;  // 32 x 32, 16 x 16, 8 x 8 levels of one chunk; conv 6 rows of one image
};
Geo geometry(int cap) {
  Geo g;
  g.cap = cap;
  g.nchunk = (cap + NP - 1) / NP;
  g.A = tc_rows((long)NP * RA);
  g.B = tc_rows((long)NP * RB);
  g.C = tc_rows((long)NP * RC);
  g.D = tc_rows(cap);
  return g;
}

struct DhnWs {
  char* sift;                // SIFT's workspace
  float* pyr;                // the gray crop and its pyramid levels
  int* state;                // SeqState words: [chunk][level A, B, C][len[2], stop_layer, -], then conv 6's
  __nv_bfloat16 *uh, *ul;    // conv 0 output (level A) / polyphase input of conv 2
  __nv_bfloat16 *vh, *vl;    // conv 1 output (level A) / polyphase input of conv 4
  __nv_bfloat16 *bh, *bl;    // conv 2 output / conv 3 output (two maps at level B)
  __nv_bfloat16 *b2h, *b2l;
  __nv_bfloat16 *ch, *cl;    // conv 4 output / conv 5 output (level C, 128 channels)
  __nv_bfloat16 *c2h, *c2l;
  __nv_bfloat16 *gh, *gl;    // [D rows, 8192] conv 6 input rows
  float* dout;               // [D rows, 128]
  size_t bytes[DHN_LAYOUT_BUFFERS];  // sizes of the buffers dhn_workspace_layout reports, in its order
};

size_t carve(char* base, const Geo& g, size_t sift_bytes, int H, int W, DhnWs* w) {
  WsBump b{base, 0};
  constexpr size_t A = 1024;
  w->sift = b.take<char>(sift_bytes, A);
  w->pyr = b.take<float>((size_t)pyr_floats(H, W), A);
  w->state = b.take<int>((size_t)(g.nchunk * 3 + 1) * 4, A);
  w->bytes[15] = b.last;
  const size_t u = (size_t)std::max(g.A.rows, 4 * g.B.rows) * 64, v = (size_t)std::max(g.A.rows, 4 * g.C.rows) * 64;
  const size_t bb = (size_t)g.B.rows * 64, cc = (size_t)g.C.rows * 128;
  __nv_bfloat16** maps[12] = {&w->uh, &w->ul, &w->vh, &w->vl, &w->bh, &w->bl, &w->b2h, &w->b2l, &w->ch, &w->cl, &w->c2h, &w->c2l};
  const size_t n[12] = {u, u, v, v, bb, bb, bb, bb, cc, cc, cc, cc};
  for (int i = 0; i < 12; ++i) {
    *maps[i] = b.take<__nv_bfloat16>(n[i], A);
    w->bytes[i] = b.last;
  }
  w->gh = b.take<__nv_bfloat16>((size_t)g.D.rows * K6, A); w->bytes[12] = b.last;
  w->gl = b.take<__nv_bfloat16>((size_t)g.D.rows * K6, A); w->bytes[13] = b.last;
  w->dout = b.take<float>((size_t)g.D.rows * DESC, A); w->bytes[14] = b.last;
  return b.bytes();
}

__device__ __forceinline__ int n_valid(const int* count, long cap) {
  const int n = *count;
  return n < 0 ? 0 : (n > cap ? (int)cap : n);
}

// kornia's rgb_to_grayscale (0.299 r + 0.587 g + 0.114 b, unfused, in that order) of the crop [:h, :w]
__global__ void __launch_bounds__(256) dhn_gray_kernel(const float* __restrict__ img, int C, int H, int W, int h, int w,
                                                       float* __restrict__ out) {
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= (long)h * w) return;
  const long p = (i / w) * W + i % w, plane = (long)H * W;
  float g = img[p];
  if (C == 3) g = __fadd_rn(__fadd_rn(__fmul_rn(0.299f, img[p]), __fmul_rn(0.587f, img[p + plane])), __fmul_rn(0.114f, img[p + 2 * plane]));
  out[i] = g;
}

__device__ __forceinline__ int reflect(int p, int n) {  // torch's "reflect" padding (edge not repeated), |overhang| <= 2 < n
  return p < 0 ? -p : (p >= n ? 2 * n - 2 - p : p);
}

// kornia's pyrdown: filter2d with the 5x5 binomial kernel / 256 (reflect borders), then F.interpolate(size=(ho, wo),
// bilinear, align_corners=False): source (d + 0.5) (in / out) - 0.5, clamped at 0
__global__ void __launch_bounds__(256) dhn_pyrdown_kernel(const float* __restrict__ in, int hi, int wi, float* __restrict__ out,
                                                          int ho, int wo) {
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= (long)ho * wo) return;
  const int oy = (int)(i / wo), ox = (int)(i % wo);
  const float k5[5] = {1.f, 4.f, 6.f, 4.f, 1.f};
  const float sy = fmaxf(((float)hi / (float)ho) * (oy + 0.5f) - 0.5f, 0.f), sx = fmaxf(((float)wi / (float)wo) * (ox + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < hi - 1), x1 = x0 + (x0 < wi - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  auto blur = [&](int y, int x) {
    float s = 0.f;
#pragma unroll
    for (int dy = 0; dy < 5; ++dy) {
      const float* row = in + (long)reflect(y + dy - 2, hi) * wi;
      float r = 0.f;
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) r += k5[dx] * row[reflect(x + dx - 2, wi)];
      s += k5[dy] * r;
    }
    return s * (1.f / 256.f);
  };
  out[i] = (1.f - ly) * ((1.f - lx) * blur(y0, x0) + lx * blur(y0, x1)) + ly * ((1.f - lx) * blur(y1, x0) + lx * blur(y1, x1));
}

// the tc_rows_state words of every chunk and level, and of conv 6, from the device-side keypoint count
__global__ void dhn_state_kernel(const int* __restrict__ count, long cap, int nchunk, int lpa, int lpb, int lpc, int lpd,
                                 int* __restrict__ st) {
  const int n = n_valid(count, cap);
  auto put = [&](int* s, long used, int lp) {
    s[0] = (int)(used < lp ? used : lp);
    s[1] = (int)(used - lp < 0 ? 0 : (used - lp > lp ? lp : used - lp));
    s[2] = 0; s[3] = 0;
  };
  for (int c = 0; c < nchunk; ++c) {
    const long m = max(0, min(n - c * NP, NP));
    put(st + (c * 3 + 0) * 4, m * RA, lpa);
    put(st + (c * 3 + 1) * 4, m * RB, lpb);
    put(st + (c * 3 + 2) * 4, m * RC, lpc);
  }
  put(st + nchunk * 12, n, lpd);
}

// One block per keypoint of the chunk: kornia's level selection and patch grid, the bilinear 32 x 32 patch, HardNet's
// input normalisation and conv 0 (folded BatchNorm, ReLU) -> padded NHWC bf16 hi / lo [34 x 34 rows, 64 channels]
__global__ void __launch_bounds__(256) dhn_patch_kernel(const float* __restrict__ pyr, const PyrTab t, const float* __restrict__ kpts,
                                                        const float* __restrict__ scales, const float* __restrict__ oris,
                                                        const int* __restrict__ count, long cap, int k0, const float* __restrict__ w0,
                                                        const float* __restrict__ b0, __nv_bfloat16* __restrict__ oh,
                                                        __nv_bfloat16* __restrict__ ol) {
  __shared__ float sp[34 * 34];  // normalised patch, pixel (i, j) at (i + 1, j + 1), zero border
  __shared__ float sw[32 * 9 + 32];
  __shared__ float red[8];
  const int p = blockIdx.x, tid = threadIdx.x;
  const int k = k0 + p;
  if (k >= n_valid(count, cap)) return;
  for (int i = tid; i < 32 * 9; i += 256) sw[i] = w0[i];
  if (tid < 32) sw[32 * 9 + tid] = b0[tid];
  for (int i = tid; i < 34 * 34; i += 256) sp[i] = 0.f;
  // LAF = [[s cos, s sin, x], [-s sin, s cos, y]], s = 6 size; its level: floor(clamp(log2(2 sqrt(|det| + 1e-10) / 32),
  // 0, max(0, min(h, w) // 32 - 1))), computed in double
  const double x = kpts[2 * k], y = kpts[2 * k + 1], s = 6.0 * (double)scales[k], th = (double)oris[k];
  const double a = s * cos(th), b = s * sin(th);
  const double lv = floor(fmin(fmax(log2(2.0 * sqrt(fabs(a * a + b * b + 1e-10)) / PS), 0.0),
                               (double)max(0, min(t.h[0], t.w[0]) / PS - 1)));
  const int L = (int)lv;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (L < t.n) {
    const int hl = t.h[L], wl = t.w[L];
    const double h0 = t.h[0] - 1, w0d = t.w[0] - 1;
    const double m = (double)min(hl - 1, wl - 1) / fmin(h0, w0d);  // normalise against level 0, denormalise at L
    const double A00 = a * m, A01 = b * m, A10 = -b * m, A11 = a * m;
    const double cx = x / w0d * (wl - 1), cy = y / h0 * (hl - 1);
    const double fx = (double)wl / (wl - 1), fy = (double)hl / (hl - 1);  // 2 g / (w - 1) - 1, then grid_sample's unnormalise
    const float* img = pyr + t.off[L];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int e = tid + 256 * q, i = e / PS, j = e % PS;
      const double xs = (2 * j + 1) / (double)PS - 1.0, ys = (2 * i + 1) / (double)PS - 1.0;
      const double gx = A00 * xs + A01 * ys + cx, gy = A10 * xs + A11 * ys + cy;
      const float px = (float)fmin(fmax(gx * fx - 0.5, 0.0), (double)(wl - 1));
      const float py = (float)fmin(fmax(gy * fy - 0.5, 0.0), (double)(hl - 1));
      const int x0 = (int)floorf(px), y0 = (int)floorf(py);
      const int x1 = min(x0 + 1, wl - 1), y1 = min(y0 + 1, hl - 1);
      const float lx = px - (float)x0, ly = py - (float)y0;
      v[q] = (1.f - ly) * ((1.f - lx) * img[(long)y0 * wl + x0] + lx * img[(long)y0 * wl + x1]) +
             ly * ((1.f - lx) * img[(long)y1 * wl + x0] + lx * img[(long)y1 * wl + x1]);
    }
  }
  auto block_sum = [&](float r) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = r;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    return tot;
  };
  const float mean = block_sum(v[0] + v[1] + v[2] + v[3]) * (1.f / (PS * PS));
  float d2 = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) d2 += (v[q] - mean) * (v[q] - mean);
  const float sd = sqrtf(block_sum(d2) * (1.f / (PS * PS - 1)));
  const float inv = 1.f / (sd + 1e-6f);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int e = tid + 256 * q;
    sp[(e / PS + 1) * 34 + e % PS + 1] = (v[q] - mean) * inv;
  }
  __syncthreads();
  // conv 0: thread item = (padded pixel, 8-channel group); groups 4..7 are the zero channels 32..63
  __nv_bfloat16* bh = oh + (long)p * RA * 64;
  __nv_bfloat16* bl = ol + (long)p * RA * 64;
  for (int it = tid; it < RA * 8; it += 256) {
    const int pix = it >> 3, g = it & 7, yy = pix / 34, xx = pix % 34;
    float o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] = 0.f;
    if (g < 4 && yy >= 1 && yy <= PS && xx >= 1 && xx <= PS) {
      float px[9];
#pragma unroll
      for (int tp = 0; tp < 9; ++tp) px[tp] = sp[(yy - 1 + tp / 3) * 34 + xx - 1 + tp % 3];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int co = g * 8 + c;
        float acc = sw[32 * 9 + co];
#pragma unroll
        for (int tp = 0; tp < 9; ++tp) acc = fmaf(px[tp], sw[co * 9 + tp], acc);
        o[c] = fmaxf(acc, 0.f);
      }
    }
    uint32_t hv[4], lv4[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      __nv_bfloat162 h2, l2;
      tc_split(o[2 * c], h2.x, l2.x);
      tc_split(o[2 * c + 1], h2.y, l2.y);
      hv[c] = *reinterpret_cast<const uint32_t*>(&h2);
      lv4[c] = *reinterpret_cast<const uint32_t*>(&l2);
    }
    *reinterpret_cast<uint4*>(bh + (long)pix * 64 + g * 8) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
    *reinterpret_cast<uint4*>(bl + (long)pix * 64 + g * 8) = make_uint4(lv4[0], lv4[1], lv4[2], lv4[3]);
  }
}

// the four polyphase images of each keypoint's padded 64-channel map (win x win per patch) in the output's padded frame
// (wo2 x wo2 per patch): phase q = 2 py + px holds padded input pixel (2 (i - 1) + py, 2 (j - 1) + px) at frame position
// (i, j), i, j >= 1 (row 0 / column 0 are zero), starting at row q pstride
__global__ void __launch_bounds__(256) dhn_phase_kernel(const __nv_bfloat16* __restrict__ ih, const __nv_bfloat16* __restrict__ il,
                                                        int win, int wo2, const int* __restrict__ count, long cap, int k0, long pstride,
                                                        __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol) {
  const long it = blockIdx.x * 256L + threadIdx.x;
  const int rpo = wo2 * wo2;
  const long per_phase = (long)NP * rpo * 8;
  if (it >= 4 * per_phase) return;
  const int q = (int)(it / per_phase);
  const long r = it % per_phase;
  const int p = (int)(r / (rpo * 8)), pos = (int)(r / 8 % rpo), g = (int)(r % 8);
  if (k0 + p >= n_valid(count, cap)) return;
  const int i = pos / wo2, j = pos % wo2;
  uint4 h = make_uint4(0, 0, 0, 0), l = h;
  if (i >= 1 && j >= 1) {
    const long src = ((long)p * win * win + (long)(2 * (i - 1) + (q >> 1)) * win + 2 * (j - 1) + (q & 1)) * 64 + g * 8;
    h = *reinterpret_cast<const uint4*>(ih + src);
    l = *reinterpret_cast<const uint4*>(il + src);
  }
  const long dst = (q * pstride + (long)p * rpo + pos) * 64 + g * 8;
  *reinterpret_cast<uint4*>(oh + dst) = h;
  *reinterpret_cast<uint4*>(ol + dst) = l;
}

// conv 6 input row of keypoint k0 + p: the 8 x 8 interior of its conv 5 output, column (ky 8 + kx) 128 + ci
__global__ void __launch_bounds__(256) dhn_gather_kernel(const __nv_bfloat16* __restrict__ ih, const __nv_bfloat16* __restrict__ il,
                                                         const int* __restrict__ count, long cap, int k0, __nv_bfloat16* __restrict__ gh,
                                                         __nv_bfloat16* __restrict__ gl) {
  const int p = blockIdx.x;
  const long k = k0 + p;
  if (k >= n_valid(count, cap)) return;
  for (int v = threadIdx.x; v < K6 / 8; v += 256) {
    const int col = v * 8, tp = col / 128, ci = col % 128;
    const long src = ((long)p * RC + (tp / 8 + 1) * 10 + tp % 8 + 1) * 128 + ci;
    *reinterpret_cast<uint4*>(gh + k * K6 + col) = *reinterpret_cast<const uint4*>(ih + src);
    *reinterpret_cast<uint4*>(gl + k * K6 + col) = *reinterpret_cast<const uint4*>(il + src);
  }
}

// F.normalize of conv 6's output (folded BatchNorm included) -> descriptors; rows past the count are zero
__global__ void __launch_bounds__(DESC) dhn_finish_kernel(const float* __restrict__ g, const int* __restrict__ count, long cap,
                                                          float* __restrict__ desc) {
  __shared__ float red[DESC / 32];
  const long j = blockIdx.x;
  const int c = threadIdx.x;
  if (j >= n_valid(count, cap)) {
    desc[j * DESC + c] = 0.f;
    return;
  }
  const float v = g[j * DESC + c];
  float ss = v * v;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  if ((c & 31) == 0) red[c >> 5] = ss;
  __syncthreads();
  desc[j * DESC + c] = v / fmaxf(sqrtf(red[0] + red[1] + red[2] + red[3]), 1e-12f);
}

}  // namespace

struct DhnHandle {
  DhnConfig cfg;
  SiftConfig sift;
  TcConvWeights* cw;  // region l = conv l, BatchNorm folded: conv 0 [32, 9] (CUDA cores); convs 1..6 [256, K]
};

namespace {

size_t ws_bytes(const DhnHandle* h, int H, int W) {
  DhnWs w;
  return carve(nullptr, geometry(h->cfg.max_num_keypoints), sift_detect_workspace_bytes(h->sift, H, W), H, W, &w);
}

// HardNet descriptors of the first count[0] keypoints of one image (crop ih x iw of image [C, H, W]) -> desc [out_rows, 128]
int run_hardnet(DhnHandle* h, const Geo& g, const DhnWs& w, const float* image, int C, int H, int W, int ih, int iw, long ncap,
                const float* kpts, const float* scales, const float* oris, const int* count, float* desc, long out_rows,
                cudaStream_t s) {
  const PyrTab t = pyr_tab(ih, iw);
  dhn_gray_kernel<<<(unsigned)(((long)ih * iw + 255) / 256), 256, 0, s>>>(image, C, H, W, ih, iw, w.pyr);
  LG_CHECK_LAUNCH();
  for (int l = 1; l < t.n; ++l) {
    const long n = (long)t.h[l] * t.w[l];
    dhn_pyrdown_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.pyr + t.off[l - 1], t.h[l - 1], t.w[l - 1], w.pyr + t.off[l],
                                                                   t.h[l], t.w[l]);
    LG_CHECK_LAUNCH();
  }
  const int nchunk = (int)((ncap + NP - 1) / NP);
  dhn_state_kernel<<<1, 1, 0, s>>>(count, ncap, nchunk, g.A.Lp, g.B.Lp, g.C.Lp, g.D.Lp, w.state);
  LG_CHECK_LAUNCH();
  TcConvWeights& cw = *h->cw;
  for (int c = 0; c < nchunk; ++c) {
    const int k0 = c * NP;
    const int* sw = w.state + c * 12;  // levels A, B, C of this chunk
    dhn_patch_kernel<<<NP, 256, 0, s>>>(w.pyr, t, kpts, scales, oris, count, ncap, k0, cw.wpk + cw.w_off[0], cw.wpk + cw.b_off[0],
                                        w.uh, w.ul);
    LG_CHECK_LAUNCH();
    LG_RC(tc_conv(cw, tc_rows_state(g.A, sw), {.in_h = w.uh, .in_l = w.ul, .cin = 64, .taps = 9, .region = 1, .relu = 1, .B = NP,
                  .H = PS, .W = PS, .out_h = w.vh, .out_l = w.vl, .cout = 64}, s));
    const long nb = 4L * NP * RB * 8;
    dhn_phase_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, s>>>(w.vh, w.vl, 34, 18, count, ncap, k0, g.B.rows, w.uh, w.ul);
    LG_CHECK_LAUNCH();
    LG_RC(tc_conv(cw, tc_rows_state(g.B, sw + 4), {.in_h = w.uh, .in_l = w.ul, .cin = 64, .taps = 9, .pstride = (int)g.B.rows,
                  .region = 2, .relu = 1, .B = NP, .H = 16, .W = 16, .out_h = w.bh, .out_l = w.bl, .cout = 64}, s));
    LG_RC(tc_conv(cw, tc_rows_state(g.B, sw + 4), {.in_h = w.bh, .in_l = w.bl, .cin = 64, .taps = 9, .region = 3, .relu = 1,
                  .B = NP, .H = 16, .W = 16, .out_h = w.b2h, .out_l = w.b2l, .cout = 64}, s));
    const long nc = 4L * NP * RC * 8;
    dhn_phase_kernel<<<(unsigned)((nc + 255) / 256), 256, 0, s>>>(w.b2h, w.b2l, 18, 10, count, ncap, k0, g.C.rows, w.vh, w.vl);
    LG_CHECK_LAUNCH();
    LG_RC(tc_conv(cw, tc_rows_state(g.C, sw + 8), {.in_h = w.vh, .in_l = w.vl, .cin = 64, .taps = 9, .pstride = (int)g.C.rows,
                  .region = 4, .relu = 1, .B = NP, .H = 8, .W = 8, .out_h = w.ch, .out_l = w.cl, .cout = 128}, s));
    LG_RC(tc_conv(cw, tc_rows_state(g.C, sw + 8), {.in_h = w.ch, .in_l = w.cl, .cin = 128, .taps = 9, .region = 5, .relu = 1,
                  .B = NP, .H = 8, .W = 8, .out_h = w.c2h, .out_l = w.c2l, .cout = 128}, s));
    dhn_gather_kernel<<<NP, 256, 0, s>>>(w.c2h, w.c2l, count, ncap, k0, w.gh, w.gl);
    LG_CHECK_LAUNCH();
  }
  LG_RC(tc_conv(cw, tc_rows_state(g.D, w.state + nchunk * 12),
                {.in_h = w.gh, .in_l = w.gl, .cin = K6, .taps = 1, .region = 6, .cout = DESC, .out_f32 = w.dout, .ldo = DESC}, s));
  if (out_rows > 0) {
    dhn_finish_kernel<<<(unsigned)out_rows, DESC, 0, s>>>(w.dout, count, ncap, desc);
    LG_CHECK_LAUNCH();
  }
  return 0;
}

int check_args(const DhnHandle* h, const float* image, int channels, const int32_t* image_size, int B, int H, int W,
               const char* null_msg) {
  if (!h || !image) return lg_set_error(null_msg);
  if (B <= 0 || H <= 0 || W <= 0) return lg_set_error("doghardnet: empty batch or image");
  if (channels != 1 && channels != 3) return lg_set_error("doghardnet: channels must be 1 or 3");
  for (int b = 0; image_size && b < B; ++b)
    if (image_size[2 * b] < 1 || image_size[2 * b] > W || image_size[2 * b + 1] < 1 || image_size[2 * b + 1] > H)
      return lg_set_error("doghardnet: image_size outside the image");
  return 0;
}

}  // namespace

extern "C" size_t dhn_weight_blob_floats(void) { return layer_blob_off(NL); }

extern "C" int dhn_create(const DhnConfig* cfg, const float* weights_dev, size_t n_floats, void* stream_, DhnHandle** out) {
  if (!cfg || !weights_dev || !out) return lg_set_error("dhn_create: null argument");
  if (cfg->abi_version != DHN_ABI_VERSION) return lg_set_error("dhn_create: ABI version mismatch");
  if (n_floats != dhn_weight_blob_floats()) return lg_set_error("dhn_create: weight blob has the wrong size");
  if (cfg->num_octave_layers < 1 || cfg->num_octave_layers > 8)
    return lg_set_error("dhn_create: num_octaves (OpenCV's nOctaveLayers) must be in [1, 8]");
  if (cfg->max_num_keypoints <= 0) return lg_set_error("dhn_create: max_num_keypoints must be positive");
  if (cfg->nms_radius < -1) return lg_set_error("dhn_create: nms_radius must be >= 0, or -1 for None");
  cudaStream_t stream = (cudaStream_t)stream_;
  DhnHandle* h = new (std::nothrow) DhnHandle{};
  if (!h) return lg_set_error("dhn_create: out of host memory");
  h->cfg = *cfg;
  h->sift = SiftConfig{SIFT_ABI_VERSION, cfg->num_octave_layers, cfg->nms_radius, cfg->max_num_keypoints, 0, 0,
                       cfg->detection_threshold, cfg->edge_threshold};
  struct Guard {
    DhnHandle* h;
    ~Guard() { if (h) dhn_destroy(h); }
  } guard{h};
  TcConvRegion reg[NL];
  for (int l = 0; l < NL; ++l) {
    const HLayer& L = HL[l];
    const int taps = L.k * L.k, cp = l == 0 ? 1 : (l == NL - 1 ? L.cin : (L.cin + 63) / 64 * 64);
    const float* w = weights_dev + layer_blob_off(l);
    const float* mean = w + (size_t)L.cout * L.cin * taps;
    reg[l] = {.w = w, .bn_mean = mean, .bn_var = mean + L.cout, .cin = L.cin, .cpad = cp, .taps = taps, .rows = l == 0 ? 32 : 256,
              .K = taps * cp, .ncopy = L.cout};
  }
  LG_RC(tc_conv_weights_create(&h->cw, reg, NL, stream));
  guard.h = nullptr;
  *out = h;
  return 0;
}

extern "C" int dhn_destroy(DhnHandle* h) {
  if (!h) return 0;
  tc_conv_weights_destroy(h->cw);
  delete h;
  return 0;
}

extern "C" int64_t dhn_max_keypoints(const DhnHandle* h, int32_t, int32_t) { return h ? h->cfg.max_num_keypoints : 0; }

extern "C" size_t dhn_workspace_bytes(const DhnHandle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  return ws_bytes(h, H, W);
}

extern "C" int64_t dhn_workspace_layout(const DhnHandle* h, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes) {
  if (!h || H <= 0 || W <= 0) return 0;
  DhnWs w;
  char* const base = reinterpret_cast<char*>(kLayoutBase);
  const size_t total = carve(base, geometry(h->cfg.max_num_keypoints), sift_detect_workspace_bytes(h->sift, H, W), H, W, &w);
  const void* p[DHN_LAYOUT_BUFFERS] = {w.uh, w.ul, w.vh,  w.vl,  w.bh, w.bl, w.b2h, w.b2l,
                                       w.ch, w.cl, w.c2h, w.c2l, w.gh, w.gl, w.dout, w.state};
  for (int i = 0; i < DHN_LAYOUT_BUFFERS; ++i) {
    if (offsets) offsets[i] = (int64_t)((const char*)p[i] - base);
    if (bytes) bytes[i] = (int64_t)w.bytes[i];
  }
  return (int64_t)total;
}

extern "C" int dhn_forward(DhnHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B, int32_t H,
                           int32_t W, int64_t cap, float* keypoints, float* scales, float* oris, float* scores,
                           float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!keypoints || !scales || !oris || !scores || !descriptors || !counts) return lg_set_error("dhn_forward: null argument");
  LG_RC(check_args(h, image, channels, image_size, B, H, W, "dhn_forward: null argument"));
  if (cap < h->cfg.max_num_keypoints) return lg_set_error("dhn_forward: output capacity below dhn_max_keypoints()");
  if (!workspace || workspace_bytes < ws_bytes(h, H, W)) return lg_set_error("dhn_forward: workspace too small");
  const Geo g = geometry(h->cfg.max_num_keypoints);
  DhnWs w;
  carve((char*)workspace, g, sift_detect_workspace_bytes(h->sift, H, W), H, W, &w);
  cudaStream_t s = (cudaStream_t)stream_;
  for (int b = 0; b < B; ++b) {
    const int iw = image_size ? image_size[2 * b] : W, ih = image_size ? image_size[2 * b + 1] : H;
    const float* img = image + (long)b * channels * H * W;
    float* kp = keypoints + b * cap * 2;
    LG_RC(sift_detect_image(h->sift, img, channels, H, W, ih, iw, w.sift, cap, kp, scales + b * cap, oris + b * cap,
                            scores + b * cap, counts + b, s));
    LG_RC(run_hardnet(h, g, w, img, channels, H, W, ih, iw, g.cap, kp, scales + b * cap, oris + b * cap, counts + b,
                      descriptors + b * cap * DESC, cap, s));
  }
  return 0;
}

extern "C" int dhn_describe(DhnHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B, int32_t H,
                            int32_t W, int64_t cap, const float* keypoints, const float* scales, const float* oris,
                            const int32_t* counts, float* descriptors, void* workspace, size_t workspace_bytes, void* stream_) {
  if (cap > 0 && (!keypoints || !scales || !oris || !counts || !descriptors)) return lg_set_error("dhn_describe: null argument");
  LG_RC(check_args(h, image, channels, image_size, B, H, W, "dhn_describe: null argument"));
  if (cap < 0 || cap > h->cfg.max_num_keypoints) return lg_set_error("dhn_describe: cap must be in [0, dhn_max_keypoints()]");
  if (cap == 0) return 0;
  if (!workspace || workspace_bytes < ws_bytes(h, H, W)) return lg_set_error("dhn_describe: workspace too small");
  const Geo g = geometry(h->cfg.max_num_keypoints);
  DhnWs w;
  carve((char*)workspace, g, sift_detect_workspace_bytes(h->sift, H, W), H, W, &w);
  cudaStream_t s = (cudaStream_t)stream_;
  for (int b = 0; b < B; ++b) {
    const int iw = image_size ? image_size[2 * b] : W, ih = image_size ? image_size[2 * b + 1] : H;
    LG_RC(run_hardnet(h, g, w, image + (long)b * channels * H * W, channels, H, W, ih, iw, cap, keypoints + b * cap * 2,
                      scales + b * cap, oris + b * cap, counts + b, descriptors + b * cap * DESC, cap, s));
  }
  return 0;
}
