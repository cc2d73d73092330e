// ALIKED extractor forward (include/aliked_b200.h; reference lightglue/aliked.py), fp32 on CUDA cores.
//
// Stages, all on the given stream:
//   pad      replicate-pad the RGB image to a multiple of 32 (InputPadder)
//   encoder  block1 (two 3x3 conv + folded BN + SELU), 2x2 average pool, block2 (ResBlock), 4x4 pool, block3 / block4
//            (ResBlocks of deformable 3x3 convolutions: offset conv + bias, clamp to +-max(h, w) / 4, bilinear taps with
//            torchvision's zero-outside rule)
//   head     the 128-channel (dim) aggregated feature x1234 is never stored: at a full-resolution pixel it is
//            [SELU(conv1 x1), up2(SELU(conv2 x2)), up8(SELU(conv3 x3)), up32(SELU(conv4 x4))] with the three low-resolution
//            maps kept and the first quarter recomputed from x1 (c1 values).  One kernel evaluates it at every padded pixel
//            for the score head's 1x1 layer and the inverse L2 norm; SDDH evaluates it again at its sparse samples.
//   score    three 3x3 convolutions without bias (SELU, SELU, sigmoid) on the padded frame, then the crop
//   DKD      simple_nms and candidate compaction / top-k with SuperPoint's functors and kernels (sp_pipeline.h, sp_tc.cu),
//            borders, threshold / mean fallback, zero-score filler in top-k mode, 5x5 soft-argmax, score sampling
//   SDDH     one block per keypoint: 3x3 patch, offset MLP, M bilinear samples, sf_conv + SELU, agg_weights, L2 norm
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/aliked_b200.h"
#include "lg_internal.h"
#include "sp_pipeline.h"
#include "sp_tc.h"

namespace {

constexpr int AL_N_LIMIT_MAX = 20000;  // ALIKED.n_limit_max
constexpr int AL_MAXDIM = 128;
constexpr int AL_MAXM = 32;
constexpr float AL_SELU_ALPHA = 1.6732632423543772848170429916717f;
constexpr float AL_SELU_SCALE = 1.0507009873554804934193349852946f;

__device__ __forceinline__ float selu(float x) { return x > 0.f ? AL_SELU_SCALE * x : AL_SELU_SCALE * AL_SELU_ALPHA * expm1f(x); }

enum { ACT_NONE = 0, ACT_SELU = 1, ACT_SIGMOID = 2, ACT_CLAMP = 3 };
__device__ __forceinline__ float act(float v, int a, float lim) {
  switch (a) {
    case ACT_SELU: return selu(v);
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case ACT_CLAMP: return fminf(fmaxf(v, -lim), lim);
    default: return v;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// weight layout: the blob's tensors (state_dict order, see the header) and the folded copies of the BN convolutions
// ---------------------------------------------------------------------------------------------------------------------
enum {
  // per block b (0..3) the tensors are addressed through BlockIdx below
  T_CONV1 = 0, T_CONV2, T_CONV3, T_CONV4, T_SH0, T_SH2, T_SH4, T_SH6, T_AGG, T_SOC0W, T_SOC0B, T_SOC2W, T_SOC2B, T_SFW, T_HEAD_N
};
struct BlockIdx {
  size_t off1w, off1b, w1, bn1, off2w, off2b, w2, bn2, dsw, dsb;  // float offsets into the blob (bn*: 4 x c tensors)
  int cin, cout, dcn, res;
};
struct Layout {
  BlockIdx blk[4];
  size_t head[T_HEAD_N];
  size_t total;
  // folded BN convolutions: weight and bias of (block, conv) at fold_w[2 * blk + conv], fold_b[...], float offsets into `fold`
  size_t fold_w[8], fold_b[8], fold_total;
};

bool valid(const AlConfig& c) {
  return c.c1 > 0 && c.c2 > 0 && c.c3 > 0 && c.c4 > 0 && c.dim == c.c4 && c.dim % 4 == 0 && c.dim <= AL_MAXDIM && c.K == 3 &&
         c.M > 0 && c.M <= AL_MAXM && c.nms_radius >= 0;
}

Layout make_layout(const AlConfig& c) {
  Layout L{};
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += n; return r; };
  const int cin[4] = {3, c.c1, c.c2, c.c3}, cout[4] = {c.c1, c.c2, c.c3, c.c4};
  for (int b = 0; b < 4; ++b) {
    BlockIdx& k = L.blk[b];
    k.cin = cin[b]; k.cout = cout[b]; k.dcn = b >= 2; k.res = b >= 1;
    for (int cv = 0; cv < 2; ++cv) {
      const int ci = cv == 0 ? k.cin : k.cout;
      size_t ow = 0, ob = 0, w, bn;
      if (k.dcn) { ow = take((size_t)18 * ci * 9); ob = take(18); }
      w = take((size_t)k.cout * ci * 9);
      bn = take((size_t)4 * k.cout);
      if (cv == 0) { k.off1w = ow; k.off1b = ob; k.w1 = w; k.bn1 = bn; } else { k.off2w = ow; k.off2b = ob; k.w2 = w; k.bn2 = bn; }
    }
    if (k.res) { k.dsw = take((size_t)k.cout * k.cin); k.dsb = take(k.cout); }
  }
  const int q = c.dim / 4;
  L.head[T_CONV1] = take((size_t)q * c.c1);
  L.head[T_CONV2] = take((size_t)q * c.c2);
  L.head[T_CONV3] = take((size_t)q * c.c3);
  L.head[T_CONV4] = take((size_t)q * c.dim);
  L.head[T_SH0] = take((size_t)8 * c.dim);
  L.head[T_SH2] = take(4 * 8 * 9);
  L.head[T_SH4] = take(4 * 4 * 9);
  L.head[T_SH6] = take(1 * 4 * 9);
  L.head[T_AGG] = take((size_t)c.M * c.dim * c.dim);
  L.head[T_SOC0W] = take((size_t)2 * c.M * c.dim * c.K * c.K);
  L.head[T_SOC0B] = take((size_t)2 * c.M);
  L.head[T_SOC2W] = take((size_t)4 * c.M * c.M);
  L.head[T_SOC2B] = take((size_t)2 * c.M);
  L.head[T_SFW] = take((size_t)c.dim * c.dim);
  L.total = o;
  size_t f = 0;
  for (int b = 0; b < 4; ++b)
    for (int cv = 0; cv < 2; ++cv) {
      const int ci = cv == 0 ? L.blk[b].cin : L.blk[b].cout, co = L.blk[b].cout;
      L.fold_w[2 * b + cv] = f; f += (size_t)co * ci * 9;
      L.fold_b[2 * b + cv] = f; f += co;
    }
  L.fold_total = f;
  return L;
}

// W' = W * gamma / sqrt(var + eps), b' = beta - mean * gamma / sqrt(var + eps), in double (eps = 1e-5, nn.BatchNorm2d)
__global__ void al_fold_bn_kernel(const float* __restrict__ w, const float* __restrict__ bn, float* __restrict__ wo,
                                  float* __restrict__ bo, int cout, int per) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)cout * per) return;
  const int co = (int)(i / per);
  const double s = (double)bn[co] / sqrt((double)bn[3 * cout + co] + 1e-5);
  wo[i] = (float)((double)w[i] * s);
  if (i % per == 0) bo[co] = (float)((double)bn[cout + co] - (double)bn[2 * cout + co] * s);
}

// ---------------------------------------------------------------------------------------------------------------------
// encoder kernels
// ---------------------------------------------------------------------------------------------------------------------
__global__ void al_pad_kernel(const float* __restrict__ img, float* __restrict__ out, int BC, int H, int W, int Hp, int Wp,
                              int top, int left) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)BC * Hp * Wp) return;
  const int x = (int)(i % Wp);
  const long r = i / Wp;
  const int y = (int)(r % Hp);
  const long bc = r / Hp;
  const int sy = min(max(y - top, 0), H - 1), sx = min(max(x - left, 0), W - 1);
  out[i] = img[(bc * H + sy) * W + sx];
}

#define AL_CO_T 8
#define AL_PX_T 4
// k x k convolution (k = 1 or 3, stride 1, zero padding k / 2) [+ bias] [+ residual] then activation; 8 output channels x
// 4 consecutive pixels per thread
__global__ void __launch_bounds__(256) al_conv_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                      const float* __restrict__ bias, const float* __restrict__ res,
                                                      float* __restrict__ out, int B, int Cin, int Cout, int H, int W, int k,
                                                      int a, float lim) {
  const int wt = (W + AL_PX_T - 1) / AL_PX_T, cg = (Cout + AL_CO_T - 1) / AL_CO_T;
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * cg * H * wt) return;
  const int xt = (int)(i % wt);
  long r = i / wt;
  const int y = (int)(r % H);
  r /= H;
  const int g = (int)(r % cg), b = (int)(r / cg);
  const int x0 = xt * AL_PX_T, co0 = g * AL_CO_T, pad = k / 2;
  float acc[AL_CO_T][AL_PX_T];
#pragma unroll
  for (int c = 0; c < AL_CO_T; ++c)
#pragma unroll
    for (int p = 0; p < AL_PX_T; ++p) acc[c][p] = (bias && co0 + c < Cout) ? bias[co0 + c] : 0.f;
  const float* inb = in + (long)b * Cin * H * W;
  for (int ci = 0; ci < Cin; ++ci) {
    const float* plane = inb + (long)ci * H * W;
    for (int ky = 0; ky < k; ++ky) {
      const int yy = y + ky - pad;
      if (yy < 0 || yy >= H) continue;
      float v[AL_PX_T + 2];
#pragma unroll
      for (int t = 0; t < AL_PX_T + 2; ++t) {
        const int xx = x0 + t - pad;
        v[t] = (t < AL_PX_T + k - 1 && xx >= 0 && xx < W) ? __ldg(plane + (long)yy * W + xx) : 0.f;
      }
#pragma unroll
      for (int c = 0; c < AL_CO_T; ++c) {
        if (co0 + c >= Cout) break;
        const float* wr = w + (((long)(co0 + c) * Cin + ci) * k + ky) * k;
        for (int kx = 0; kx < k; ++kx) {
          const float wv = __ldg(wr + kx);
#pragma unroll
          for (int p = 0; p < AL_PX_T; ++p) acc[c][p] = fmaf(v[p + kx], wv, acc[c][p]);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < AL_CO_T; ++c) {
    if (co0 + c >= Cout) break;
#pragma unroll
    for (int p = 0; p < AL_PX_T; ++p) {
      if (x0 + p >= W) break;
      const long o = (((long)b * Cout + co0 + c) * H + y) * W + x0 + p;
      out[o] = act(acc[c][p] + (res ? res[o] : 0.f), a, lim);
    }
  }
}

// torchvision deform_conv2d's bilinear tap: 0 when (py, px) lies at or beyond one pixel outside the map, corners outside
// contribute 0
struct Tap { int i00, i01, i10, i11; float w00, w01, w10, w11; };
__device__ __forceinline__ Tap make_tap(float py, float px, int H, int W) {
  Tap t{-1, -1, -1, -1, 0.f, 0.f, 0.f, 0.f};
  if (py <= -1.f || py >= (float)H || px <= -1.f || px >= (float)W) return t;
  const int y0 = (int)floorf(py), x0 = (int)floorf(px), y1 = y0 + 1, x1 = x0 + 1;
  const float ly = py - (float)y0, lx = px - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
  t.w00 = hy * hx; t.w01 = hy * lx; t.w10 = ly * hx; t.w11 = ly * lx;
  if (y0 >= 0 && x0 >= 0) t.i00 = y0 * W + x0;
  if (y0 >= 0 && x1 <= W - 1) t.i01 = y0 * W + x1;
  if (y1 <= H - 1 && x0 >= 0) t.i10 = y1 * W + x0;
  if (y1 <= H - 1 && x1 <= W - 1) t.i11 = y1 * W + x1;
  return t;
}
__device__ __forceinline__ float tap_val(const float* __restrict__ plane, const Tap& t) {
  float v = 0.f;
  if (t.i00 >= 0) v += t.w00 * __ldg(plane + t.i00);
  if (t.i01 >= 0) v += t.w01 * __ldg(plane + t.i01);
  if (t.i10 >= 0) v += t.w10 * __ldg(plane + t.i10);
  if (t.i11 >= 0) v += t.w11 * __ldg(plane + t.i11);
  return v;
}

// deformable 3x3 convolution (stride 1, padding 1) + folded-BN bias [+ residual] then activation; offsets [B, 18, H, W]
// with (dy, dx) of tap t = 3 i + j in channels (2 t, 2 t + 1); one pixel x 8 output channels per thread
__global__ void __launch_bounds__(128) al_deform_kernel(const float* __restrict__ in, const float* __restrict__ off,
                                                        const float* __restrict__ w, const float* __restrict__ bias,
                                                        const float* __restrict__ res, float* __restrict__ out, int B, int Cin,
                                                        int Cout, int H, int W, int a) {
  const int cg = (Cout + AL_CO_T - 1) / AL_CO_T;
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const long HW = (long)H * W;
  if (i >= (long)B * cg * HW) return;
  const long p = i % HW;
  const int g = (int)((i / HW) % cg), b = (int)(i / HW / cg);
  const int y = (int)(p / W), x = (int)(p % W), co0 = g * AL_CO_T;
  float acc[AL_CO_T];
#pragma unroll
  for (int c = 0; c < AL_CO_T; ++c) acc[c] = co0 + c < Cout ? bias[co0 + c] : 0.f;
  const float* ob = off + (long)b * 18 * HW + p;
  const float* inb = in + (long)b * Cin * HW;
  for (int t = 0; t < 9; ++t) {
    const float py = (float)(y - 1 + t / 3) + ob[(2 * t) * HW], px = (float)(x - 1 + t % 3) + ob[(2 * t + 1) * HW];
    const Tap tp = make_tap(py, px, H, W);
    for (int ci = 0; ci < Cin; ++ci) {
      const float v = tap_val(inb + ci * HW, tp);
#pragma unroll
      for (int c = 0; c < AL_CO_T; ++c)
        if (co0 + c < Cout) acc[c] = fmaf(__ldg(w + ((long)(co0 + c) * Cin + ci) * 9 + t), v, acc[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < AL_CO_T; ++c) {
    if (co0 + c >= Cout) break;
    const long o = ((long)b * Cout + co0 + c) * HW + p;
    out[o] = act(acc[c] + (res ? res[o] : 0.f), a, 0.f);
  }
}

__global__ void al_avgpool_kernel(const float* __restrict__ in, float* __restrict__ out, long BC, int H, int W, int k) {
  const int Ho = H / k, Wo = W / k;
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= BC * Ho * Wo) return;
  const int x = (int)(i % Wo);
  const long r = i / Wo;
  const int y = (int)(r % Ho);
  const float* p = in + (r / Ho) * H * W + (long)(y * k) * W + x * k;
  float s = 0.f;
  for (int dy = 0; dy < k; ++dy)
    for (int dx = 0; dx < k; ++dx) s += p[(long)dy * W + dx];
  out[i] = s / (float)(k * k);
}

// ---------------------------------------------------------------------------------------------------------------------
// the aggregated feature x1234 at a padded-frame pixel
// ---------------------------------------------------------------------------------------------------------------------
struct Feat {
  const float* x1;                  // [B, c1, Hp, Wp]
  const float* a2, *a3, *a4;        // SELU(conv2 x2) [B, q, Hp/2, Wp/2], ... /8, /32
  const float* w1;                  // conv1.weight [q, c1]
  int c1, q, Hp, Wp;
};
// bilinear, align_corners=True, scale s: the source row / column of an output index (upsample_bilinear2d's arithmetic)
__device__ __forceinline__ void src_idx(int dst, int in, float scale, int& i0, int& i1, float& l0, float& l1) {
  const float s = scale * (float)dst;
  i0 = (int)s;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = s - (float)i0;
  l0 = 1.f - l1;
}
__device__ __forceinline__ float up_val(const float* __restrict__ plane, int h, int w, int y, int x, int Hp, int Wp) {
  const float sy = h > 1 ? (float)(h - 1) / (float)(Hp - 1) : 0.f, sx = w > 1 ? (float)(w - 1) / (float)(Wp - 1) : 0.f;
  int y0, y1, x0, x1;
  float ly0, ly1, lx0, lx1;
  src_idx(y, h, sy, y0, y1, ly0, ly1);
  src_idx(x, w, sx, x0, x1, lx0, lx1);
  return ly0 * (lx0 * __ldg(plane + y0 * w + x0) + lx1 * __ldg(plane + y0 * w + x1)) +
         ly1 * (lx0 * __ldg(plane + y1 * w + x0) + lx1 * __ldg(plane + y1 * w + x1));
}
// channel c of x1234 at padded pixel (y, x) of image b
__device__ __forceinline__ float feat_at(const Feat& f, int b, int y, int x, int c) {
  const long P = (long)f.Hp * f.Wp;
  const int part = c / f.q, cc = c % f.q;
  if (part == 0) {
    const float* xp = f.x1 + (long)b * f.c1 * P + (long)y * f.Wp + x;
    float s = 0.f;
    for (int k = 0; k < f.c1; ++k) s = fmaf(__ldg(f.w1 + cc * f.c1 + k), __ldg(xp + k * P), s);
    return selu(s);
  }
  const int d = part == 1 ? 2 : (part == 2 ? 8 : 32);
  const int h = f.Hp / d, w = f.Wp / d;
  const float* a = part == 1 ? f.a2 : (part == 2 ? f.a3 : f.a4);
  return up_val(a + ((long)b * f.q + cc) * h * w, h, w, y, x, f.Hp, f.Wp);
}

// every padded pixel: score_head.0 (1x1, dim -> 8) + SELU, and 1 / max(|x1234|, 1e-12) (F.normalize)
__global__ void __launch_bounds__(128) al_head_kernel(Feat f, const float* __restrict__ wh0, float* __restrict__ s1,
                                                      float* __restrict__ invn, int B) {
  const long P = (long)f.Hp * f.Wp;
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * P) return;
  const int b = (int)(i / P);
  const long p = i % P;
  const int y = (int)(p / f.Wp), x = (int)(p % f.Wp);
  const int dim = 4 * f.q;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float ss = 0.f;
  for (int c = 0; c < dim; ++c) {
    const float v = feat_at(f, b, y, x, c);
    ss = fmaf(v, v, ss);
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = fmaf(__ldg(wh0 + o * dim + c), v, acc[o]);
  }
#pragma unroll
  for (int o = 0; o < 8; ++o) s1[((long)b * 8 + o) * P + p] = selu(acc[o]);
  invn[i] = 1.f / fmaxf(sqrtf(ss), 1e-12f);
}

__global__ void al_crop_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int Hp, int Wp, int top,
                               int left) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * H * W) return;
  const int x = (int)(i % W);
  const long r = i / W;
  const int y = (int)(r % H), b = (int)(r / H);
  out[i] = in[((long)b * Hp + y + top) * Wp + x + left];
}

// ---------------------------------------------------------------------------------------------------------------------
// DKD
// ---------------------------------------------------------------------------------------------------------------------
// nms_scores := 0 on the borders: the first r rows / columns, and the last r (or, with image_size, rows >= h_i - r and
// columns >= w_i - r, with Python's slice rule for a negative start)
__global__ void al_borders_kernel(float* __restrict__ s, const float* __restrict__ image_size, int B, int H, int W, int r) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H), b = (int)(i / ((long)H * W));
  int ys, xs;
  if (image_size) {
    ys = (int)(long long)image_size[2 * b + 1] - r;
    xs = (int)(long long)image_size[2 * b] - r;
    if (ys < 0) ys = max(ys + H, 0);
    if (xs < 0) xs = max(xs + W, 0);
  } else {  // t[-r:]; t[-0:] is the whole axis
    ys = r > 0 ? max(H - r, 0) : 0;
    xs = r > 0 ? max(W - r, 0) : 0;
  }
  if (y < r || x < r || y >= ys || x >= xs) s[i] = 0.f;
}

// threshold mode: per image the count of NMS scores above `thr` and the mean of the score map (one block per image)
__global__ void __launch_bounds__(512) al_stats_kernel(const float* __restrict__ nms, const float* __restrict__ score,
                                                        int* __restrict__ cnt, float* __restrict__ mean, long HW, float thr) {
  __shared__ int sc[16];
  __shared__ double sd[16];
  const int b = blockIdx.x, tid = threadIdx.x;
  int c = 0;
  double s = 0.0;
  for (long j = tid; j < HW; j += 512) {
    c += nms[b * HW + j] > thr ? 1 : 0;
    s += (double)score[b * HW + j];
  }
  for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, o); s += __shfl_xor_sync(0xffffffffu, s, o); }
  if ((tid & 31) == 0) { sc[tid >> 5] = c; sd[tid >> 5] = s; }
  __syncthreads();
  if (tid == 0) {
    int ct = 0;
    double st = 0.0;
    for (int w = 0; w < 16; ++w) { ct += sc[w]; st += sd[w]; }
    cnt[b] = ct;
    mean[b] = (float)(st / (double)HW);
  }
}
// nms := nms if nms > thr_b else -1, thr_b = thr, or the image's mean score when thr <= 0 or no pixel of the whole batch
// passes thr (DKD.forward); the compaction then keeps the positive values
__global__ void al_mask_kernel(float* __restrict__ nms, const int* __restrict__ cnt, const float* __restrict__ mean, int B,
                               long HW, float thr) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * HW) return;
  int tot = 0;
  for (int b = 0; b < B; ++b) tot += cnt[b];
  const float t = (thr > 0.f && tot > 0) ? thr : mean[i / HW];
  if (!(nms[i] > t)) nms[i] = -1.f;
}
// top-k mode with fewer than k NMS maxima: fill with zero-score pixels in row-major order (the reference's torch.topk
// picks them in an unspecified order).  One thread per image.
__global__ void al_fill_topk_kernel(const float* __restrict__ nms, int* __restrict__ sel_pos, float* __restrict__ sel_score,
                                    int* __restrict__ n_sel, int B, long HW, int k, long out_cap) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int n = n_sel[b];
  for (long j = 0; j < HW && n < k; ++j)
    if (!(nms[b * HW + j] > 0.f)) { sel_pos[b * out_cap + n] = (int)j; sel_score[b * out_cap + n] = 0.f; ++n; }
  n_sel[b] = n;
}

// bilinear grid_sample, align_corners=True, zeros outside, of a [H, W] plane at normalised (gx, gy)
__device__ __forceinline__ float grid_sample1(const float* __restrict__ p, int H, int W, float gx, float gy) {
  const float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)(W - 1));
  const float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)(H - 1));
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
  const float nw = (fx + 1.f - ix) * (fy + 1.f - iy), ne = (ix - fx) * (fy + 1.f - iy);
  const float sw = (fx + 1.f - ix) * (iy - fy), se = (ix - fx) * (iy - fy);
  float v = 0.f;
  if (y0 >= 0 && y0 < H && x0 >= 0 && x0 < W) v += p[y0 * W + x0] * nw;
  if (y0 >= 0 && y0 < H && x1 >= 0 && x1 < W) v += p[y0 * W + x1] * ne;
  if (y1 >= 0 && y1 < H && x0 >= 0 && x0 < W) v += p[y1 * W + x0] * sw;
  if (y1 >= 0 && y1 < H && x1 >= 0 && x1 < W) v += p[y1 * W + x1] * se;
  return v;
}

// soft-argmax on the (2r+1)^2 window (zero padded), normalised keypoint, sampled score, output keypoint in pixels
__global__ void al_refine_kernel(const float* __restrict__ score, const int* __restrict__ n_sel, const int* __restrict__ sel_pos,
                                 float* __restrict__ kpn, float* __restrict__ kpts, float* __restrict__ kscores, int B, int H,
                                 int W, int r, long out_cap) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= (long)B * out_cap) return;
  const long b = i / out_cap, j = i % out_cap;
  if (j >= n_sel[b]) {
    kpn[2 * i] = kpn[2 * i + 1] = 0.f;
    kpts[2 * i] = kpts[2 * i + 1] = 0.f;
    kscores[i] = 0.f;
    return;
  }
  const float* p = score + b * (long)H * W;
  const int pos = sel_pos[i], xn = pos % W, yn = pos / W;
  float m = -INFINITY;
  for (int dy = -r; dy <= r; ++dy)
    for (int dx = -r; dx <= r; ++dx) {
      const int y = yn + dy, x = xn + dx;
      m = fmaxf(m, (y >= 0 && y < H && x >= 0 && x < W) ? p[y * W + x] : 0.f);
    }
  float se = 0.f, sx = 0.f, sy = 0.f;
  for (int dy = -r; dy <= r; ++dy)
    for (int dx = -r; dx <= r; ++dx) {
      const int y = yn + dy, x = xn + dx;
      const float v = (y >= 0 && y < H && x >= 0 && x < W) ? p[y * W + x] : 0.f;
      const float e = expf((v - m) / 0.1f);
      se += e; sx = fmaf(e, (float)dx, sx); sy = fmaf(e, (float)dy, sy);
    }
  // (xy_nms + residual) / wh * 2 - 1, rounded step by step as the reference's tensor ops: SDDH truncates the result
  const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
  const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)xn, __fdiv_rn(sx, se)), wm1), 2.f), 1.f);
  const float gy = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)yn, __fdiv_rn(sy, se)), hm1), 2.f), 1.f);
  kpn[2 * i] = gx;
  kpn[2 * i + 1] = gy;
  kscores[i] = grid_sample1(p, H, W, gx, gy);
  kpts[2 * i] = __fdiv_rn(__fmul_rn(wm1, __fadd_rn(gx, 1.f)), 2.f);
  kpts[2 * i + 1] = __fdiv_rn(__fmul_rn(hm1, __fadd_rn(gy, 1.f)), 2.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// SDDH: one block of 128 threads per keypoint slot
// ---------------------------------------------------------------------------------------------------------------------
struct Sddh {
  Feat f;
  const float* invn;                           // [B, Hp, Wp]
  const float *oc0w, *oc0b, *oc2w, *oc2b, *sfw, *agg;
  int dim, M, H, W, top, left;                 // cropped extents and crop origin in the padded frame
};
// normalised feature channel c at cropped pixel (y, x)
__device__ __forceinline__ float nfeat(const Sddh& s, int b, int y, int x, int c) {
  const int yp = y + s.top, xp = x + s.left;
  return feat_at(s.f, b, yp, xp, c) * s.invn[((long)b * s.f.Hp + yp) * s.f.Wp + xp];
}

__global__ void __launch_bounds__(128) al_sddh_kernel(Sddh s, const int* __restrict__ n_sel, const float* __restrict__ kpn,
                                                      float* __restrict__ desc, long out_cap) {
  __shared__ float patch[9][AL_MAXDIM];
  __shared__ float hid[2 * AL_MAXM];
  __shared__ float off[2 * AL_MAXM];
  __shared__ float feat[AL_MAXM][AL_MAXDIM];
  __shared__ float sf[AL_MAXM][AL_MAXDIM];
  __shared__ float red[4];
  const long j = blockIdx.x, b = blockIdx.y, i = b * out_cap + j;
  const int t = threadIdx.x, dim = s.dim, M = s.M, H = s.H, W = s.W;
  float* dd = desc + i * dim;
  if (j >= n_sel[b]) {
    if (t < dim) dd[t] = 0.f;
    return;
  }
  const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
  // (kpts / 2 + 0.5) * wh, rounded as the reference's tensor ops
  const float kx = __fmul_rn(__fadd_rn(__fmul_rn(kpn[2 * i], 0.5f), 0.5f), wm1);
  const float ky = __fmul_rn(__fadd_rn(__fmul_rn(kpn[2 * i + 1], 0.5f), 0.5f), hm1);
  // get_patches: corner = long(long(k) - ps / 2 + 1), clamped to [0, w - 1 - ps]
  int cx = (int)((float)(long long)kx - 1.5f + 1.f), cy = (int)((float)(long long)ky - 1.5f + 1.f);
  cx = min(max(cx, 0), W - 1 - 3);
  cy = min(max(cy, 0), H - 1 - 3);
  if (t < dim)
    for (int q = 0; q < 9; ++q) patch[q][t] = nfeat(s, (int)b, cy + q / 3, cx + q % 3, t);
  __syncthreads();
  // offset MLP: 3x3 valid conv (dim -> 2M) + bias, SELU, 1x1 (2M -> 2M) + bias, clamp; one warp per output
  const int warp = t >> 5, lane = t & 31;
  for (int o = warp; o < 2 * M; o += 4) {
    float a = 0.f;
    for (int e = lane; e < dim * 9; e += 32) {
      const int c = e / 9, q = e % 9;
      a = fmaf(__ldg(s.oc0w + (long)o * dim * 9 + e), patch[q][c], a);
    }
    for (int w = 16; w > 0; w >>= 1) a += __shfl_xor_sync(0xffffffffu, a, w);
    if (lane == 0) hid[o] = selu(a + s.oc0b[o]);
  }
  __syncthreads();
  const float lim = (float)max(H, W) / 4.f;
  if (t < 2 * M) {
    float a = s.oc2b[t];
    for (int e = 0; e < 2 * M; ++e) a = fmaf(__ldg(s.oc2w + t * 2 * M + e), hid[e], a);
    off[t] = fminf(fmaxf(a, -lim), lim);
  }
  __syncthreads();
  // M bilinear samples (grid_sample, align_corners=True, zeros) of the normalised map at kpt + offset
  if (t < dim)
    for (int p = 0; p < M; ++p) {
      const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fadd_rn(kx, off[p])), wm1), 1.f);
      const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fadd_rn(ky, off[M + p])), hm1), 1.f);
      const float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), wm1);
      const float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), hm1);
      const float fx = floorf(ix), fy = floorf(iy);
      const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
      const float nw = (fx + 1.f - ix) * (fy + 1.f - iy), ne = (ix - fx) * (fy + 1.f - iy);
      const float sw = (fx + 1.f - ix) * (iy - fy), se = (ix - fx) * (iy - fy);
      float v = 0.f;
      if (y0 >= 0 && y0 < H && x0 >= 0 && x0 < W) v += nfeat(s, (int)b, y0, x0, t) * nw;
      if (y0 >= 0 && y0 < H && x1 >= 0 && x1 < W) v += nfeat(s, (int)b, y0, x1, t) * ne;
      if (y1 >= 0 && y1 < H && x0 >= 0 && x0 < W) v += nfeat(s, (int)b, y1, x0, t) * sw;
      if (y1 >= 0 && y1 < H && x1 >= 0 && x1 < W) v += nfeat(s, (int)b, y1, x1, t) * se;
      feat[p][t] = v;
    }
  __syncthreads();
  // sf_conv (1x1, no bias) + SELU, then desc[d] = sum_{p, c} sf[p][c] agg[p][c][d]
  if (t < dim)
    for (int p = 0; p < M; ++p) {
      float a = 0.f;
      for (int c = 0; c < dim; ++c) a = fmaf(__ldg(s.sfw + t * dim + c), feat[p][c], a);
      sf[p][t] = selu(a);
    }
  __syncthreads();
  float d = 0.f;
  if (t < dim)
    for (int p = 0; p < M; ++p)
      for (int c = 0; c < dim; ++c) d = fmaf(sf[p][c], __ldg(s.agg + ((long)p * dim + c) * dim + t), d);
  float ss = d * d;
  for (int w = 16; w > 0; w >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, w);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  const float tot = red[0] + red[1] + red[2] + red[3];
  if (t < dim) dd[t] = d / fmaxf(sqrtf(tot), 1e-12f);
}

unsigned blocks(long n, int t) { return (unsigned)((n + t - 1) / t); }

struct Geo {
  int Hp, Wp, top, left;
};
Geo geometry(int H, int W) {
  const int ph = (32 - H % 32) % 32, pw = (32 - W % 32) % 32;
  return Geo{H + ph, W + pw, ph / 2, pw / 2};
}

// workspace carve; `base` may be null to size it
struct Ws {
  float *img, *ta, *x1, *s1, *invn;                 // padded full resolution
  float *p1, *t2, *d2, *x2, *a2;                    // 1/2
  float *p2, *o3, *t3, *d3, *x3, *a3;               // 1/8
  float *p3, *o4, *t4, *d4, *x4, *a4;               // 1/32
  float *score, *nms, *n1, *n2, *n3, *kpn, *mean;   // cropped / per keypoint / per image
  int* cnt;
  SpWorkspace sp;                                   // the fields SuperPoint's compaction / selection use
  size_t bytes;
};
void carve(char* base, const AlConfig& c, int B, int H, int W, long cap, Ws* w) {
  WsBump bp{base, 0};
  auto take = [&](size_t n) { return bp.take<float>(n); };
  const Geo g = geometry(H, W);
  const size_t P0 = (size_t)B * g.Hp * g.Wp, P1 = P0 / 4, P2 = P0 / 64, P3 = P0 / 1024, PX = (size_t)B * H * W;
  const int q = c.dim / 4;
  w->img = take(3 * P0);
  w->ta = take((size_t)(c.c1 > 8 ? c.c1 : 8) * P0);
  w->x1 = take((size_t)c.c1 * P0);
  w->s1 = take(8 * P0);
  w->invn = take(P0);
  w->p1 = take(c.c1 * P1); w->t2 = take(c.c2 * P1); w->d2 = take(c.c2 * P1);
  w->x2 = take(c.c2 * P1); w->a2 = take(q * P1);
  w->p2 = take(c.c2 * P2); w->o3 = take(18 * P2); w->t3 = take(c.c3 * P2);
  w->d3 = take(c.c3 * P2); w->x3 = take(c.c3 * P2); w->a3 = take(q * P2);
  w->p3 = take(c.c3 * P3); w->o4 = take(18 * P3); w->t4 = take(c.c4 * P3);
  w->d4 = take(c.c4 * P3); w->x4 = take(c.c4 * P3); w->a4 = take(q * P3);
  w->score = take(PX); w->nms = take(PX);
  w->n1 = take(PX); w->n2 = take(PX); w->n3 = take(PX);
  w->kpn = take((size_t)B * cap * 2);
  w->mean = take(B);
  w->cnt = bp.take<int>(B);
  SpWorkspace& s = w->sp;
  s = SpWorkspace{};
  s.t0 = w->nms;
  s.cand_score = take(PX);
  s.cand_pos = bp.take<int>(PX);
  s.sel_score = take((size_t)B * cap);
  s.sel_pos = bp.take<int>((size_t)B * cap);
  s.row_count = bp.take<int>((size_t)B * H);
  s.row_start = bp.take<int>((size_t)B * H);
  s.n_cand = bp.take<int>(B);
  s.n_sel = bp.take<int>(B);
  w->bytes = bp.bytes();
}

int64_t max_keypoints(const AlConfig& c, int H, int W) {
  const int64_t k = c.max_num_keypoints > 0 ? c.max_num_keypoints : AL_N_LIMIT_MAX;
  return k < (int64_t)H * W ? k : (int64_t)H * W;
}

}  // namespace

struct AlHandle {
  AlConfig cfg;
  Layout L;
  float* wts;   // device copy of the blob
  float* fold;  // folded BN convolutions
};

extern "C" size_t al_weight_blob_floats(const AlConfig* cfg) { return (cfg && valid(*cfg)) ? make_layout(*cfg).total : 0; }

extern "C" int al_create(const AlConfig* cfg, const float* weights_dev, size_t n_floats, void* stream_, AlHandle** out) {
  if (!cfg || !weights_dev || !out) return lg_set_error("al_create: null argument");
  if (cfg->abi_version != AL_ABI_VERSION) return lg_set_error("al_create: ABI version mismatch");
  if (!valid(*cfg)) return lg_set_error("al_create: bad conf (needs dim == c4, dim % 4 == 0, dim <= 128, K == 3, 0 < M <= 32)");
  const Layout L = make_layout(*cfg);
  if (n_floats != L.total) return lg_set_error("al_create: weight blob has the wrong size");
  cudaStream_t stream = (cudaStream_t)stream_;
  AlHandle* h = new AlHandle{*cfg, L, nullptr, nullptr};
  struct Guard {  // every failure path below releases the handle and what it owns
    AlHandle* h;
    ~Guard() { if (h) al_destroy(h); }
  } guard{h};
  LG_CU(cudaMalloc(&h->wts, (L.total + L.fold_total) * sizeof(float)));
  h->fold = h->wts + L.total;
  LG_CU(cudaMemcpyAsync(h->wts, weights_dev, L.total * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  for (int b = 0; b < 4; ++b)
    for (int cv = 0; cv < 2; ++cv) {
      const BlockIdx& k = L.blk[b];
      const int ci = cv == 0 ? k.cin : k.cout, per = ci * 9;
      al_fold_bn_kernel<<<blocks((long)k.cout * per, 256), 256, 0, stream>>>(
          h->wts + (cv == 0 ? k.w1 : k.w2), h->wts + (cv == 0 ? k.bn1 : k.bn2), h->fold + L.fold_w[2 * b + cv],
          h->fold + L.fold_b[2 * b + cv], k.cout, per);
      LG_CHECK_LAUNCH();
    }
  guard.h = nullptr;
  *out = h;
  return 0;
}

extern "C" int al_destroy(AlHandle* h) {
  if (!h) return 0;
  cudaFree(h->wts);
  delete h;
  return 0;
}

extern "C" int64_t al_max_keypoints(const AlHandle* h, int32_t H, int32_t W) { return h ? max_keypoints(h->cfg, H, W) : 0; }

extern "C" size_t al_workspace_bytes(const AlHandle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  Ws w;
  carve(nullptr, h->cfg, B, H, W, max_keypoints(h->cfg, H, W), &w);
  return w.bytes;
}

extern "C" int al_forward(AlHandle* h, const float* image, const float* image_size, int32_t B, int32_t H, int32_t W, int64_t cap,
                          float* keypoints, float* scores, float* descriptors, int32_t* counts, void* workspace,
                          size_t workspace_bytes, void* stream_) {
  if (!h || !image || !keypoints || !scores || !descriptors || !counts) return lg_set_error("al_forward: null argument");
  if (B <= 0 || H < 8 || W < 8) return lg_set_error("al_forward: H and W must be at least 8");
  const AlConfig& c = h->cfg;
  const bool topk = !(c.detection_threshold > 0.f) && c.max_num_keypoints > 0;
  if (topk && (int64_t)c.max_num_keypoints > (int64_t)H * W)
    return lg_set_error("al_forward: max_num_keypoints exceeds the number of pixels (top-k mode)");
  if (cap < max_keypoints(c, H, W)) return lg_set_error("al_forward: output capacity below al_max_keypoints()");
  Ws w;
  carve((char*)workspace, c, B, H, W, cap, &w);
  if (!workspace || workspace_bytes < w.bytes) return lg_set_error("al_forward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream_;
  const Layout& L = h->L;
  const float* wb = h->wts;
  const Geo g = geometry(H, W);
  const int q = c.dim / 4;

  auto conv = [&](const float* in, const float* wt, const float* bias, const float* res, float* out, int Cin, int Cout, int hh,
                  int ww, int k, int a, float lim) {
    const long n = (long)B * ((Cout + AL_CO_T - 1) / AL_CO_T) * hh * ((ww + AL_PX_T - 1) / AL_PX_T);
    al_conv_kernel<<<blocks(n, 256), 256, 0, st>>>(in, wt, bias, res, out, B, Cin, Cout, hh, ww, k, a, lim);
  };
  auto pool = [&](const float* in, float* out, int C, int hh, int ww, int k) {
    al_avgpool_kernel<<<blocks((long)B * C * (hh / k) * (ww / k), 256), 256, 0, st>>>(in, out, (long)B * C, hh, ww, k);
  };
  // ResBlock (block2: plain convolutions; block3 / block4: deformable)
  auto resblock = [&](int bi, const float* x, float* off, float* t, float* d, float* out, int hh, int ww) {
    const BlockIdx& k = L.blk[bi];
    const float *w1 = h->fold + L.fold_w[2 * bi], *b1 = h->fold + L.fold_b[2 * bi];
    const float *w2 = h->fold + L.fold_w[2 * bi + 1], *b2 = h->fold + L.fold_b[2 * bi + 1];
    conv(x, wb + k.dsw, wb + k.dsb, nullptr, d, k.cin, k.cout, hh, ww, 1, ACT_NONE, 0.f);  // downsample (1x1 + bias)
    if (!k.dcn) {
      conv(x, w1, b1, nullptr, t, k.cin, k.cout, hh, ww, 3, ACT_SELU, 0.f);
      conv(t, w2, b2, d, out, k.cout, k.cout, hh, ww, 3, ACT_SELU, 0.f);
      return;
    }
    const float lim = (float)(hh > ww ? hh : ww) / 4.f;
    const long n = (long)B * ((k.cout + AL_CO_T - 1) / AL_CO_T) * hh * ww;
    conv(x, wb + k.off1w, wb + k.off1b, nullptr, off, k.cin, 18, hh, ww, 3, ACT_CLAMP, lim);
    al_deform_kernel<<<blocks(n, 128), 128, 0, st>>>(x, off, w1, b1, nullptr, t, B, k.cin, k.cout, hh, ww, ACT_SELU);
    conv(t, wb + k.off2w, wb + k.off2b, nullptr, off, k.cout, 18, hh, ww, 3, ACT_CLAMP, lim);
    al_deform_kernel<<<blocks(n, 128), 128, 0, st>>>(t, off, w2, b2, d, out, B, k.cout, k.cout, hh, ww, ACT_SELU);
  };

  // ---- extract_dense_map
  al_pad_kernel<<<blocks((long)B * 3 * g.Hp * g.Wp, 256), 256, 0, st>>>(image, w.img, B * 3, H, W, g.Hp, g.Wp, g.top, g.left);
  conv(w.img, h->fold + L.fold_w[0], h->fold + L.fold_b[0], nullptr, w.ta, 3, c.c1, g.Hp, g.Wp, 3, ACT_SELU, 0.f);
  conv(w.ta, h->fold + L.fold_w[1], h->fold + L.fold_b[1], nullptr, w.x1, c.c1, c.c1, g.Hp, g.Wp, 3, ACT_SELU, 0.f);
  const int H1 = g.Hp / 2, W1 = g.Wp / 2, H2 = g.Hp / 8, W2 = g.Wp / 8, H3 = g.Hp / 32, W3 = g.Wp / 32;
  pool(w.x1, w.p1, c.c1, g.Hp, g.Wp, 2);
  resblock(1, w.p1, nullptr, w.t2, w.d2, w.x2, H1, W1);
  pool(w.x2, w.p2, c.c2, H1, W1, 4);
  resblock(2, w.p2, w.o3, w.t3, w.d3, w.x3, H2, W2);
  pool(w.x3, w.p3, c.c3, H2, W2, 4);
  resblock(3, w.p3, w.o4, w.t4, w.d4, w.x4, H3, W3);
  conv(w.x2, wb + L.head[T_CONV2], nullptr, nullptr, w.a2, c.c2, q, H1, W1, 1, ACT_SELU, 0.f);
  conv(w.x3, wb + L.head[T_CONV3], nullptr, nullptr, w.a3, c.c3, q, H2, W2, 1, ACT_SELU, 0.f);
  conv(w.x4, wb + L.head[T_CONV4], nullptr, nullptr, w.a4, c.dim, q, H3, W3, 1, ACT_SELU, 0.f);
  const Feat f{w.x1, w.a2, w.a3, w.a4, wb + L.head[T_CONV1], c.c1, q, g.Hp, g.Wp};
  al_head_kernel<<<blocks((long)B * g.Hp * g.Wp, 128), 128, 0, st>>>(f, wb + L.head[T_SH0], w.s1, w.invn, B);
  float* s2 = w.ta;  // block1's scratch is free again
  float* s3 = w.ta + (size_t)4 * B * g.Hp * g.Wp;
  conv(w.s1, wb + L.head[T_SH2], nullptr, nullptr, s2, 8, 4, g.Hp, g.Wp, 3, ACT_SELU, 0.f);
  conv(s2, wb + L.head[T_SH4], nullptr, nullptr, s3, 4, 4, g.Hp, g.Wp, 3, ACT_SELU, 0.f);
  conv(s3, wb + L.head[T_SH6], nullptr, nullptr, w.img, 4, 1, g.Hp, g.Wp, 3, ACT_SIGMOID, 0.f);
  al_crop_kernel<<<blocks((long)B * H * W, 256), 256, 0, st>>>(w.img, w.score, B, H, W, g.Hp, g.Wp, g.top, g.left);
  LG_CHECK_LAUNCH();

  // ---- DKD: simple_nms with SuperPoint's functors; cand_score is scratch until the compaction
  SpCudaExec ex{st};
  const long n = (long)B * H * W;
  const int r = c.nms_radius;
  LG_RC(sp_simple_nms(ex, w.score, w.nms, B, H, W, r, w.n2, w.n1, w.nms, w.sp.cand_score, w.n3));
  al_borders_kernel<<<blocks(n, 256), 256, 0, st>>>(w.nms, image_size, B, H, W, r);
  const SpCudaStages stages{st};
  const long pcap = (long)H * W;
  if (topk) {
    LG_RC(stages.compact(ex, w.sp, B, H, W, 0.f, pcap));  // the positive NMS maxima
    LG_RC(stages.select(ex, w.sp, B, c.max_num_keypoints, pcap, cap, 1));
    al_fill_topk_kernel<<<blocks(B, 32), 32, 0, st>>>(w.nms, w.sp.sel_pos, w.sp.sel_score, w.sp.n_sel, B, pcap,
                                                      c.max_num_keypoints, cap);
  } else {
    al_stats_kernel<<<B, 512, 0, st>>>(w.nms, w.score, w.cnt, w.mean, pcap, c.detection_threshold);
    al_mask_kernel<<<blocks(n, 256), 256, 0, st>>>(w.nms, w.cnt, w.mean, B, pcap, c.detection_threshold);
    const int n_limit = c.max_num_keypoints > 0 ? c.max_num_keypoints : AL_N_LIMIT_MAX;
    LG_RC(stages.compact(ex, w.sp, B, H, W, 0.f, pcap));
    LG_RC(stages.select(ex, w.sp, B, n_limit, pcap, cap, 0));
  }
  LG_CHECK_LAUNCH();
  al_refine_kernel<<<blocks((long)B * cap, 128), 128, 0, st>>>(w.score, w.sp.n_sel, w.sp.sel_pos, w.kpn, keypoints, scores, B, H,
                                                               W, r, cap);
  // ---- SDDH
  const Sddh sd{f, w.invn, wb + L.head[T_SOC0W], wb + L.head[T_SOC0B], wb + L.head[T_SOC2W], wb + L.head[T_SOC2B],
                wb + L.head[T_SFW], wb + L.head[T_AGG], c.dim, c.M, H, W, g.top, g.left};
  if (cap > 0) al_sddh_kernel<<<dim3((unsigned)cap, B), 128, 0, st>>>(sd, w.sp.n_sel, w.kpn, descriptors, cap);
  LG_CHECK_LAUNCH();
  LG_CU(cudaMemcpyAsync(counts, w.sp.n_sel, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return 0;
}
