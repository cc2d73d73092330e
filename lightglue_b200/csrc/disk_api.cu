// C ABI of the DISK extractor (include/disk_b200.h): kornia's DISK U-Net (lightglue/disk.py -> kornia.feature.DISK),
// NMS, the kthvalue top-k and the descriptor lookup.
//
// Every convolution is kornia's `Conv` block: InstanceNorm2d -> PReLU -> 5x5 Conv2d (padding 2, zero padding applied to
// the PReLU output).  Each layer runs as
//   statistics of its input (per image and channel: fixed-order Welford chunks merged with Chan's formula -- centred,
//   deterministic, no atomics) -> one "prepare" pass (gather: pooled / upsampled + concatenated; normalise; PReLU) that
//   writes the zero-padded NHWC operand (2-pixel border) -> the convolution.
// down1 .. up2 run on the tensor cores (tc_conv, 25 taps, split-bf16 operands, fp32 output without activation); their
// inputs are zero-padded to 64 / 128 channels (DESIGN.md §6).  down0 (K = 75) runs on the CUDA cores with the image's
// instance norm and PReLU fused in.  The last convolution (80 -> 129) is split: its heatmap channel is a dense fp32
// 5x5x80 dot per pixel; its 128 descriptor channels are computed only at the selected keypoints, as one split-bf16 GEMM
// over gathered im2col rows (K = 2000, padded to 2048).
//
// Feature maps: fp32 or bf16, NHWC with a 2-pixel zero border, row = b (H+4)(W+4) + (y+2)(W+4) + (x+2), as tc_conv
// reads them; each level holds the rows of its tc_rows plan (lg_tc.h).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <new>

#include "../../include/disk_b200.h"
#include "lg_internal.h"
#include "lg_tc.h"
#include "sp_tc.h"
#include "ws_bump.h"

namespace {

constexpr int NL = 9;
struct DLayer { int cin, cout, level; };
// down0..down4, up0..up3 (kornia: Unet(in_features=3, size=5, down=[16, 32, 64, 64, 64], up=[64, 64, 64, 129]))
constexpr DLayer DL[NL] = {{3, 16, 0},   {16, 32, 1},  {32, 64, 2},  {64, 64, 3}, {64, 64, 4},
                           {128, 64, 3}, {128, 64, 2}, {96, 64, 1},  {80, 129, 0}};
constexpr int TAPS = 25;
constexpr int DESC = 128, X3C = 80, DK = TAPS * X3C, DKP = 2048;  // descriptor head: K = 2000, padded to 32 blocks of 64
constexpr int MAXC = 128;       // widest layer input
constexpr int HEAT = NL - 1;    // packed region of the heatmap channel
constexpr int STAT_CHUNK = 1024;  // pixels per partial-statistics block

int cpad(int c) { return (c + 63) / 64 * 64; }
size_t layer_blob_off(int l) {  // slope [cin], weight [cout, cin, 5, 5], bias [cout]
  size_t o = 0;
  for (int i = 0; i < l; ++i) o += (size_t)DL[i].cin + (size_t)DL[i].cout * DL[i].cin * TAPS + DL[i].cout;
  return o;
}

struct Geo {
  int B, H, W, Hp, Wp;
  TcRows lv[5];     // level i: Hp >> i by Wp >> i
  long ccap, ocap;  // candidates per image (NMS packing bound), output rows per image
  TcRows ld;        // descriptor GEMM rows (B ocap)
};

long nms_bound(int w, int H, int W) {
  const long s = w / 2 + 1;
  return ((H + s - 1) / s) * ((W + s - 1) / s);
}
long out_cap(const DiskConfig& c, int H, int W) {
  const long nb = nms_bound(c.nms_window_size, H, W);
  return c.max_num_keypoints < 0 ? nb : std::max<long>(1, std::min<long>(c.max_num_keypoints, nb));
}
Geo geometry(const DiskConfig& c, int B, int H, int W) {
  Geo g{};
  g.B = B; g.H = H; g.W = W;
  g.Hp = c.pad_if_not_divisible ? (H + 15) / 16 * 16 : H;
  g.Wp = c.pad_if_not_divisible ? (W + 15) / 16 * 16 : W;
  for (int i = 0; i < 5; ++i) g.lv[i] = tc_rows((long)B * ((g.Hp >> i) + 4) * ((g.Wp >> i) + 4));
  g.ccap = nms_bound(c.nms_window_size, H, W);
  g.ocap = out_cap(c, H, W);
  g.ld = tc_rows((long)B * g.ocap);
  return g;
}

struct DiskWs {
  int* state;  // [6][4]: SeqState words (len[2], stop_layer, -) of the five levels and the descriptor GEMM
  float *part, *mean, *rstd;
  float* raw[NL - 1];  // raw outputs of down0..down4, up0..up2 (fp32, padded NHWC, cout channels)
  __nv_bfloat16 *ah, *al;  // operand of the tensor-core convolutions
  float* x3;               // up3 input (fp32, padded NHWC, 80 channels)
  float *heat, *kept;      // [B, H, W]
  int *row_count, *row_start, *n_cand, *cand_pos;
  float* cand_score;
  int *sel_pos, *n_sel;
  float* sel_score;
  __nv_bfloat16 *dh, *dl;  // im2col rows of the descriptor head
  float* dout;             // [rows, 128]
  size_t bytes[DISK_LAYOUT_BUFFERS];  // sizes of the buffers disk_workspace_layout reports, in its order
};

size_t carve(char* base, const Geo& g, DiskWs* w) {
  WsBump b{base, 0};
  constexpr size_t A = 1024;
  const int B = g.B;
  w->state = b.take<int>(24, A);
  w->bytes[12] = b.last;
  const long nchunk0 = ((long)g.Hp * g.Wp + STAT_CHUNK - 1) / STAT_CHUNK;
  w->part = b.take<float>((size_t)B * nchunk0 * MAXC * 3, A);
  w->mean = b.take<float>((size_t)B * MAXC, A);
  w->rstd = b.take<float>((size_t)B * MAXC, A);
  size_t amax = 0;
  for (int l = 0; l < NL - 1; ++l) {
    w->raw[l] = b.take<float>((size_t)g.lv[DL[l].level].rows * DL[l].cout, A);
    w->bytes[l] = b.last;
    if (l > 0) amax = std::max(amax, (size_t)g.lv[DL[l].level].rows * cpad(DL[l].cin));
  }
  w->ah = b.take<__nv_bfloat16>(amax, A);
  w->al = b.take<__nv_bfloat16>(amax, A);
  w->x3 = b.take<float>((size_t)g.lv[0].rows * X3C, A);
  w->bytes[8] = b.last;
  const size_t hw = (size_t)B * g.H * g.W;
  w->heat = b.take<float>(hw, A);
  w->kept = b.take<float>(hw, A);
  w->row_count = b.take<int>((size_t)B * g.H, A);
  w->row_start = b.take<int>((size_t)B * g.H, A);
  w->n_cand = b.take<int>(B, A);
  w->cand_pos = b.take<int>((size_t)B * g.ccap, A);
  w->cand_score = b.take<float>((size_t)B * g.ccap, A);
  w->sel_pos = b.take<int>((size_t)B * g.ocap, A);
  w->sel_score = b.take<float>((size_t)B * g.ocap, A);
  w->n_sel = b.take<int>(B, A);
  w->dh = b.take<__nv_bfloat16>((size_t)g.ld.rows * DKP, A);
  w->bytes[9] = b.last;
  w->dl = b.take<__nv_bfloat16>((size_t)g.ld.rows * DKP, A);
  w->bytes[10] = b.last;
  w->dout = b.take<float>((size_t)g.ld.rows * DESC, A);
  w->bytes[11] = b.last;
  return b.bytes();
}

// ------------------------------------------------------------------------------------------------------------------
// layer inputs: up to two channel segments, each read directly, 2x2 average pooled, bilinearly upsampled x2
// (align_corners=False) from a padded fp32 map, or taken from the NCHW image (zero outside H x W: the right / bottom pad)
// ------------------------------------------------------------------------------------------------------------------
enum { SRC_DIRECT = 0, SRC_POOL = 1, SRC_UP = 2, SRC_IMAGE = 3 };
struct Seg {
  const float* p;
  int C, ld, mode, Hs, Ws;  // channels, row stride (image: its channel count), source extents
};
struct Prep {
  Seg s[2];
  int B, H, W, C;  // layer resolution, C = s[0].C + s[1].C
};

__device__ __forceinline__ float at_pad(const Seg& s, int b, int y, int x, int c) {
  return s.p[(((long)b * (s.Hs + 4) + y + 2) * (s.Ws + 4) + x + 2) * s.ld + c];
}
__device__ __forceinline__ float seg_val(const Seg& s, int b, int y, int x, int c) {
  if (s.mode == SRC_DIRECT) return at_pad(s, b, y, x, c);
  if (s.mode == SRC_POOL)
    return (at_pad(s, b, 2 * y, 2 * x, c) + at_pad(s, b, 2 * y, 2 * x + 1, c) + at_pad(s, b, 2 * y + 1, 2 * x, c) +
            at_pad(s, b, 2 * y + 1, 2 * x + 1, c)) * 0.25f;
  if (s.mode == SRC_UP) {
    const float sy = fmaxf((y + 0.5f) * 0.5f - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * 0.5f - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = min(y0 + 1, s.Hs - 1), x1 = min(x0 + 1, s.Ws - 1);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    return (1.f - ly) * ((1.f - lx) * at_pad(s, b, y0, x0, c) + lx * at_pad(s, b, y0, x1, c)) +
           ly * ((1.f - lx) * at_pad(s, b, y1, x0, c) + lx * at_pad(s, b, y1, x1, c));
  }
  if (y >= s.Hs || x >= s.Ws) return 0.f;
  return s.p[(((long)b * s.ld + c % s.ld) * s.Hs + y) * s.Ws + x];
}
__device__ __forceinline__ float prep_val(const Prep& p, int b, int y, int x, int c) {
  return c < p.s[0].C ? seg_val(p.s[0], b, y, x, c) : seg_val(p.s[1], b, y, x, c - p.s[0].C);
}
__device__ __forceinline__ float prelu(float v, float a) { return v >= 0.f ? v : a * v; }

__device__ __forceinline__ void chan_merge(float& n, float& m, float& q, float n2, float m2, float q2) {
  if (n2 == 0.f) return;
  const float nn = n + n2, d = m2 - m;
  m += d * (n2 / nn);
  q += q2 + d * d * (n * n2 / nn);
  n = nn;
}

// per (chunk of STAT_CHUNK pixels, image): (count, mean, M2) of every channel; thread t: channel t % C, pixel lane t / C
__global__ void __launch_bounds__(256) disk_stats_partial_kernel(const Prep p, float* __restrict__ part, int nchunk) {
  __shared__ float sn[256], sm[256], sq[256];
  const int chunk = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int C = p.C, lanes = 256 / C;
  const long npix = (long)p.H * p.W;
  const long p0 = (long)chunk * STAT_CHUNK, p1 = min(p0 + STAT_CHUNK, npix);
  float n = 0.f, mean = 0.f, m2 = 0.f;
  if (t < lanes * C) {
    const int c = t % C;
    for (long q = p0 + t / C; q < p1; q += lanes) {
      const float v = prep_val(p, b, (int)(q / p.W), (int)(q % p.W), c);
      n += 1.f;
      const float d = v - mean;
      mean += d / n;
      m2 = fmaf(d, v - mean, m2);
    }
  }
  sn[t] = n; sm[t] = mean; sq[t] = m2;
  __syncthreads();
  if (t < C) {
    for (int l = 1; l < lanes; ++l) chan_merge(n, mean, m2, sn[l * C + t], sm[l * C + t], sq[l * C + t]);
    float* o = part + (((long)b * nchunk + chunk) * C + t) * 3;
    o[0] = n; o[1] = mean; o[2] = m2;
  }
}
// chunks merged in order -> mean, 1 / sqrt(biased variance + 1e-5) per (image, channel) (F.instance_norm)
__global__ void __launch_bounds__(MAXC) disk_stats_final_kernel(const float* __restrict__ part, int nchunk, int C,
                                                                float* __restrict__ mean, float* __restrict__ rstd) {
  const int b = blockIdx.x, c = threadIdx.x;
  if (c >= C) return;
  float n = 0.f, m = 0.f, q = 0.f;
  for (int k = 0; k < nchunk; ++k) {
    const float* o = part + (((long)b * nchunk + k) * C + c) * 3;
    chan_merge(n, m, q, o[0], o[1], o[2]);
  }
  mean[b * MAXC + c] = m;
  rstd[b * MAXC + c] = 1.f / sqrtf(q / n + 1e-5f);
}

// the prepare pass: normalised, PReLU'd layer input -> padded NHWC [rows, cp] (bf16 hi / lo, or fp32 when of != null);
// padding pixels, channels >= C and rows past the last image are zero
__global__ void __launch_bounds__(256) disk_apply_kernel(const Prep p, const float* __restrict__ mean, const float* __restrict__ rstd,
                                                         const float* __restrict__ slope, int cp, long rows,
                                                         __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol,
                                                         float* __restrict__ of) {
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= rows * cp) return;
  const long row = i / cp;
  const int c = (int)(i % cp);
  const int W4 = p.W + 4;
  const long plane = (long)(p.H + 4) * W4;
  const long b = row / plane, pp = row % plane;
  const int y = (int)(pp / W4) - 2, x = (int)(pp % W4) - 2;
  float v = 0.f;
  if (c < p.C && b < p.B && y >= 0 && y < p.H && x >= 0 && x < p.W)
    v = prelu((prep_val(p, (int)b, y, x, c) - mean[b * MAXC + c]) * rstd[b * MAXC + c], slope[c]);
  if (of) of[i] = v;
  else tc_split(v, oh[i], ol[i]);
}

// down0: the image's instance norm and PReLU fused into the 3 -> 16 convolution (K = 75), fp32; one thread per pixel of
// the padded frame Hp x Wp
__global__ void __launch_bounds__(256) disk_down0_kernel(const float* __restrict__ img, int Cimg, int B, int H, int W, int Hp, int Wp,
                                                         const float* __restrict__ mean, const float* __restrict__ rstd,
                                                         const float* __restrict__ blob, float* __restrict__ out) {
  __shared__ float sw[3 + 16 * 75 + 16];  // slopes, weights [co][ci][tap], bias
  for (int i = threadIdx.x; i < 3 + 16 * 75 + 16; i += 256) sw[i] = blob[i];
  __syncthreads();
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= (long)B * Hp * Wp) return;
  const int x = (int)(i % Wp), y = (int)((i / Wp) % Hp), b = (int)(i / ((long)Hp * Wp));
  float acc[16];
#pragma unroll
  for (int co = 0; co < 16; ++co) acc[co] = sw[3 + 16 * 75 + co];
  for (int ci = 0; ci < 3; ++ci) {
    const float mu = mean[b * MAXC + ci], rs = rstd[b * MAXC + ci], a = sw[ci];
    const float* im = img + ((long)b * Cimg + ci % Cimg) * H * W;
#pragma unroll
    for (int t = 0; t < 25; ++t) {
      const int yy = y + t / 5 - 2, xx = x + t % 5 - 2;
      float v = 0.f;
      if (yy >= 0 && yy < Hp && xx >= 0 && xx < Wp) v = prelu((((yy < H && xx < W) ? im[(long)yy * W + xx] : 0.f) - mu) * rs, a);
#pragma unroll
      for (int co = 0; co < 16; ++co) acc[co] = fmaf(v, sw[3 + (co * 3 + ci) * 25 + t], acc[co]);
    }
  }
  float* o = out + (((long)b * (Hp + 4) + y + 2) * (Wp + 4) + x + 2) * 16;
#pragma unroll
  for (int co = 0; co < 16; co += 4) *reinterpret_cast<float4*>(o + co) = make_float4(acc[co], acc[co + 1], acc[co + 2], acc[co + 3]);
}

// heatmap channel of up3 over the cropped H x W pixels: 5x5x80 fp32 dot with the padded up3 input
__global__ void __launch_bounds__(256) disk_heatmap_kernel(const float* __restrict__ x3, const float* __restrict__ w,
                                                           const float* __restrict__ bias, int B, int H, int W, int Hp, int Wp,
                                                           float* __restrict__ heat) {
  __shared__ float4 sw[DK / 4];
  for (int i = threadIdx.x; i < DK / 4; i += 256) sw[i] = reinterpret_cast<const float4*>(w)[i];
  __syncthreads();
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= (long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H), b = (int)(i / ((long)H * W));
  const float* base = x3 + (((long)b * (Hp + 4) + y) * (Wp + 4) + x) * X3C;  // tap (0, 0) = pixel (y - 2, x - 2)
  float acc = 0.f;
  for (int t = 0; t < 25; ++t) {
    const float4* q = reinterpret_cast<const float4*>(base + ((long)(t / 5) * (Wp + 4) + t % 5) * X3C);
#pragma unroll
    for (int j = 0; j < X3C / 4; ++j) {
      const float4 v = q[j], k = sw[t * (X3C / 4) + j];
      acc = fmaf(v.x, k.x, acc); acc = fmaf(v.y, k.y, acc); acc = fmaf(v.z, k.z, acc); acc = fmaf(v.w, k.w, acc);
    }
  }
  heat[i] = acc + bias[0];
}

// NMS (max_pool2d(w, stride 1, padding w/2, return_indices) == own index): a pixel is kept iff no earlier pixel of its
// window (row-major) is >= and no later one is >; kept pixels keep their value, the others become -inf
__global__ void __launch_bounds__(256) disk_nms_kernel(const float* __restrict__ heat, float* __restrict__ kept, int B, int H, int W,
                                                       int r) {
  const long i = blockIdx.x * 256L + threadIdx.x;
  if (i >= (long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  const float* hb = heat + (i - (long)y * W - x);
  const float v = heat[i];
  bool keep = true;
  for (int dy = -r; dy <= r && keep; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -r; dx <= r; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W || (dy == 0 && dx == 0)) continue;
      const float q = hb[(long)yy * W + xx];
      if ((dy < 0 || (dy == 0 && dx < 0)) ? q >= v : q > v) { keep = false; break; }
    }
  }
  kept[i] = keep ? v : -INFINITY;
}

// im2col rows of the descriptor head: row b out_cap + j <- the 5x5x80 up3 inputs around pixel sel_pos[row] (column
// tap 80 + ci, zero past 2000), bf16 hi / lo; slots past n_sel[b] and rows past the last image are zero
__global__ void __launch_bounds__(256) disk_gather_kernel(const float* __restrict__ x3, const int* __restrict__ n_sel,
                                                          const int* __restrict__ sel_pos, int B, int W, int Hp, int Wp, long out_cap,
                                                          __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol) {
  const long row = blockIdx.x;
  const long b = row / out_cap, j = row % out_cap;
  const bool valid = b < B && j < n_sel[b];
  const int pos = valid ? sel_pos[row] : 0;
  const int y = pos / W, x = pos % W;
  const float* base = x3 + (((long)b * (Hp + 4) + y) * (Wp + 4) + x) * X3C;
  for (int col = threadIdx.x; col < DKP; col += 256) {
    float v = 0.f;
    if (valid && col < DK) {
      const int t = col / X3C, ci = col % X3C;
      v = base[((long)(t / 5) * (Wp + 4) + t % 5) * X3C + ci];
    }
    tc_split(v, oh[row * DKP + col], ol[row * DKP + col]);
  }
}

// outputs of slot (j, b) (row b out_stride + j): descriptor (L2-normalised when `normalize`: F.normalize, eps 1e-12),
// keypoint (x, y), score of selection row b sel_cap + j; zeros past n_sel[b]
__global__ void __launch_bounds__(DESC) disk_finish_kernel(const float* __restrict__ g, const int* __restrict__ n_sel,
                                                           const int* __restrict__ sel_pos, const float* __restrict__ sel_score, int W,
                                                           long sel_cap, long out_stride, int normalize, float* __restrict__ kpts,
                                                           float* __restrict__ scores, float* __restrict__ desc) {
  __shared__ float red[DESC / 32];
  const long j = blockIdx.x, b = blockIdx.y, row = b * out_stride + j, srow = b * sel_cap + j;
  const int c = threadIdx.x;
  if (j >= n_sel[b]) {
    desc[row * DESC + c] = 0.f;
    if (c == 0 && kpts) { kpts[2 * row] = 0.f; kpts[2 * row + 1] = 0.f; scores[row] = 0.f; }
    return;
  }
  float v = g[srow * DESC + c];
  if (normalize) {
    float ss = v * v;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
    if ((c & 31) == 0) red[c >> 5] = ss;
    __syncthreads();
    const float tot = red[0] + red[1] + red[2] + red[3];
    v = v / fmaxf(sqrtf(tot), 1e-12f);
  }
  desc[row * DESC + c] = v;
  if (c == 0 && kpts) {
    const int pos = sel_pos[srow];
    kpts[2 * row] = (float)(pos % W);
    kpts[2 * row + 1] = (float)(pos / W);
    scores[row] = sel_score[srow];
  }
}

__global__ void disk_fill_kernel(int* p, int n, int v) {
  if ((int)threadIdx.x < n) p[threadIdx.x] = v;
}

}  // namespace

struct DiskHandle {
  DiskConfig cfg;
  float* wts;  // device copy of the weight blob
  // packed regions: l - 1 = layer l (1..7) [256, 25 cpad(cin)]; NL - 2 = up3's descriptor head [256, 2048]; HEAT = up3's
  // heatmap channel [1, 2000] (tap 80 + ci)
  TcConvWeights* cw;
};

namespace {

int launch_stats(const Prep& p, const DiskWs& w, cudaStream_t s) {
  const int nchunk = (int)(((long)p.H * p.W + STAT_CHUNK - 1) / STAT_CHUNK);
  disk_stats_partial_kernel<<<dim3(nchunk, p.B), 256, 0, s>>>(p, w.part, nchunk);
  disk_stats_final_kernel<<<p.B, MAXC, 0, s>>>(w.part, nchunk, p.C, w.mean, w.rstd);
  return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("disk: statistics launch failed");
}

// the input of layer l >= 1 (kornia's Unet.forward)
Prep layer_input(const Geo& g, const DiskWs& w, int l) {
  Prep p{};
  const int L = DL[l].level, S = DL[l - 1].level;
  p.B = g.B; p.H = g.Hp >> L; p.W = g.Wp >> L; p.C = DL[l].cin;
  if (l <= 4) {  // avg_pool2d(2) of the previous down block's output
    p.s[0] = Seg{w.raw[l - 1], DL[l - 1].cout, DL[l - 1].cout, SRC_POOL, g.Hp >> S, g.Wp >> S};
  } else {  // cat([upsample(bottom), horizontal])
    const int hl = 8 - l;  // horizontal: down block 3, 2, 1, 0
    const int Hz = DL[hl].level;
    p.s[0] = Seg{w.raw[l - 1], DL[l - 1].cout, DL[l - 1].cout, SRC_UP, g.Hp >> S, g.Wp >> S};
    p.s[1] = Seg{w.raw[hl], DL[hl].cout, DL[hl].cout, SRC_DIRECT, g.Hp >> Hz, g.Wp >> Hz};
  }
  return p;
}

// the U-Net up to the heatmap: writes w.x3 (up3 input) and heat [B, H, W]; the state words of the levels and of `ld`,
// the row plan the descriptor GEMM will run on
int run_unet(DiskHandle* h, const float* image, int Cimg, const Geo& g, const TcRows& ld, const DiskWs& w, float* heat,
             cudaStream_t s) {
  const TcRows plans[6] = {g.lv[0], g.lv[1], g.lv[2], g.lv[3], g.lv[4], ld};
  LG_RC(tc_rows_words(plans, 6, w.state, s));
  {  // down0
    Prep p{};
    p.B = g.B; p.H = g.Hp; p.W = g.Wp; p.C = 3;
    p.s[0] = Seg{image, 3, Cimg, SRC_IMAGE, g.H, g.W};
    LG_RC(launch_stats(p, w, s));
    const long n = (long)g.B * g.Hp * g.Wp;
    disk_down0_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(image, Cimg, g.B, g.H, g.W, g.Hp, g.Wp, w.mean, w.rstd, h->wts,
                                                                  w.raw[0]);
    LG_CHECK_LAUNCH();
  }
  for (int l = 1; l < NL; ++l) {
    const Prep p = layer_input(g, w, l);
    const TcRows& L = g.lv[DL[l].level];
    LG_RC(launch_stats(p, w, s));
    const float* slope = h->wts + layer_blob_off(l);
    const int cp = l < NL - 1 ? cpad(DL[l].cin) : X3C;
    const long n = L.rows * cp;
    disk_apply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, w.mean, w.rstd, slope, cp, L.rows, w.ah, w.al,
                                                                  l < NL - 1 ? nullptr : w.x3);
    LG_CHECK_LAUNCH();
    if (l == NL - 1) break;
    LG_RC(tc_conv(*h->cw, tc_rows_state(L, w.state + 4 * DL[l].level), {.in_h = w.ah, .in_l = w.al, .cin = cp, .taps = TAPS,
                  .region = l - 1, .B = g.B, .H = p.H, .W = p.W, .cout = DL[l].cout, .out_f32 = w.raw[l], .ldo = DL[l].cout}, s));
  }
  const long n = (long)g.B * g.H * g.W;
  const TcConvWeights& cw = *h->cw;
  disk_heatmap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.x3, cw.wpk + cw.w_off[HEAT], cw.wpk + cw.b_off[HEAT], g.B, g.H,
                                                                  g.W, g.Hp, g.Wp, heat);
  LG_CHECK_LAUNCH();
  return 0;
}

// descriptor head at the pixels sel_pos (n_sel per image, oc selection slots per image) -> desc [B, out_stride, 128];
// its state words (w.state + 20) must be those of tc_rows(B oc), written by run_unet
int run_desc(DiskHandle* h, const Geo& g, const DiskWs& w, const int* n_sel, const int* sel_pos, const float* sel_score, long oc,
             long out_stride, int normalize, float* kpts, float* scores, float* desc, cudaStream_t s) {
  if (oc <= 0 || out_stride <= 0) return 0;
  const TcRows ld = tc_rows((long)g.B * oc);
  disk_gather_kernel<<<(unsigned)ld.rows, 256, 0, s>>>(w.x3, n_sel, sel_pos, g.B, g.W, g.Hp, g.Wp, oc, w.dh, w.dl);
  LG_CHECK_LAUNCH();
  LG_RC(tc_conv(*h->cw, tc_rows_state(ld, w.state + 20), {.in_h = w.dh, .in_l = w.dl, .cin = DKP, .taps = 1, .region = NL - 2,
                .cout = DESC, .out_f32 = w.dout, .ldo = DESC}, s));
  disk_finish_kernel<<<dim3((unsigned)out_stride, g.B), DESC, 0, s>>>(w.dout, n_sel, sel_pos, sel_score, g.W, oc, out_stride,
                                                                      normalize, kpts, scores, desc);
  LG_CHECK_LAUNCH();
  return 0;
}

int check_size(const DiskConfig& c, int B, int H, int W, int Cimg) {
  if (B <= 0 || H <= 0 || W <= 0) return lg_set_error("disk: B, H and W must be positive");
  if (Cimg != 1 && Cimg != 3) return lg_set_error("disk: the image must have 1 or 3 channels");
  if (!c.pad_if_not_divisible && (H % 16 || W % 16))
    return lg_set_error("disk: H and W must be multiples of 16 when pad_if_not_divisible is off");
  const int Hp = (H + 15) / 16, Wp = (W + 15) / 16;
  if ((long)Hp * Wp < 2) return lg_set_error("disk: the padded image needs at least two pixels at 1/16 resolution");
  return 0;
}

}  // namespace

extern "C" size_t disk_weight_blob_floats(void) { return layer_blob_off(NL); }

extern "C" int disk_create(const DiskConfig* cfg, const float* weights_dev, size_t n_floats, void* stream_, DiskHandle** out) {
  if (!cfg || !weights_dev || !out) return lg_set_error("disk_create: null argument");
  if (cfg->abi_version != DISK_ABI_VERSION) return lg_set_error("disk_create: ABI version mismatch");
  if (n_floats != disk_weight_blob_floats()) return lg_set_error("disk_create: weight blob has the wrong size");
  if (cfg->nms_window_size < 1 || cfg->nms_window_size % 2 == 0) return lg_set_error("disk_create: nms_window_size must be odd");
  if (cfg->max_num_keypoints < -1) return lg_set_error("disk_create: max_num_keypoints must be -1 (None) or >= 0");
  cudaStream_t stream = (cudaStream_t)stream_;
  DiskHandle* h = new (std::nothrow) DiskHandle{};
  if (!h) return lg_set_error("disk_create: out of host memory");
  h->cfg = *cfg;
  struct Guard {
    DiskHandle* h;
    ~Guard() { if (h) disk_destroy(h); }
  } guard{h};
  LG_CU(cudaMalloc(&h->wts, n_floats * sizeof(float)));
  LG_CU(cudaMemcpyAsync(h->wts, weights_dev, n_floats * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  TcConvRegion reg[NL];
  for (int l = 1; l < NL; ++l) {  // up3 (l = NL - 1): the descriptor head, then the heatmap channel
    const float* w = h->wts + layer_blob_off(l) + DL[l].cin;
    const float* b = w + (size_t)DL[l].cout * DL[l].cin * TAPS;
    const int cin = DL[l].cin, cp = cpad(cin);
    if (l < NL - 1) {
      reg[l - 1] = {.w = w, .b = b, .cin = cin, .cpad = cp, .taps = TAPS, .rows = 256, .K = TAPS * cp, .ncopy = DL[l].cout};
    } else {
      reg[l - 1] = {.w = w, .b = b, .cin = X3C, .cpad = X3C, .taps = TAPS, .rows = 256, .K = DKP, .ncopy = DESC};
      reg[HEAT] = {.w = w, .b = b, .cin = X3C, .cpad = X3C, .taps = TAPS, .rows = 1, .K = DK, .co0 = DESC, .ncopy = 1};
    }
  }
  LG_RC(tc_conv_weights_create(&h->cw, reg, NL, stream));
  guard.h = nullptr;
  *out = h;
  return 0;
}

extern "C" int disk_destroy(DiskHandle* h) {
  if (!h) return 0;
  tc_conv_weights_destroy(h->cw);
  cudaFree(h->wts);
  delete h;
  return 0;
}

extern "C" int64_t disk_max_keypoints(const DiskHandle* h, int32_t H, int32_t W) {
  return h && H > 0 && W > 0 ? out_cap(h->cfg, H, W) : 0;
}

extern "C" size_t disk_workspace_bytes(const DiskHandle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  DiskWs w;
  return carve(nullptr, geometry(h->cfg, B, H, W), &w);
}

extern "C" int64_t disk_workspace_layout(const DiskHandle* h, int32_t B, int32_t H, int32_t W, int64_t* offsets,
                                         int64_t* bytes) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  DiskWs w;
  char* const base = reinterpret_cast<char*>(kLayoutBase);
  const size_t total = carve(base, geometry(h->cfg, B, H, W), &w);
  const void* p[DISK_LAYOUT_BUFFERS] = {w.raw[0], w.raw[1], w.raw[2], w.raw[3], w.raw[4], w.raw[5], w.raw[6],
                                        w.raw[7], w.x3,     w.dh,     w.dl,     w.dout,   w.state};
  for (int i = 0; i < DISK_LAYOUT_BUFFERS; ++i) {
    if (offsets) offsets[i] = (int64_t)((const char*)p[i] - base);
    if (bytes) bytes[i] = (int64_t)w.bytes[i];
  }
  return (int64_t)total;
}

extern "C" int disk_forward(DiskHandle* h, const float* image, int32_t C, int32_t B, int32_t H, int32_t W, int64_t cap,
                            float* keypoints, float* scores, float* descriptors, int32_t* counts, void* workspace,
                            size_t workspace_bytes, void* stream_) {
  if (!h || !image || !keypoints || !scores || !descriptors || !counts) return lg_set_error("disk_forward: null argument");
  LG_RC(check_size(h->cfg, B, H, W, C));
  if (cap < disk_max_keypoints(h, H, W)) return lg_set_error("disk_forward: output capacity below disk_max_keypoints()");
  const Geo g = geometry(h->cfg, B, H, W);
  DiskWs w;
  if (!workspace || workspace_bytes < carve(nullptr, g, &w)) return lg_set_error("disk_forward: workspace too small");
  carve((char*)workspace, g, &w);
  cudaStream_t s = (cudaStream_t)stream_;
  LG_RC(run_unet(h, image, C, g, g.ld, w, w.heat, s));
  const long n = (long)B * H * W;
  const int r = h->cfg.nms_window_size / 2;
  disk_nms_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.heat, w.kept, B, H, W, r);
  LG_CHECK_LAUNCH();
  LG_RC(kp_compact(w.kept, B, H, W, h->cfg.detection_threshold, g.ccap, w.row_count, w.row_start, w.n_cand, w.cand_pos,
                   w.cand_score, s));
  LG_RC(kp_select_above_kth(w.n_cand, w.cand_pos, w.cand_score, w.sel_pos, w.sel_score, w.n_sel, B, h->cfg.max_num_keypoints,
                            g.ccap, g.ocap, s));
  LG_RC(run_desc(h, g, w, w.n_sel, w.sel_pos, w.sel_score, g.ocap, cap, 1, keypoints, scores, descriptors, s));
  LG_CU(cudaMemcpyAsync(counts, w.n_sel, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  return 0;
}

extern "C" int disk_heads(DiskHandle* h, const float* image, int32_t C, int32_t B, int32_t H, int32_t W, const int32_t* pos,
                          int32_t P, float* heatmap, float* descriptors, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!h || !image || !heatmap || (P > 0 && (!pos || !descriptors))) return lg_set_error("disk_heads: null argument");
  LG_RC(check_size(h->cfg, B, H, W, C));
  if (P < 0 || P > disk_max_keypoints(h, H, W)) return lg_set_error("disk_heads: P must be in [0, disk_max_keypoints()]");
  if (B > 1024) return lg_set_error("disk_heads: at most 1024 images");
  const Geo g = geometry(h->cfg, B, H, W);
  DiskWs w;
  if (!workspace || workspace_bytes < carve(nullptr, g, &w)) return lg_set_error("disk_heads: workspace too small");
  carve((char*)workspace, g, &w);
  cudaStream_t s = (cudaStream_t)stream_;
  LG_RC(run_unet(h, image, C, g, tc_rows((long)B * P), w, heatmap, s));
  disk_fill_kernel<<<1, 1024, 0, s>>>(w.n_sel, B, P);
  LG_CHECK_LAUNCH();
  return run_desc(h, g, w, w.n_sel, pos, nullptr, P, P, 0, nullptr, nullptr, descriptors, s);
}
