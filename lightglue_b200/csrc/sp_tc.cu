// SuperPoint encoder + heads on the tensor cores (SURVEY.md 8f1; reference lightglue/superpoint.py:137-153, 171-190,
// 220-221): the twelve convolutions as implicit GEMMs through the wgmma / TMA linear kernel the matcher uses (tc_conv,
// on the packed weights of a TcConvWeights and the row plan of lg_tc.h), split-bf16 operands (hi + lo, three MMAs per
// product: ~fp32 accuracy), fp32 accumulate.
//
// Data layout: every feature map is a ZERO-PADDED NHWC image stored as a matrix [rows, C] of bf16 hi / lo images, row =
// padded pixel b (H+2)(W+2) + y (W+2) + x.  A 3x3 tap (dy, dx) of such a map is the same matrix shifted by
// dy (W+2) + dx rows, so the convolution is a GEMM with K = 9 Cin whose A tiles TMA fetches with a row offset (rows
// outside the matrix read as zeros); the epilogue re-zeroes the padding pixels so that the next layer's taps see the
// zero padding of nn.Conv2d(padding=1).  conv1a (Cin = 1: K = 9) and the 2x2 max-poolings are small CUDA-core kernels
// in the same layout; the two 1x1 heads write fp32, which two transposition kernels hand to the post-processing
// functors of sp_pipeline.h (65-way soft-max, NMS, top-k, descriptor sampling) in their NCHW layout.
// The fp32 CUDA-core functor path (sp_pipeline.h SpConv) stays as the checker (SpConfig.precision = 0).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "sp_pipeline.h"
#include "sp_tc.h"

namespace {

// conv1a (1 -> 64, 3x3, zero padding) + bias + ReLU from the fp32 image into the padded NHWC hi / lo layout; eight threads
// per padded pixel (eight channels each: one 16-byte store per image), weights in shared memory; padding pixels and the
// rows past the last image are written as zeros
__global__ void __launch_bounds__(256) sp_conv1a_kernel(const float* __restrict__ img, const float* __restrict__ w,
                                                        const float* __restrict__ bias, __nv_bfloat16* __restrict__ oh,
                                                        __nv_bfloat16* __restrict__ ol, int B, int H, int W, long rows_total) {
  __shared__ float sw[64 * 9 + 64];
  for (int i = threadIdx.x; i < 64 * 9 + 64; i += 256) sw[i] = i < 64 * 9 ? w[i] : bias[i - 64 * 9];
  __syncthreads();
  const long i = blockIdx.x * 256L + threadIdx.x;
  const long row = i / 8;
  const int c0 = (int)(i % 8) * 8;
  if (row >= rows_total) return;
  const int W2 = W + 2;
  const long plane = (long)(H + 2) * W2;
  const long b = row / plane, pp = row % plane;
  const int y = (int)(pp / W2) - 1, x = (int)(pp % W2) - 1;
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = 0.f;
  if (b < B && y >= 0 && y < H && x >= 0 && x < W) {
    const float* im = img + b * (long)H * W;
    float px[9];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int yy = y + ky - 1, xx = x + kx - 1;
        px[ky * 3 + kx] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? im[(long)yy * W + xx] : 0.f;
      }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float a = sw[64 * 9 + c0 + c];
#pragma unroll
      for (int t = 0; t < 9; ++t) a = fmaf(px[t], sw[(c0 + c) * 9 + t], a);
      v[c] = fmaxf(a, 0.f);
    }
  }
  uint32_t hv[4], lv[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    __nv_bfloat162 h2, l2;
    tc_split(v[2 * c], h2.x, l2.x);
    tc_split(v[2 * c + 1], h2.y, l2.y);
    hv[c] = *reinterpret_cast<const uint32_t*>(&h2);
    lv[c] = *reinterpret_cast<const uint32_t*>(&l2);
  }
  *reinterpret_cast<uint4*>(oh + row * 64 + c0) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
  *reinterpret_cast<uint4*>(ol + row * 64 + c0) = make_uint4(lv[0], lv[1], lv[2], lv[3]);
}

// 2x2 max pooling, stride 2 (superpoint.py:135), padded NHWC (H, W) -> padded NHWC (H/2, W/2); one thread per (output
// padded pixel, channel pair).  The pooled value keeps the (hi, lo) pair of the winning element: hi + lo is exact.
__global__ void __launch_bounds__(256) sp_pool_kernel(const __nv_bfloat16* __restrict__ ih, const __nv_bfloat16* __restrict__ il,
                                                      __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol, int B, int H,
                                                      int W, int C, long rows_out_total) {
  const int cpn = C / 2;
  const long i = blockIdx.x * 256L + threadIdx.x;
  const long row = i / cpn;
  const int cp = (int)(i % cpn);
  if (row >= rows_out_total) return;
  const int Ho = H / 2, Wo = W / 2, W2o = Wo + 2, W2i = W + 2;
  const long plane_o = (long)(Ho + 2) * W2o, plane_i = (long)(H + 2) * W2i;
  const long b = row / plane_o, pp = row % plane_o;
  const int yo = (int)(pp / W2o), xo = (int)(pp % W2o);
  __nv_bfloat162 bh = __floats2bfloat162_rn(0.f, 0.f), bl = bh;
  if (b < B && yo >= 1 && yo <= Ho && xo >= 1 && xo <= Wo) {
    const long base = b * plane_i + (long)(2 * yo - 1) * W2i + (2 * xo - 1);
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const long r = base + (t / 2) * W2i + (t % 2);
      const __nv_bfloat162 h2 = *reinterpret_cast<const __nv_bfloat162*>(ih + r * C + 2 * cp);
      const __nv_bfloat162 l2 = *reinterpret_cast<const __nv_bfloat162*>(il + r * C + 2 * cp);
      const float a0 = __bfloat162float(h2.x) + __bfloat162float(l2.x), a1 = __bfloat162float(h2.y) + __bfloat162float(l2.y);
      if (a0 > m0) { m0 = a0; bh.x = h2.x; bl.x = l2.x; }
      if (a1 > m1) { m1 = a1; bh.y = h2.y; bl.y = l2.y; }
    }
  }
  *reinterpret_cast<__nv_bfloat162*>(oh + row * C + 2 * cp) = bh;
  *reinterpret_cast<__nv_bfloat162*>(ol + row * C + 2 * cp) = bl;
}

// padded NHWC fp32 [rows, ld] (first C channels) -> dense NCHW fp32 [B, C, H, W]
__global__ void __launch_bounds__(256) sp_to_nchw_kernel(const float* __restrict__ in, int ld, float* __restrict__ out, int B, int C,
                                                         int H, int W) {
  const long i = blockIdx.x * 256L + threadIdx.x;
  const long n = (long)B * C * H * W;
  if (i >= n) return;
  const int c = (int)(i % C);
  long r = i / C;
  const int x = (int)(r % W); r /= W;
  const int y = (int)(r % H);
  const long b = r / H;
  const long prow = b * (long)(H + 2) * (W + 2) + (long)(y + 1) * (W + 2) + (x + 1);
  out[((b * C + c) * H + y) * W + x] = in[prow * ld + c];
}

// ------------------------------------------------------------------------------------------------------------------
// Warp / block versions of the three heavy post-processing stages (same results as the functors SpRowCount / SpRowScan /
// SpRowWrite, SpSelect, SpSample of sp_pipeline.h, which stay the semantic definition and the fp32 path's implementation)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sp_row_count_kernel(const float* __restrict__ scores, int* __restrict__ row_count, long rows,
                                                           int W, float thr) {
  const long r = blockIdx.x * 8L + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= rows) return;
  const float* p = scores + r * W;
  int c = 0;
  for (int x = lane; x < W; x += 32) c += p[x] > thr ? 1 : 0;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
  if (lane == 0) row_count[r] = c;
}
// exclusive scan of the row counts of one image (one block per image)
__global__ void __launch_bounds__(1024) sp_row_scan_kernel(const int* __restrict__ row_count, int* __restrict__ row_start,
                                                           int* __restrict__ n_cand, int H) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < H; base += 1024) {
    const int y = base + tid;
    const int v = y < H ? row_count[(long)b * H + y] : 0;
    int incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, off);
      if ((tid & 31) >= off) incl += t;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
      int w = wsum[tid];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, off);
        if (tid >= off) w += t;
      }
      wsum[tid] = w;
    }
    __syncthreads();
    const int c = carry;
    if (y < H) row_start[(long)b * H + y] = c + ((tid >> 5) ? wsum[(tid >> 5) - 1] : 0) + incl - v;
    __syncthreads();
    if (tid == 0) carry = c + wsum[31];
    __syncthreads();
  }
  if (tid == 0) n_cand[b] = carry;
}
__global__ void __launch_bounds__(256) sp_row_write_kernel(const float* __restrict__ scores, const int* __restrict__ row_start,
                                                           int* __restrict__ cand_pos, float* __restrict__ cand_score, long rows,
                                                           int H, int W, float thr, long cap) {
  const long r = blockIdx.x * 8L + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= rows) return;
  const long b = r / H;
  const int y = (int)(r % H);
  const float* p = scores + r * W;
  long o = b * cap + row_start[r];
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane;
    const float v = x < W ? p[x] : 0.f;
    const bool f = x < W && v > thr;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (f) {
      const long q = o + __popc(m & ((1u << lane) - 1u));
      cand_pos[q] = y * W + x;
      cand_score[q] = v;
    }
    o += __popc(m);
  }
}

// top-k (71-76): radix select of the k-th largest score (4 x 8 bits), equals taken in candidate order, then the rank of
// every survivor among the survivors (score descending, candidate index ascending) -- what SpSelect computes by
// counting over ALL candidates.  One block per image; k <= SP_SEL_KMAX.
#define SP_SEL_KMAX 4096
__device__ __forceinline__ unsigned sp_key(float f) {  // order-preserving map float -> unsigned
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// radix select over the n scores s (blockDim 1024, 4 x 8 bits): on entry s_prefix = 0 and s_remaining = k; on exit
// s_prefix is the key of the k-th largest score and s_remaining how many candidates with exactly that key rank <= k
__device__ void radix_kth_largest(const float* s, int n, int* hist, unsigned& s_prefix, int& s_remaining) {
  const int tid = threadIdx.x;
  for (int pass = 3; pass >= 0; --pass) {
    for (int i = tid; i < 256; i += 1024) hist[i] = 0;
    __syncthreads();
    const unsigned prefix = s_prefix;
    const unsigned himask = pass == 3 ? 0u : (0xffffffffu << (8 * (pass + 1)));
    for (int j = tid; j < n; j += 1024) {
      const unsigned key = sp_key(s[j]);
      if ((key & himask) == (prefix & himask)) atomicAdd(&hist[(key >> (8 * pass)) & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int rem = s_remaining, d = 255;
      for (; d > 0; --d) {
        if (hist[d] >= rem) break;
        rem -= hist[d];
      }
      s_prefix = prefix | ((unsigned)d << (8 * pass));
      s_remaining = rem;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024) sp_select_kernel(const int* __restrict__ n_cand, const int* __restrict__ cand_pos,
                                                         const float* __restrict__ cand_score, int* __restrict__ sel_pos,
                                                         float* __restrict__ sel_score, int* __restrict__ n_sel, int k, long cap,
                                                         long out_cap, int rank_all) {
  __shared__ float ss[SP_SEL_KMAX];
  __shared__ int sj[SP_SEL_KMAX];
  __shared__ int hist[256];
  __shared__ int wsum[32];
  __shared__ unsigned s_prefix;
  __shared__ int s_remaining, s_count, s_carry;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = n_cand[b];
  const float* s = cand_score + (long)b * cap;
  const int* pos = cand_pos + (long)b * cap;
  if (!(k > 0 && (n > k || (rank_all && n > 0)))) {  // nothing to drop or rank: row-major order is kept (the reference returns early)
    const int m = n < out_cap ? n : (int)out_cap;
    if (tid == 0) n_sel[b] = m;
    for (int j = tid; j < m; j += 1024) { sel_pos[(long)b * out_cap + j] = pos[j]; sel_score[(long)b * out_cap + j] = s[j]; }
    return;
  }
  if (n < k) k = n;  // rank_all with fewer candidates than k: keep (and rank) them all
  if (tid == 0) { s_prefix = 0u; s_remaining = k; s_count = 0; s_carry = 0; n_sel[b] = k; }
  __syncthreads();
  radix_kth_largest(s, n, hist, s_prefix, s_remaining);
  const unsigned T = s_prefix;   // key of the k-th largest score
  const int take_eq = s_remaining;  // how many candidates with exactly that score are kept: the first ones
  for (int base = 0; base < n; base += 1024) {
    const int j = base + tid;
    const unsigned key = j < n ? sp_key(s[j]) : 0u;
    const bool gt = j < n && key > T, eq = j < n && key == T;
    // rank of this candidate among the equals, in candidate order (block-wide exclusive scan + running carry)
    const unsigned m = __ballot_sync(0xffffffffu, eq);
    const int in_warp = __popc(m & ((1u << (tid & 31)) - 1u));
    if ((tid & 31) == 0) wsum[tid >> 5] = __popc(m);
    __syncthreads();
    if (tid < 32) {
      int w = wsum[tid], incl = w;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (tid >= off) incl += t;
      }
      wsum[tid] = incl - w;  // exclusive
      if (tid == 31) hist[0] = incl;  // total equals of this chunk
    }
    __syncthreads();
    const int eq_rank = s_carry + wsum[tid >> 5] + in_warp;
    if (gt || (eq && eq_rank < take_eq)) {
      const int slot = atomicAdd(&s_count, 1);
      if (slot < SP_SEL_KMAX) { ss[slot] = s[j]; sj[slot] = j; }
    }
    __syncthreads();
    if (tid == 0) s_carry += hist[0];
    __syncthreads();
  }
  const int cnt = s_count < k ? s_count : k;  // == k
  for (int i = tid; i < cnt; i += 1024) {
    const float me = ss[i];
    const int mj = sj[i];
    int rank = 0;
    for (int t = 0; t < cnt; ++t) rank += (ss[t] > me || (ss[t] == me && sj[t] < mj)) ? 1 : 0;
    if (rank < out_cap) { sel_pos[(long)b * out_cap + rank] = pos[mj]; sel_score[(long)b * out_cap + rank] = me; }
  }
}

// kornia's DISK top-k (n = k_max >= 0): k = min(n + 1, count), keep the candidates strictly above the k-th largest score,
// then the first n of them, all in candidate (row-major) order.  k_max < 0: every candidate.  One block per image.
__global__ void __launch_bounds__(1024) kp_select_above_kernel(const int* __restrict__ n_cand, const int* __restrict__ cand_pos,
                                                               const float* __restrict__ cand_score, int* __restrict__ sel_pos,
                                                               float* __restrict__ sel_score, int* __restrict__ n_sel, int k_max,
                                                               long cap, long out_cap) {
  __shared__ int hist[256];
  __shared__ int wsum[32];
  __shared__ unsigned s_prefix;
  __shared__ int s_remaining, s_carry;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = n_cand[b];
  const float* s = cand_score + (long)b * cap;
  const int* pos = cand_pos + (long)b * cap;
  const long lim = k_max < 0 ? out_cap : (k_max < out_cap ? k_max : out_cap);
  if (k_max < 0 || n == 0) {
    const int m = n < lim ? n : (int)lim;
    if (tid == 0) n_sel[b] = m;
    for (int j = tid; j < m; j += 1024) { sel_pos[(long)b * out_cap + j] = pos[j]; sel_score[(long)b * out_cap + j] = s[j]; }
    return;
  }
  if (tid == 0) { s_prefix = 0u; s_remaining = k_max < n ? k_max + 1 : n; s_carry = 0; }
  __syncthreads();
  radix_kth_largest(s, n, hist, s_prefix, s_remaining);
  const unsigned T = s_prefix;
  for (int base = 0; base < n; base += 1024) {
    const int j = base + tid;
    const bool gt = j < n && sp_key(s[j]) > T;
    const unsigned m = __ballot_sync(0xffffffffu, gt);
    const int in_warp = __popc(m & ((1u << (tid & 31)) - 1u));
    if ((tid & 31) == 0) wsum[tid >> 5] = __popc(m);
    __syncthreads();
    if (tid < 32) {
      int w = wsum[tid], incl = w;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (tid >= off) incl += t;
      }
      wsum[tid] = incl - w;
      if (tid == 31) hist[0] = incl;
    }
    __syncthreads();
    const int rank = s_carry + wsum[tid >> 5] + in_warp;
    if (gt && rank < lim) { sel_pos[(long)b * out_cap + rank] = pos[j]; sel_score[(long)b * out_cap + rank] = s[j]; }
    __syncthreads();
    if (tid == 0) s_carry += hist[0];
    __syncthreads();
  }
  if (tid == 0) n_sel[b] = s_carry < lim ? s_carry : (int)lim;
}

// one block (256 threads = the 256 descriptor channels) per keypoint slot: bilinear sample + L2 normalisation (79-96)
__global__ void __launch_bounds__(256) sp_sample_kernel(const int* __restrict__ n_sel, const int* __restrict__ sel_pos,
                                                        const float* __restrict__ sel_score, const float* __restrict__ dense,
                                                        float* __restrict__ kpts, float* __restrict__ kscores, float* __restrict__ desc,
                                                        int Hc, int Wc, long out_cap) {
  __shared__ float red[8];
  const long j = blockIdx.x, b = blockIdx.y;
  const long i = b * out_cap + j;
  const int c = threadIdx.x;
  float* dd = desc + i * SP_DESC;
  if (j >= n_sel[b]) {  // padding slots: zeros
    if (c == 0) { kpts[i * 2] = 0.f; kpts[i * 2 + 1] = 0.f; kscores[i] = 0.f; }
    dd[c] = 0.f;
    return;
  }
  const int W = Wc * SP_CELL;
  const int pos = sel_pos[i];
  const float x = (float)(pos % W), y = (float)(pos / W);
  if (c == 0) { kpts[i * 2] = x; kpts[i * 2 + 1] = y; kscores[i] = sel_score[i]; }
  const float s = (float)SP_CELL;
  const float gx = (x - s / 2 + 0.5f) / ((float)Wc * s - s / 2 - 0.5f) * 2.f - 1.f;
  const float gy = (y - s / 2 + 0.5f) / ((float)Hc * s - s / 2 - 0.5f) * 2.f - 1.f;
  const float px = (gx + 1.f) * 0.5f * (float)(Wc - 1), py = (gy + 1.f) * 0.5f * (float)(Hc - 1);
  const float fx = floorf(px), fy = floorf(py);
  const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
  const float ax = px - fx, ay = py - fy;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  const bool v00 = x0 >= 0 && x0 < Wc && y0 >= 0 && y0 < Hc, v01 = x1 >= 0 && x1 < Wc && y0 >= 0 && y0 < Hc;
  const bool v10 = x0 >= 0 && x0 < Wc && y1 >= 0 && y1 < Hc, v11 = x1 >= 0 && x1 < Wc && y1 >= 0 && y1 < Hc;
  const long plane = (long)Hc * Wc;
  const float* p = dense + (b * SP_DESC + c) * plane;
  float v = 0.f;
  if (v00) v += p[(long)y0 * Wc + x0] * w00;
  if (v01) v += p[(long)y0 * Wc + x1] * w01;
  if (v10) v += p[(long)y1 * Wc + x0] * w10;
  if (v11) v += p[(long)y1 * Wc + x1] * w11;
  float ss = v * v;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  if ((c & 31) == 0) red[c >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int wv = 0; wv < 8; ++wv) tot += red[wv];
  dd[c] = v * (1.f / fmaxf(sqrtf(tot), 1e-12f));
}

// the padded maps of the four resolutions H >> i, W >> i (1-pixel border)
void sp_levels(int B, int H, int W, TcRows lv[4]) {
  for (int i = 0; i < 4; ++i) lv[i] = tc_rows((long)B * ((H >> i) + 2) * ((W >> i) + 2));
}

}  // namespace

int kp_compact(const float* scores, int B, int H, int W, float thr, long cap, int* row_count, int* row_start, int* n_cand,
               int* cand_pos, float* cand_score, cudaStream_t stream) {
  const long rows = (long)B * H;
  sp_row_count_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(scores, row_count, rows, W, thr);
  sp_row_scan_kernel<<<B, 1024, 0, stream>>>(row_count, row_start, n_cand, H);
  sp_row_write_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(scores, row_start, cand_pos, cand_score, rows, H, W, thr, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("candidate compaction launch failed");
}
int kp_select_above_kth(const int* n_cand, const int* cand_pos, const float* cand_score, int* sel_pos, float* sel_score, int* n_sel,
                        int B, int k_max, long cap, long out_cap, cudaStream_t stream) {
  kp_select_above_kernel<<<B, 1024, 0, stream>>>(n_cand, cand_pos, cand_score, sel_pos, sel_score, n_sel, k_max, cap, out_cap);
  return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("top-k launch failed");
}

// SpCudaStages: the Stages policy of sp_run_post for the CUDA build of the tensor-core mode
int SpCudaStages::compact_impl(const SpWorkspace& ws, int B, int H, int W, float thr, long cap) const {
  return kp_compact(ws.t0, B, H, W, thr, cap, ws.row_count, ws.row_start, ws.n_cand, ws.cand_pos, ws.cand_score, stream);
}
int SpCudaStages::select_impl(const SpWorkspace& ws, int B, int k, long cap, long out_cap, int rank_all) const {
  sp_select_kernel<<<B, 1024, 0, stream>>>(ws.n_cand, ws.cand_pos, ws.cand_score, ws.sel_pos, ws.sel_score, ws.n_sel, k, cap, out_cap,
                                           rank_all);
  return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("superpoint: top-k launch failed");
}
int SpCudaStages::sample_impl(const SpWorkspace& ws, float* kpts, float* kscores, float* desc, int B, int Hc, int Wc,
                              long out_cap) const {
  if (out_cap <= 0) return 0;
  sp_sample_kernel<<<dim3((unsigned)out_cap, B), 256, 0, stream>>>(ws.n_sel, ws.sel_pos, ws.sel_score, ws.dense, kpts, kscores, desc,
                                                                   Hc, Wc, out_cap);
  return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("superpoint: descriptor sampling launch failed");
}

SpTcPlan sp_tc_plan(int B, int H, int W) {
  TcRows lv[4];
  sp_levels(B, H, W, lv);
  // Every write into the ping-pong images X / Y (conv1a, the poolings, the 3x3 convolutions) covers all 2 Lp rows of its
  // level, padding rows included, with Cout channels; the widest map at each level is 64, 64, 128 (conv3a, conv3b, the
  // third pooling, conv4a) and 256 channels (convPa, convDa).  On large images the full-resolution map is the largest, but
  // on small ones every level pads up to the same 256 rows and the 1/4- and 1/8-resolution maps outgrow it.
  const int xy_channels[4] = {64, 64, 128, 256};
  size_t xy = 0;
  for (int i = 0; i < 4; ++i) xy = std::max(xy, (size_t)lv[i].rows * xy_channels[i] * 2);
  const size_t bytes[SPT_NBUF] = {
      xy, xy, xy, xy,                    // X hi / lo, Y hi / lo
      (size_t)lv[3].rows * 128 * 2,      // features hi / lo (conv4b)
      (size_t)lv[3].rows * 128 * 2,
      (size_t)lv[3].rows * 96 * 4,       // logits fp32 [rows, 96] (convPb)
      (size_t)lv[3].rows * 256 * 4,      // dense descriptors fp32 [rows, 256] (convDb)
      64 * sizeof(int),                  // per-level (len[2], stop_layer[1])
  };
  SpTcPlan p{};
  size_t n = 0;
  for (int i = 0; i < SPT_NBUF; ++i) {
    n = (n + 1023) & ~(size_t)1023;
    p.off[i] = n;
    p.bytes[i] = bytes[i];
    n += bytes[i];
  }
  p.total = (n + 1023) & ~(size_t)1023;
  return p;
}

int sp_tc_create(TcConvWeights** out, const float* wts_dev, cudaStream_t stream) {
  TcConvRegion reg[11];
  for (int l = 1; l < 12; ++l) {
    const SpLayer& L = SP_LAYERS[l];
    const int taps = L.k * L.k;
    const float* w = wts_dev + sp_layer_offset(l);
    reg[l - 1] = {.w = w, .b = w + (size_t)L.cout * L.cin * taps, .cin = L.cin, .cpad = L.cin, .taps = taps, .rows = 256,
                  .K = taps * L.cin, .ncopy = L.cout};
  }
  return tc_conv_weights_create(out, reg, 11, stream);
}

// image [B,1,H,W] fp32 -> logits_nchw [B,65,H/8,W/8], dense_nchw [B,256,H/8,W/8] (un-normalised), fp32
int sp_tc_backbone(TcConvWeights* t, const float* wts_dev, const float* image, int B, int H, int W, void* workspace,
                   float* logits_nchw, float* dense_nchw, cudaStream_t stream) {
  TcRows lv[4];
  sp_levels(B, H, W, lv);
  const SpTcPlan plan = sp_tc_plan(B, H, W);
  char* base = (char*)workspace;
  auto at = [&](int buf) { return (__nv_bfloat16*)(base + plan.off[buf]); };
  __nv_bfloat16* X[2] = {at(SPT_XH), at(SPT_XL)};
  __nv_bfloat16* Y[2] = {at(SPT_YH), at(SPT_YL)};
  __nv_bfloat16* F[2] = {at(SPT_FH), at(SPT_FL)};
  float* logits_f = (float*)(base + plan.off[SPT_LOGITS]);
  float* dense_f = (float*)(base + plan.off[SPT_DENSE]);
  int* stw = (int*)(base + plan.off[SPT_STATE]);
  LG_RC(tc_rows_words(lv, 4, stw, stream));
  auto conv = [&](int l, int li, __nv_bfloat16** in, __nv_bfloat16** out, float* out_f32, int ldo, int relu) {
    const SpLayer& L = SP_LAYERS[l];
    return tc_conv(*t, tc_rows_state(lv[li], stw + 4 * li), {.in_h = in[0], .in_l = in[1], .cin = L.cin, .taps = L.k * L.k,
                   .region = l - 1, .relu = relu, .B = B, .H = H >> li, .W = W >> li, .out_h = out ? out[0] : nullptr,
                   .out_l = out ? out[1] : nullptr, .cout = L.cout, .out_f32 = out_f32, .ldo = ldo}, stream);
  };
  auto pool = [&](int li, int C, __nv_bfloat16** in, __nv_bfloat16** out) {  // level li -> li + 1
    const long n = lv[li + 1].rows * (C / 2);
    sp_pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(in[0], in[1], out[0], out[1], B, H >> li, W >> li, C,
                                                                   lv[li + 1].rows);
    return cudaGetLastError() == cudaSuccess ? 0 : lg_set_error("sp_pool_kernel launch failed");
  };
  int rc = 0;
  {  // conv1a on the CUDA cores (K = 9)
    const float* w = wts_dev + sp_layer_offset(0);
    const long n = lv[0].rows * 8;
    sp_conv1a_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(image, w, w + 64 * 9, X[0], X[1], B, H, W, lv[0].rows);
    if (cudaGetLastError() != cudaSuccess) return lg_set_error("sp_conv1a_kernel launch failed");
  }
  if ((rc = conv(1, 0, X, Y, nullptr, 0, 1))) return rc;
  if ((rc = pool(0, 64, Y, X))) return rc;
  if ((rc = conv(2, 1, X, Y, nullptr, 0, 1))) return rc;
  if ((rc = conv(3, 1, Y, X, nullptr, 0, 1))) return rc;
  if ((rc = pool(1, 64, X, Y))) return rc;
  if ((rc = conv(4, 2, Y, X, nullptr, 0, 1))) return rc;
  if ((rc = conv(5, 2, X, Y, nullptr, 0, 1))) return rc;
  if ((rc = pool(2, 128, Y, X))) return rc;
  if ((rc = conv(6, 3, X, Y, nullptr, 0, 1))) return rc;
  if ((rc = conv(7, 3, Y, F, nullptr, 0, 1))) return rc;            // shared features [rows3, 128]
  if ((rc = conv(8, 3, F, X, nullptr, 0, 1))) return rc;            // detector head (184-185)
  if ((rc = conv(9, 3, X, nullptr, logits_f, 96, 0))) return rc;
  if ((rc = conv(10, 3, F, Y, nullptr, 0, 1))) return rc;           // descriptor head (220-221)
  if ((rc = conv(11, 3, Y, nullptr, dense_f, 256, 0))) return rc;
  const int Hc = H / 8, Wc = W / 8;
  {
    const long n = (long)B * 65 * Hc * Wc;
    sp_to_nchw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(logits_f, 96, logits_nchw, B, 65, Hc, Wc);
    const long m = (long)B * 256 * Hc * Wc;
    sp_to_nchw_kernel<<<(unsigned)((m + 255) / 256), 256, 0, stream>>>(dense_f, 256, dense_nchw, B, 256, Hc, Wc);
    if (cudaGetLastError() != cudaSuccess) return lg_set_error("sp_to_nchw_kernel launch failed");
  }
  return 0;
}
