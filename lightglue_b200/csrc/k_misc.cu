// Non-GEMM kernels shared by every precision mode: keypoint normalisation + Fourier encoding,
// adaptive depth/width machinery (token confidence, stop vote, order-preserving compaction) and the
// assignment tail (dual-softmax log-assignment, mutual-nearest filter, output assembly).
// lightglue.py line numbers refer to /root/reference/lightglue/lightglue.py.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "block_scan.cuh"
#include "lg_internal.h"
#include "tc_common.cuh"

using tc::cluster_sync_all;

// ------------------------------------------------------------------------------------------------
// normalize_keypoints (31-43) + LearnableFourierPositionalEncoding (76-81)
// One CTA per (sequence); cos/sin stored once per frequency (the reference duplicates each over the
// adjacent channel pair with repeat_interleave(2); the consumer indexes freq = d / 2 instead).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) posenc_kernel(PosencArgs a) {
  const int s = blockIdx.x, S = 2 * a.B;
  const bool im1 = s >= a.B;
  const int b = im1 ? s - a.B : s;
  const int stride = im1 ? a.N : a.M;                  // rows per pair in the (padded) input slabs
  const int* lens = im1 ? a.lens1 : a.lens0;
  const int n = lens ? min(max(lens[b], 0), stride) : stride;
  const float* kp = (im1 ? a.kpts1 : a.kpts0) + (long)b * stride * 2;
  const float* size = im1 ? a.size1 : a.size0;
  const float* sc = im1 ? a.scales1 : a.scales0;
  const float* orr = im1 ? a.oris1 : a.oris0;
  __shared__ float red[4][8];
  __shared__ float sz[2];
  const int tid = threadIdx.x;
  if (size) {
    if (tid < 2) sz[tid] = size[b * 2 + tid];
  } else {  // size = 1 + max - min over the keypoints (35-36)
    float mx0 = -INFINITY, mx1 = -INFINITY, mn0 = INFINITY, mn1 = INFINITY;
    for (int i = tid; i < n; i += 256) {
      const float x = kp[i * 2], y = kp[i * 2 + 1];
      mx0 = fmaxf(mx0, x); mn0 = fminf(mn0, x); mx1 = fmaxf(mx1, y); mn1 = fminf(mn1, y);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off)); mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, off));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off)); mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, off));
    }
    if (tid % 32 == 0) { red[0][tid / 32] = mx0; red[1][tid / 32] = mn0; red[2][tid / 32] = mx1; red[3][tid / 32] = mn1; }
    __syncthreads();
    if (tid == 0) {
      float a0 = red[0][0], b0 = red[1][0], a1 = red[2][0], b1 = red[3][0];
      for (int w = 1; w < 8; ++w) {
        a0 = fmaxf(a0, red[0][w]); b0 = fminf(b0, red[1][w]); a1 = fmaxf(a1, red[2][w]); b1 = fminf(b1, red[3][w]);
      }
      sz[0] = 1.f + a0 - b0; sz[1] = 1.f + a1 - b1;
    }
  }
  __syncthreads();
  const float shx = sz[0] / 2.f, shy = sz[1] / 2.f, scale = fmaxf(sz[0], sz[1]) / 2.f;  // (40-41)
  float* out = a.cs + (long)s * a.Lp * 64;
  (void)S;
  // the rows of a sequence are spread over gridDim.y CTAs (each repeats the cheap bounding-box reduction above)
  for (int e = blockIdx.y * 256 + tid; e < n * 32; e += 256 * gridDim.y) {
    const int i = e / 32, f = e % 32;
    const float x = (kp[i * 2] - shx) / scale, y = (kp[i * 2 + 1] - shy) / scale;  // (42)
    const float* w = a.wr + f * a.pos_dim;
    float pr = x * w[0] + y * w[1];
    if (a.pos_dim == 4) pr += sc[(long)b * stride + i] * w[2] + orr[(long)b * stride + i] * w[3];  // (495-501)
    float sn, cs;
    sincosf(pr, &sn, &cs);
    out[(long)i * 64 + f] = cs;
    out[(long)i * 64 + 32 + f] = sn;
  }
}

int misc_posenc(const PosencArgs& a, cudaStream_t stream) {
  const int mx = a.M > a.N ? a.M : a.N;
  int chunks = (mx * 32 + 256 * 16 - 1) / (256 * 16);  // ~16 encodings per thread
  if (chunks < 1) chunks = 1;
  if (chunks > 64) chunks = 64;
  posenc_kernel<<<dim3(2 * a.B, chunks), 256, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}

__global__ void pack_desc_kernel(const float* __restrict__ d0, const float* __restrict__ d1, float* __restrict__ out, int B,
                                 int M, int N, int Lp, int d, const int* __restrict__ lens0, const int* __restrict__ lens1,
                                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int s = blockIdx.y, r = blockIdx.x;
  const bool im1 = s >= B;
  const int* lens = im1 ? lens1 : lens0;
  const int n = lens ? min(lens[im1 ? s - B : s], im1 ? N : M) : (im1 ? N : M);
  if (r >= n) return;
  const float* src = (im1 ? d1 + ((long)(s - B) * N + r) * d : d0 + ((long)s * M + r) * d);
  float* dst = out + ((long)s * Lp + r) * d;
  for (int c = threadIdx.x * 4; c < d; c += blockDim.x * 4) {
    const float4 t = *reinterpret_cast<const float4*>(src + c);
    *reinterpret_cast<float4*>(dst + c) = t;
    if (hi) {  // bf16 hi (/ lo) images for the tensor-core linears, written in the same pass
      const __nv_bfloat162 h0 = __floats2bfloat162_rn(t.x, t.y), h1 = __floats2bfloat162_rn(t.z, t.w);
      const long o = ((long)s * Lp + r) * d + c;
      *reinterpret_cast<__nv_bfloat162*>(hi + o) = h0;
      *reinterpret_cast<__nv_bfloat162*>(hi + o + 2) = h1;
      if (lo) {
        *reinterpret_cast<__nv_bfloat162*>(lo + o) =
            __floats2bfloat162_rn(t.x - __bfloat162float(h0.x), t.y - __bfloat162float(h0.y));
        *reinterpret_cast<__nv_bfloat162*>(lo + o + 2) =
            __floats2bfloat162_rn(t.z - __bfloat162float(h1.x), t.w - __bfloat162float(h1.y));
      }
    }
  }
}

int misc_pack_desc(const float* d0, const float* d1, float* out, int B, int M, int N, int Lp, int d, const int* lens0,
                   const int* lens1, cudaStream_t stream, void* hi, void* lo) {
  const int mx = M > N ? M : N;
  if (mx == 0) return 0;
  pack_desc_kernel<<<dim3(mx, 2 * B), 64, 0, stream>>>(d0, d1, out, B, M, N, Lp, d, lens0, lens1, (__nv_bfloat16*)hi,
                                                       (__nv_bfloat16*)lo);
  LG_CHECK_LAUNCH();
  return 0;
}

__global__ void init_state_kernel(int* len, int* ind, int* prune, int* stop_layer, int* below, int n_below, int B, int M,
                                  int N, int Lp, const int* lens0, const int* lens1) {
  const int s = blockIdx.x;
  const int b = s >= B ? s - B : s;
  const int l0 = lens0 ? min(max(lens0[b], 0), M) : M, l1 = lens1 ? min(max(lens1[b], 0), N) : N;
  const int mylen = s >= B ? l1 : l0;
  if (threadIdx.x == 0) {
    len[s] = mylen;
    if (s < B) stop_layer[s] = (l0 == 0 || l1 == 0) ? 1 : 0;  // an empty image: the pair never runs (568-588)
  }
  if (s == 0)
    for (int i = threadIdx.x; i < n_below; i += blockDim.x) below[i] = 0;
  for (int r = threadIdx.x; r < Lp; r += blockDim.x) {
    ind[(long)s * Lp + r] = r;
    prune[(long)s * Lp + r] = r < mylen ? 1 : 0;  // torch.ones_like(ind) (535-536); padding rows report 0
  }
}

int misc_init_state(int* len, int* ind, int* prune, int* stop_layer, int* below, int n_below, int B, int M, int N, int Lp,
                    const int* lens0, const int* lens1, cudaStream_t stream) {
  init_state_kernel<<<2 * B, 256, 0, stream>>>(len, ind, prune, stop_layer, below, n_below, B, M, N, Lp, lens0, lens1);
  LG_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Adaptive depth / width.  score: one warp per token computes token confidence (84-94) and
// matchability (298-299), the keep flag of get_pruning_mask (636-643) and the per-pair count of
// low-confidence tokens for check_if_stop (645-656).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_dot256(const float* __restrict__ x, const float* __restrict__ w, int lane) {
  const float4 a0 = *reinterpret_cast<const float4*>(x + lane * 8), a1 = *reinterpret_cast<const float4*>(x + lane * 8 + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(w + lane * 8), b1 = *reinterpret_cast<const float4*>(w + lane * 8 + 4);
  float acc = a0.x * b0.x;
  acc = fmaf(a0.y, b0.y, acc); acc = fmaf(a0.z, b0.z, acc); acc = fmaf(a0.w, b0.w, acc);
  acc = fmaf(a1.x, b1.x, acc); acc = fmaf(a1.y, b1.y, acc); acc = fmaf(a1.z, b1.z, acc); acc = fmaf(a1.w, b1.w, acc);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  return acc;
}
__device__ __forceinline__ float sigmoidf_(float z) { return 1.f / (1.f + expf(-z)); }

__global__ void __launch_bounds__(256) adapt_score_kernel(AdaptArgs a, SeqState st) {
  const int s = blockIdx.y;
  const int r = blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int pair = s >= st.B ? s - st.B : s;
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  const bool live = r < st.len[s] && st.stop_layer[pair] == 0;
  if (live) {
    const float* x = a.x + ((long)s * st.Lp + r) * LG_DIM;
    bool keep = true, below = false;
    float conf = 0.f;
    if (a.tok_w) {
      conf = sigmoidf_(warp_dot256(x, a.tok_w, lane) + a.tok_b[0]);
      below = conf < a.thr;
    }
    if (a.mat_w) {
      const float mt = sigmoidf_(warp_dot256(x, a.mat_w, lane) + a.mat_b[0]);
      keep = mt > (1.f - a.width_conf);
      if (a.tok_w) keep = keep || (conf <= a.thr);  // low-confidence points are never pruned (641-642)
    }
    if (lane == 0) {
      a.keep[(long)s * st.Lp + r] = keep ? 1 : 0;
      if (below) atomicAdd(&cnt, 1);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && cnt) atomicAdd(a.below + pair, cnt);
}

int misc_adapt_score(const AdaptArgs& a, const SeqState& st, cudaStream_t stream) {
  adapt_score_kernel<<<dim3(st.Lp / 8, st.S), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  return 0;
}

// decide: one CTA per sequence.  Evaluates the stop vote for the pair (both of its CTAs reach the
// same verdict from the same counter), and if the pair continues and this image still has more
// than `pruning_threshold` points, an order-preserving exclusive scan of the keep flags
// (== torch.where(mask)[1] order, 554/562).  Otherwise the identity map.
__global__ void __launch_bounds__(1024) adapt_decide_kernel(AdaptArgs a, SeqState st) {
  const int s = blockIdx.x;
  const int pair = s >= st.B ? s - st.B : s;
  const int len = a.len_in[s];
  const int tid = threadIdx.x;
  const int prev = st.stop_layer[pair];
  // original sizes of the pair (ragged batches carry them per pair); an empty image never runs a layer
  const int m0 = a.lens0 ? min(max(a.lens0[pair], 0), a.M) : a.M, n0 = a.lens1 ? min(max(a.lens1[pair], 0), a.N) : a.N;
  const bool was_active = m0 > 0 && n0 > 0 && ((prev == 0) || (prev == a.layer + 1));  // the sibling CTA may already have voted
  bool stop = false;
  if (was_active && a.tok_w) {
    // ratio_confident = 1 - (#conf < thr) / (m + n) > depth_confidence  (655-656); denominator is the
    // ORIGINAL m + n, numerator counts surviving points only (549)
    const float ratio = 1.0f - (float)a.below[pair] / (float)(m0 + n0);
    stop = ratio > a.depth_conf;
  }
  const bool do_prune = was_active && !stop && a.mat_w && len > a.pruning_threshold;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  // pairs that exited earlier still run the (identity) scan: the host ping-pongs the token buffers
  // every layer, so their rows must keep travelling with everyone else's.
  const unsigned char* keep = a.keep + (long)s * st.Lp;
  int* pos = a.pos + (long)s * st.Lp;
  for (int base = 0; base < len; base += 1024) {
    const int r = base + tid;
    const int flag = (r < len) ? (do_prune ? (int)keep[r] : 1) : 0;
    int incl = flag;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, off);
      if ((tid & 31) >= off) incl += t;
    }
    if ((tid & 31) == 31) warp_sums[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
      int w = warp_sums[tid];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, off);
        if (tid >= off) w += t;
      }
      warp_sums[tid] = w;  // inclusive over warps
    }
    __syncthreads();
    const int warp_off = (tid >> 5) ? warp_sums[(tid >> 5) - 1] : 0;
    const int c = carry;
    if (r < len) pos[r] = flag ? (c + warp_off + incl - 1) : -1;
    __syncthreads();
    if (tid == 0) carry = c + warp_sums[31];
    __syncthreads();
  }
  if (tid == 0) {
    a.len_out[s] = carry;
    a.did_prune[s] = do_prune ? 1 : 0;
    if (stop) a.stop_layer[pair] = a.layer + 1;
  }
}

int misc_adapt_decide(const AdaptArgs& a, const SeqState& st, cudaStream_t stream) {
  adapt_decide_kernel<<<st.S, 1024, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  return 0;
}

// gather: one warp per source row; moves the residual stream, the cached encoding (557/565) and the
// original-index map (555/563) to their compacted position; bumps the prune counters (558/566).
__global__ void __launch_bounds__(256) adapt_gather_kernel(GatherArgs a, SeqState st) {
  const int s = blockIdx.y;
  const int r = blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (blockIdx.x == 0 && threadIdx.x == 0 && s < st.B) {
    // pruning left one image of the pair without points: the reference breaks out at the top of the next layer
    // (539-540) and answers from its empty branch (568-588) with stop = (layer + 1) + 1; nothing matches
    if (a.stop_layer[s] == 0 && (a.len_out[s] == 0 || a.len_out[s + st.B] == 0)) a.stop_layer[s] = a.layer + 2;
  }
  if (r >= a.len_in[s]) return;
  const int dst = a.pos[(long)s * st.Lp + r];
  if (dst < 0) return;
  const long src_row = (long)s * st.Lp + r, dst_row = (long)s * st.Lp + dst;
  const float4* xs = reinterpret_cast<const float4*>(a.x_in + src_row * LG_DIM);
  float4* xd = reinterpret_cast<float4*>(a.x_out + dst_row * LG_DIM);
  xd[lane] = xs[lane];
  xd[lane + 32] = xs[lane + 32];
  if (lane < 16)
    reinterpret_cast<float4*>(a.cs_out + dst_row * 64)[lane] = reinterpret_cast<const float4*>(a.cs_in + src_row * 64)[lane];
  if (lane == 0) {
    const int orig = a.ind_in[src_row];
    a.ind_out[dst_row] = orig;
    if (a.did_prune[s]) a.prune[(long)s * st.Lp + orig] += 1;
  }
}

int misc_adapt_gather(const GatherArgs& a, const SeqState& st, cudaStream_t stream) {
  adapt_gather_kernel<<<dim3(st.Lp / 8, st.S), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  return 0;
}

__global__ void finalize_stop_kernel(int* stop_layer, int B, int n_layers) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B && stop_layer[i] == 0) stop_layer[i] = n_layers;
}
int misc_finalize_stop(int* stop_layer, int B, int n_layers, cudaStream_t stream) {
  finalize_stop_kernel<<<(B + 255) / 256, 256, 0, stream>>>(stop_layer, B, n_layers);
  LG_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Assignment tail.  score[i,j] = 2 S[i,j] - LSE_j S[i,:] - LSE_i S[:,j] + logsig(z0_i) + logsig(z1_j)
// (closed form of sigmoid_log_double_softmax, 265-277).  Two sweeps over 64x64 tiles of S = p0 p1^T:
//   sweep 1: per-tile row / column (max, sum-exp) partials      -> combine -> LSE vectors
//   sweep 2: recompute the tile, form the score, per-tile row / column arg-max partials
//            (optionally stream the score matrix out)            -> combine -> mutual filter
// No atomics: every partial has its own slot, so results are run-to-run deterministic.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) assign_z_kernel(AssignArgs a, SeqState st) {
  const int s = blockIdx.y;
  const int r = blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= st.len[s]) return;
  const int pair = s >= st.B ? s - st.B : s;
  const long sel = a.mat_sel_stride > 0 ? (long)(st.stop_layer[pair] - 1) : 0;
  const float* w = a.mat_w + sel * a.mat_sel_stride;
  const float* bb = a.mat_b + sel * a.mat_sel_stride;
  const float z = warp_dot256(a.x + ((long)s * st.Lp + r) * LG_DIM, w, lane) + bb[0];
  if (lane == 0) a.z[(long)s * st.Lp + r] = z;
}

__device__ __forceinline__ float logsigmoidf_(float z) {  // F.logsigmoid: min(z,0) - log1p(exp(-|z|))
  return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}

template <int SWEEP>
__global__ void __launch_bounds__(256) assign_sweep_kernel(AssignArgs a, SeqState st) {
  const int b = blockIdx.z;
  const int ti = blockIdx.y, tj = blockIdx.x;
  const int m = st.len[b], n = st.len[b + st.B];
  const int i0 = ti * 64, j0 = tj * 64;
  if (i0 >= m || j0 >= n) return;
  __shared__ float As[16][68];
  __shared__ float Bs[16][68];
  __shared__ float redv[64][17];
  __shared__ int redi[64][17];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int lr = tid / 4, lk = (tid % 4) * 4;
  const float* p0 = a.p + ((long)b * st.Lp + i0) * LG_DIM;
  const float* p1 = a.p + ((long)(b + st.B) * st.Lp + j0) * LG_DIM;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < LG_DIM; k0 += 16) {
    const float4 av = *reinterpret_cast<const float4*>(p0 + (long)lr * LG_DIM + k0 + lk);
    const float4 bv = *reinterpret_cast<const float4*>(p1 + (long)lr * LG_DIM + k0 + lk);
    As[lk + 0][lr] = av.x; As[lk + 1][lr] = av.y; As[lk + 2][lr] = av.z; As[lk + 3][lr] = av.w;
    Bs[lk + 0][lr] = bv.x; Bs[lk + 1][lr] = bv.y; Bs[lk + 2][lr] = bv.z; Bs[lk + 3][lr] = bv.w;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float af[4], bf[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) af[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bf[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(af[i], bf[j], acc[i][j]);
    }
    __syncthreads();
  }
  const long rbase = (long)b * st.Lp;
  if (SWEEP == 1) {
    // rows: (max, sumexp) over this tile's valid columns
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j0 + tx * 4 + j < n) mx = fmaxf(mx, acc[i][j]);
#pragma unroll
      for (int off = 1; off < 16; off <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float se = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j0 + tx * 4 + j < n) se += expf(acc[i][j] - mx);
#pragma unroll
      for (int off = 1; off < 16; off <<= 1) se += __shfl_xor_sync(0xffffffffu, se, off);
      const int r = i0 + ty * 4 + i;
      if (tx == 0 && r < m) {
        float* o = a.rowpart + ((rbase + r) * a.nt + tj) * 2;
        o[0] = mx; o[1] = se;
      }
    }
    // columns: reduce over the 16 ty groups through shared memory
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 4; ++i) if (i0 + ty * 4 + i < m) mx = fmaxf(mx, acc[i][j]);
      redv[tx * 4 + j][ty] = mx;
    }
    __syncthreads();
    float cmx = -INFINITY;
    if (tid < 64) {
#pragma unroll
      for (int t = 0; t < 16; ++t) cmx = fmaxf(cmx, redv[tid][t]);
    }
    __syncthreads();
    if (tid < 64) redv[tid][16] = cmx;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float cm = redv[tx * 4 + j][16];
      float se = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) if (i0 + ty * 4 + i < m) se += expf(acc[i][j] - cm);
      redv[tx * 4 + j][ty] = se;
    }
    __syncthreads();
    if (tid < 64 && j0 + tid < n) {
      float se = 0.f;
#pragma unroll
      for (int t = 0; t < 16; ++t) se += redv[tid][t];
      float* o = a.colpart + ((rbase + j0 + tid) * a.nt + ti) * 2;
      o[0] = cmx; o[1] = se;
    }
  } else {
    const float* z0 = a.z + rbase;
    const float* z1 = a.z + (long)(b + st.B) * st.Lp;
    float cterm[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = j0 + tx * 4 + j;
      cterm[j] = c < n ? logsigmoidf_(z1[c]) - a.collse[rbase + c] : 0.f;
    }
    float sc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = i0 + ty * 4 + i;
      const float rterm = r < m ? logsigmoidf_(z0[r]) - a.rowlse[rbase + r] : 0.f;
      float best = -INFINITY; int arg = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = j0 + tx * 4 + j;
        const float v = (r < m && c < n) ? 2.f * acc[i][j] + rterm + cterm[j] : -INFINITY;
        sc[i][j] = v;
        if (v > best) { best = v; arg = c; }
      }
#pragma unroll
      for (int off = 1; off < 16; off <<= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, off);
        if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
      }
      if (tx == 0 && r < m) {
        a.rowbest[(rbase + r) * a.nt + tj] = best;
        a.rowarg[(rbase + r) * a.nt + tj] = arg;
      }
      if (a.log_assignment && r < m) {
        float* o = a.log_assignment + ((long)b * (a.M + 1) + r) * (a.N + 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) if (j0 + tx * 4 + j < n) o[j0 + tx * 4 + j] = sc[i][j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float best = -INFINITY; int arg = 0x7fffffff;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (sc[i][j] > best) { best = sc[i][j]; arg = i0 + ty * 4 + i; }
      }
      redv[tx * 4 + j][ty] = best; redi[tx * 4 + j][ty] = arg;
    }
    __syncthreads();
    if (tid < 64 && j0 + tid < n) {
      float best = -INFINITY; int arg = 0x7fffffff;
#pragma unroll
      for (int t = 0; t < 16; ++t) {  // ty ascending == row index ascending: first max wins ties
        if (redv[tid][t] > best) { best = redv[tid][t]; arg = redi[tid][t]; }
      }
      a.colbest[(rbase + j0 + tid) * a.nt + ti] = best;
      a.colarg[(rbase + j0 + tid) * a.nt + ti] = arg;
    }
  }
}

// combine per-tile partials.  mode 1: (max,sumexp) -> LSE;  mode 2: (best,arg) -> slot 0
__global__ void assign_combine_kernel(AssignArgs a, SeqState st, int mode) {
  const int b = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = st.len[b], n = st.len[b + st.B];
  const long rbase = (long)b * st.Lp;
  const int ntr = (n + 63) / 64, ntc = (m + 63) / 64;  // tiles a row spans / tiles a column spans
  if (mode == 1) {
    if (idx < m) {
      const float* pt = a.rowpart + (rbase + idx) * a.nt * 2;
      float mx = -INFINITY;
      for (int t = 0; t < ntr; ++t) mx = fmaxf(mx, pt[t * 2]);
      float se = 0.f;
      for (int t = 0; t < ntr; ++t) se += pt[t * 2 + 1] * expf(pt[t * 2] - mx);
      a.rowlse[rbase + idx] = mx + logf(se);
    }
    if (idx < n) {
      const float* pt = a.colpart + (rbase + idx) * a.nt * 2;
      float mx = -INFINITY;
      for (int t = 0; t < ntc; ++t) mx = fmaxf(mx, pt[t * 2]);
      float se = 0.f;
      for (int t = 0; t < ntc; ++t) se += pt[t * 2 + 1] * expf(pt[t * 2] - mx);
      a.collse[rbase + idx] = mx + logf(se);
    }
  } else {
    if (idx < m) {
      float best = -INFINITY; int arg = 0;
      for (int t = 0; t < ntr; ++t) {
        const float v = a.rowbest[(rbase + idx) * a.nt + t];
        if (v > best) { best = v; arg = a.rowarg[(rbase + idx) * a.nt + t]; }
      }
      a.rowbest[(rbase + idx) * a.nt] = best; a.rowarg[(rbase + idx) * a.nt] = arg;
    }
    if (idx < n) {
      float best = -INFINITY; int arg = 0;
      for (int t = 0; t < ntc; ++t) {
        const float v = a.colbest[(rbase + idx) * a.nt + t];
        if (v > best) { best = v; arg = a.colarg[(rbase + idx) * a.nt + t]; }
      }
      a.colbest[(rbase + idx) * a.nt] = best; a.colarg[(rbase + idx) * a.nt] = arg;
    }
  }
}

// filter_matches (302-318) in the compact index space: row/column `idx` of pair b
__device__ __forceinline__ void assign_filter_one(const AssignArgs& a, const SeqState& st, int b, int idx) {
  const int m = st.len[b], n = st.len[b + st.B];
  const long rbase = (long)b * st.Lp;
  if (m == 0 || n == 0) {  // an empty image: nothing to match against (568-588); the arg-max slots hold no data
    if (idx < m) { a.ms0c[rbase + idx] = 0.f; a.m0c[rbase + idx] = -1; }
    if (idx < n) { a.ms1c[rbase + idx] = 0.f; a.m1c[rbase + idx] = -1; }
    return;
  }
  if (idx < m) {
    const int j = a.rowarg[(rbase + idx) * a.nt];
    const bool mutual = a.colarg[(rbase + j) * a.nt] == idx;
    const float sc = mutual ? expf(a.rowbest[(rbase + idx) * a.nt]) : 0.f;
    a.ms0c[rbase + idx] = sc;
    a.m0c[rbase + idx] = (mutual && sc > a.filter_threshold) ? j : -1;
  }
  if (idx < n) {
    const int i = a.colarg[(rbase + idx) * a.nt];
    const int ji = a.rowarg[(rbase + i) * a.nt];
    const bool mutual1 = ji == idx;                       // m0[m1[j]] == j
    const bool mutual0_i = a.colarg[(rbase + ji) * a.nt] == i;  // mutual0 at i
    const float s0 = mutual0_i ? expf(a.rowbest[(rbase + i) * a.nt]) : 0.f;
    const float sc = mutual1 ? s0 : 0.f;
    const bool valid0_i = mutual0_i && s0 > a.filter_threshold;
    a.ms1c[rbase + idx] = sc;
    a.m1c[rbase + idx] = (mutual1 && valid0_i) ? i : -1;
  }
}
__global__ void assign_filter_kernel(AssignArgs a, SeqState st) {
  assign_filter_one(a, st, blockIdx.y, blockIdx.x * blockDim.x + threadIdx.x);
}

// dustbin row / column and corner of the materialised matrix (275-276)
__global__ void assign_dustbin_kernel(AssignArgs a, SeqState st) {
  const int b = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  float* o = a.log_assignment + (long)b * (a.M + 1) * (a.N + 1);
  if (idx < a.M) o[(long)idx * (a.N + 1) + a.N] = logsigmoidf_(-a.z[(long)b * st.Lp + idx]);
  if (idx < a.N) o[(long)a.M * (a.N + 1) + idx] = logsigmoidf_(-a.z[(long)(b + st.B) * st.Lp + idx]);
  if (idx == 0) o[(long)a.M * (a.N + 1) + a.N] = 0.f;
}

// the compact `matches` / `scores` lists (593-602): ordered compaction of the valid rows of pair b by one 1024-thread block
__device__ __forceinline__ void assign_compact_pair(const AssignArgs& a, const SeqState& st, int b, int tid) {
  const int m = st.len[b];
  const long rbase = (long)b * st.Lp;
  const int* ind0 = a.ind + rbase;
  const int* ind1 = a.ind + (long)(b + st.B) * st.Lp;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < m; base += 1024) {
    const int i = base + tid;
    int j = -1; float sc = 0.f;
    if (i < m) { j = a.m0c[rbase + i]; sc = a.ms0c[rbase + i]; }
    const int slot = block_scan_step(j >= 0, tid, warp_sums, &carry);
    if (j >= 0 && slot < a.cap) {
      a.matches[((long)b * a.cap + slot) * 2] = ind0[i];
      a.matches[((long)b * a.cap + slot) * 2 + 1] = ind1[j];
      a.match_scores[(long)b * a.cap + slot] = sc;
    }
  }
  if (tid == 0) a.n_matches[b] = carry;
}

// scatter back to the original indexing (605-614) + the compact lists
__global__ void __launch_bounds__(1024) assign_output_kernel(AssignArgs a, SeqState st) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int m = st.len[b], n = st.len[b + st.B];
  const long rbase = (long)b * st.Lp;
  const int* ind0 = a.ind + rbase;
  const int* ind1 = a.ind + (long)(b + st.B) * st.Lp;
  for (int i = tid; i < a.M; i += 1024) { a.matches0[(long)b * a.M + i] = -1; a.mscores0[(long)b * a.M + i] = 0.f; }
  for (int j = tid; j < a.N; j += 1024) { a.matches1[(long)b * a.N + j] = -1; a.mscores1[(long)b * a.N + j] = 0.f; }
  __syncthreads();
  for (int j = tid; j < n; j += 1024) {
    const int i = a.m1c[rbase + j];
    a.matches1[(long)b * a.N + ind1[j]] = i < 0 ? -1 : ind0[i];
    a.mscores1[(long)b * a.N + ind1[j]] = a.ms1c[rbase + j];
  }
  for (int i = tid; i < m; i += 1024) {
    const int j = a.m0c[rbase + i];
    a.matches0[(long)b * a.M + ind0[i]] = j < 0 ? -1 : ind1[j];
    a.mscores0[(long)b * a.M + ind0[i]] = a.ms0c[rbase + i];
  }
  assign_compact_pair(a, st, b, tid);
}

// ---- the tensor-core sweeps' companions: two launches instead of five --------------------------------------------
// After sweep 1: matchability logit z (281-285) and term = logsigmoid(z) - LSE (270-274), one warp per row; the LSE comes
// from the per-slot (max, sum-exp) partials the sweep wrote (`slot_cols` columns of the partner image per slot).
__global__ void __launch_bounds__(256) assign_term_kernel(AssignArgs a, SeqState st, const float2* __restrict__ part,
                                                          int pstride, int slot_cols, float* __restrict__ term) {
  const int s = blockIdx.y;
  const int r = blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= st.len[s]) return;
  const int pair = s >= st.B ? s - st.B : s;
  const int partner = s >= st.B ? s - st.B : s + st.B;
  const long sel = a.mat_sel_stride > 0 ? (long)(st.stop_layer[pair] - 1) : 0;
  const long row = (long)s * st.Lp + r;
  const float z = warp_dot256(a.x + row * LG_DIM, a.mat_w + sel * a.mat_sel_stride, lane) + (a.mat_b + sel * a.mat_sel_stride)[0];
  const int nt = (st.len[partner] + slot_cols - 1) / slot_cols;
  const float2* pt = part + row * pstride;
  float mx = -INFINITY;
  for (int t = lane; t < nt; t += 32) mx = fmaxf(mx, pt[t].x);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  float se = 0.f;
  for (int t = lane; t < nt; t += 32) se += pt[t].y * expf(pt[t].x - mx);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) se += __shfl_xor_sync(0xffffffffu, se, off);
  if (lane == 0) {
    a.z[row] = z;
    term[row] = logsigmoidf_(z) - (mx + logf(se));
  }
}

// After sweep 2: everything from the per-slot (best, arg) partials to the outputs, one cluster of 8 CTAs per pair.
//   phase A (all CTAs)  reduce the slots of every row / column; pre-fill the outputs with "unmatched"
//   phase B (all CTAs)  mutual-nearest filter + scatter to the original indexing
//   phase C (CTA 0)     ordered compaction into the `matches` / `scores` lists
// cluster barriers (release/acquire at cluster scope) order the global-memory hand-offs between the phases.
constexpr int TAIL_CLUSTER = 8;
__global__ void __cluster_dims__(TAIL_CLUSTER, 1, 1) __launch_bounds__(1024)
assign_tail_kernel(AssignArgs a, SeqState st, const float* __restrict__ part, const int* __restrict__ part_arg, int pstride,
                   int slot_cols) {
  const int b = blockIdx.x / TAIL_CLUSTER, rank = blockIdx.x % TAIL_CLUSTER, tid = threadIdx.x;
  const int gtid = rank * 1024 + tid, gsz = TAIL_CLUSTER * 1024;
  const int m = st.len[b], n = st.len[b + st.B];
  const long rbase = (long)b * st.Lp;
  const int* ind0 = a.ind + rbase;
  const int* ind1 = a.ind + (long)(b + st.B) * st.Lp;
  if (m > 0 && n > 0) {
    for (int side = 0; side < 2; ++side) {
      const int s = b + side * st.B, len = side ? n : m;
      const int nt = ((side ? m : n) + slot_cols - 1) / slot_cols;
      float* obest = side ? a.colbest : a.rowbest;
      int* oarg = side ? a.colarg : a.rowarg;
      for (int r = gtid; r < len; r += gsz) {
        const long base = ((long)s * st.Lp + r) * pstride;
        float best = -INFINITY; int arg = 0;
        for (int t = 0; t < nt; ++t)
          if (part[base + t] > best) { best = part[base + t]; arg = part_arg[base + t]; }
        obest[(rbase + r) * a.nt] = best; oarg[(rbase + r) * a.nt] = arg;
      }
    }
  }
  for (int i = gtid; i < a.M; i += gsz) { a.matches0[(long)b * a.M + i] = -1; a.mscores0[(long)b * a.M + i] = 0.f; }
  for (int j = gtid; j < a.N; j += gsz) { a.matches1[(long)b * a.N + j] = -1; a.mscores1[(long)b * a.N + j] = 0.f; }
  cluster_sync_all();
  const int mx = m > n ? m : n;
  for (int idx = gtid; idx < mx; idx += gsz) {
    assign_filter_one(a, st, b, idx);
    if (idx < m) {
      const int j = a.m0c[rbase + idx];
      a.matches0[(long)b * a.M + ind0[idx]] = j < 0 ? -1 : ind1[j];
      a.mscores0[(long)b * a.M + ind0[idx]] = a.ms0c[rbase + idx];
    }
    if (idx < n) {
      const int i = a.m1c[rbase + idx];
      a.matches1[(long)b * a.N + ind1[idx]] = i < 0 ? -1 : ind0[i];
      a.mscores1[(long)b * a.N + ind1[idx]] = a.ms1c[rbase + idx];
    }
  }
  cluster_sync_all();
  if (rank == 0) assign_compact_pair(a, st, b, tid);
}

int misc_assign_dustbin(const AssignArgs& a, const SeqState& st, cudaStream_t stream) {
  const int mx = a.M > a.N ? a.M : a.N;
  assign_dustbin_kernel<<<dim3((mx + 256) / 256, st.B), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  return 0;
}

int misc_assign_term(const AssignArgs& a, const SeqState& st, const float* part, int pstride, int slot_cols, float* term,
                     cudaStream_t stream) {
  assign_term_kernel<<<dim3(st.Lp / 8, st.S), 256, 0, stream>>>(a, st, reinterpret_cast<const float2*>(part), pstride, slot_cols, term);
  LG_CHECK_LAUNCH();
  return 0;
}

int misc_assign_tail(const AssignArgs& a, const SeqState& st, const float* part, const int* part_arg, int pstride, int slot_cols,
                     cudaStream_t stream) {
  assign_tail_kernel<<<st.B * TAIL_CLUSTER, 1024, 0, stream>>>(a, st, part, part_arg, pstride, slot_cols);
  LG_CHECK_LAUNCH();
  return 0;
}

int misc_assign(const AssignArgs& a, const SeqState& st, cudaStream_t stream) {
  const int B = st.B;
  const int tiles = st.Lp / 64;
  assign_z_kernel<<<dim3(st.Lp / 8, st.S), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  assign_sweep_kernel<1><<<dim3(tiles, tiles, B), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  assign_combine_kernel<<<dim3((st.Lp + 255) / 256, B), 256, 0, stream>>>(a, st, 1);
  LG_CHECK_LAUNCH();
  assign_sweep_kernel<2><<<dim3(tiles, tiles, B), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  assign_combine_kernel<<<dim3((st.Lp + 255) / 256, B), 256, 0, stream>>>(a, st, 2);
  LG_CHECK_LAUNCH();
  assign_filter_kernel<<<dim3((st.Lp + 255) / 256, B), 256, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  if (a.log_assignment) {
    const int mx = a.M > a.N ? a.M : a.N;
    assign_dustbin_kernel<<<dim3((mx + 256) / 256, B), 256, 0, stream>>>(a, st);
    LG_CHECK_LAUNCH();
  }
  assign_output_kernel<<<B, 1024, 0, stream>>>(a, st);
  LG_CHECK_LAUNCH();
  return 0;
}

__global__ void export_stop_prune_kernel(const int* stop_layer, const int* prune, int* stop_out, int* prune0, int* prune1, int B,
                                         int M, int N, int Lp) {
  const int s = blockIdx.x;
  const bool im1 = s >= B;
  const int b = im1 ? s - B : s;
  if (!im1 && threadIdx.x == 0 && stop_out) stop_out[b] = stop_layer[b];
  int* dst = im1 ? prune1 : prune0;
  if (!dst) return;
  const int n = im1 ? N : M;
  for (int r = threadIdx.x; r < n; r += blockDim.x) dst[(long)b * n + r] = prune[(long)s * Lp + r];
}
int misc_export_stop_prune(const int* stop_layer, const int* prune, int* stop_out, int* prune0, int* prune1, int B, int M,
                           int N, int Lp, cudaStream_t stream) {
  export_stop_prune_kernel<<<2 * B, 256, 0, stream>>>(stop_layer, prune, stop_out, prune0, prune1, B, M, N, Lp);
  LG_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// lg_attention plumbing (kernel-level entry point): reference head layout <-> kernel operand layouts
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) attn_pack_kernel(AttnIoArgs a) {
  const int r = blockIdx.x, hh = blockIdx.y, s = blockIdx.z, d = threadIdx.x;
  const bool im1 = s >= a.B;
  const int b = im1 ? s - a.B : s, n = im1 ? a.N : a.M;
  if (r >= n) return;
  const long src = (((long)b * LG_HEADS + hh) * n + r) * LG_HDIM + d;
  const float q = (im1 ? a.q1 : a.q0)[src], k = (im1 ? a.k1 : a.k0)[src], v = (im1 ? a.v1 : a.v0)[src];
  const long sh = (long)s * LG_HEADS + hh;
  const long dst = (sh * a.Lp + r) * LG_HDIM + d;
  if (a.qf) { a.qf[dst] = q; a.kf[dst] = k; a.vf[dst] = v; }
  if (a.qh) {
    reinterpret_cast<__half*>(a.qh)[dst] = __float2half_rn(q);
    reinterpret_cast<__half*>(a.kh)[dst] = __float2half_rn(k);
    reinterpret_cast<__half*>(a.vth)[(sh * LG_HDIM + d) * a.Lp + r] = __float2half_rn(v);
  }
}
int misc_attn_pack(const AttnIoArgs& a, cudaStream_t stream) {
  const int mx = a.M > a.N ? a.M : a.N;
  attn_pack_kernel<<<dim3(mx, LG_HEADS, 2 * a.B), 64, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}

__global__ void __launch_bounds__(256) attn_unpack_kernel(AttnIoArgs a) {
  const int r = blockIdx.x, s = blockIdx.y, c = threadIdx.x;
  const bool im1 = s >= a.B;
  const int b = im1 ? s - a.B : s, n = im1 ? a.N : a.M;
  if (r >= n) return;
  const long src = ((long)s * a.Lp + r) * LG_DIM + c;
  float v;
  if (a.ctxf) v = a.ctxf[src];
  else {
    v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.ctxh)[src]);
    if (a.ctxl) v += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.ctxl)[src]);
  }
  (im1 ? a.out1 : a.out0)[((long)b * n + r) * LG_DIM + c] = v;
}
int misc_attn_unpack(const AttnIoArgs& a, cudaStream_t stream) {
  const int mx = a.M > a.N ? a.M : a.N;
  attn_unpack_kernel<<<dim3(mx, 2 * a.B), 256, 0, stream>>>(a);
  LG_CHECK_LAUNCH();
  return 0;
}
