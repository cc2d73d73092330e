// Warpgroup-MMA (wgmma) / TMA linear layers for the LG_PREC_BF16 and LG_PREC_BF16X3 paths.
//
//   C[tile rows, 256 cols per accumulator slot] = A[rows, K] * W[cols, K]^T     (fp32 accumulate in registers)
//
// * operands are bf16, K-major; tiles are staged by TMA (128-byte swizzle) into a shared-memory ring filled by one
//   producer warp; two MMA warpgroups consume it with wgmma.mma_async (M=64, N=256, K=16) and run the epilogue
//   straight from their accumulator registers;
// * LG_PREC_BF16X3 runs three passes over K into the same accumulator: A_lo*W_hi + A_hi*W_lo +
//   A_hi*W_hi with x = hi + lo, hi = bf16(x), lo = bf16(x - hi)  (~16 mantissa bits per operand);
// * A may be the concatenation of two sources along K (the FFN input cat([x, msg]), lightglue.py:172);
// * fused epilogues: bias (+ RoPE, head split, V transpose) for the QKV projections, bias + LayerNorm(512) + exact
//   GELU for ffn.0, bias + residual for ffn.3, bias * scale for input_proj / final_proj, the row reductions of the
//   assignment's similarity sweeps, bias + ReLU for the SuperPoint convolutions.
// Tiles: 128 rows x 256 columns, MMA warpgroup g owns rows 64 g .. +63; the LayerNorm variant: 64 rows x 512 columns,
// MMA warpgroup g owns the 256-column slot g and the row statistics are merged through shared memory.
// Threads: 384 = producer warpgroup (warp 0 issues the TMA loads; the warpgroup hands its registers to the others)
// + 2 MMA warpgroups.
#include <map>

#include "lg_handle.h"
#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BN = 256, BK = 64;
constexpr int W_TILE_BYTES = BN * BK * 2;  // 32 KB

enum { TEPI_QKV = 0, TEPI_LN_GELU = 2, TEPI_RESID = 3, TEPI_F32 = 4, TEPI_LSE = 5, TEPI_ARGMAX = 6, TEPI_CONV = 7 };

struct TcLinParams {
  CUtensorMap a_hi[2], a_lo[2];  // A segment 0 / 1, box 64 x tile rows
  CUtensorMap w_hi, w_lo;        // 3-D: (K, Nout, select), box 64 x 256 rows
  int kb0, kb_total, passes, n_tiles;
  int epi, rope;
  SeqState st;
  int w_select;                  // 1: third TMA coordinate / bias offset = stop_layer[pair] - 1
                                 // 2: third TMA coordinate = partner sequence (similarity sweeps of the assignment)
  float* part; int* part_arg; int part_stride;  // TEPI_LSE: (max, sumexp) pairs; TEPI_ARGMAX: best / arg, [S*Lp, part_stride]
  const float* term;             // TEPI_ARGMAX: logsigmoid(z) - LSE per token, [S, Lp]
  int reverse;  // walk the tile list from its end: a kernel that reads what the previous kernel wrote LAST finds it in L2
  float* logmat; int mat_m, mat_n;  // TEPI_ARGMAX, optional: materialise the [B, M+1, N+1] log-assignment matrix (core block)
  const float* bias; long bias_sel_stride;
  float scale;
  float* out_f32; int ldo;
  __nv_bfloat16* out_h; __nv_bfloat16* out_l; int ldb;
  __half* q; __half* k; __half* vt; const float* cs;
  const float* ln_g; const float* ln_b;
  unsigned int* dbg;
  // 3x3 convolution as a GEMM over a zero-padded NHWC image [rows = B (H+2) (W+2), Cin] (SuperPoint encoder): K block kb
  // = (tap, 64-channel block); the A tile of a tap is the same matrix shifted by (dy (W+2) + dx) rows (TMA fills the
  // rows outside the tensor with zeros).  conv_cb = Cin / 64 (0: not a convolution).  TEPI_CONV zeroes the padding
  // pixels again on the way out (conv_w2 = W + 2, conv_plane = (H+2)(W+2), conv_rows = B conv_plane) and applies ReLU.
  int conv_cb, conv_w2, conv_h, conv_w, relu;
  long conv_plane, conv_rows;
  int mma_n;  // N of the MMAs when fewer than 256 output columns exist (64 / 128; 0 = 256): the weight rows beyond are zero
};

template <int NSLOT>
struct LinCfg {
  static constexpr int TBM = NSLOT == 1 ? 128 : 64;     // rows per tile
  static constexpr int A_TILE_BYTES = TBM * BK * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + NSLOT * W_TILE_BYTES;
  static constexpr int THREADS = 384;
  static constexpr int MMA_WARPS = 8;
  static constexpr int RED_BYTES = NSLOT == 2 ? 2 * 2 * 64 * 4 : 0;  // LayerNorm: [pass][slot][row] partial sums
  static constexpr int FIXED_BYTES = RED_BYTES + 1024 + 256;         // + alignment slack + barriers
  static constexpr int SMEM_MAX = 232448;                            // 227 KB per CTA
  static constexpr int FIT = (SMEM_MAX - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 5 ? 5 : FIT;
  static_assert(STAGES >= 2, "the TMA ring needs at least two stages");
  static constexpr int SMEM = STAGES * STAGE_BYTES + FIXED_BYTES;
};

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exact (erf) GELU; erf via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7): 1 MUFU.RCP + 1 MUFU.EX2
__device__ __forceinline__ float gelu_erf(float y) {
  const float z = fabsf(y) * 0.70710678118654752f;
  const float tt = rcp_approx(fmaf(0.3275911f, z, 1.f));
  float pl = fmaf(1.061405429f, tt, -1.453152027f);
  pl = fmaf(pl, tt, 1.421413741f); pl = fmaf(pl, tt, -0.284496736f); pl = fmaf(pl, tt, 0.254829592f);
  const float ez = ex2_approx(-1.4426950408889634f * z * z);
  const float erf_abs = fmaf(-pl * tt, ez, 1.f);
  const float hy = 0.5f * y;
  return fmaf(copysignf(erf_abs, y), hy, hy);
}
__device__ __forceinline__ void mma_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // the two MMA warpgroups

struct TileInfo {
  int s, r0, n_tile, sel, len;
  long grow0;
};
// decode tile t (n-tile fastest, so neighbouring CTAs share A tiles in L2); returns false for tiles with nothing to do
template <int TBM>
__device__ __forceinline__ bool decode_tile(const TcLinParams& p, int t, int n_tiles, TileInfo& ti) {
  const int tiles_per_seq = p.st.Lp / TBM;
  ti.n_tile = t % n_tiles;
  const int rt = t / n_tiles;
  ti.s = rt / tiles_per_seq;
  ti.r0 = (rt % tiles_per_seq) * TBM;
  ti.len = p.st.len[ti.s];
  ti.grow0 = (long)ti.s * p.st.Lp + ti.r0;
  ti.sel = 0;
  const int pair = ti.s >= p.st.B ? ti.s - p.st.B : ti.s;
  const int sl = p.st.stop_layer[pair];
  bool live = ti.r0 < ti.len;
  if (p.w_select == 1) ti.sel = sl > 0 ? sl - 1 : 0;
  else if (p.w_select == 2) {
    ti.sel = ti.s >= p.st.B ? ti.s - p.st.B : ti.s + p.st.B;
    live = live && ti.n_tile * BN < p.st.len[ti.sel];  // no live columns otherwise
  } else if (sl != 0) live = false;                      // pair already exited (lightglue.py:549-550)
  return live;
}

// Persistent tile schedule: CTA c walks tiles c, c + grid, ... (skipping tiles with nothing to do)
template <int TBM>
struct TileWalk {
  int cur, step, end, n_tiles;
  __device__ TileWalk(int total_tiles, int n_tiles_) : cur(blockIdx.x), step(gridDim.x), end(total_tiles), n_tiles(n_tiles_) {}
  __device__ bool next(const TcLinParams& p, TileInfo& ti) {
    while (cur < end) {
      const int id = p.reverse ? end - 1 - cur : cur;
      cur += step;
      if (decode_tile<TBM>(p, id, n_tiles, ti)) return true;
    }
    return false;
  }
};

template <int NSLOT, int EPI>
__global__ void __launch_bounds__(LinCfg<NSLOT>::THREADS, 1) tc_linear_kernel(const __grid_constant__ TcLinParams p) {
  using C = LinCfg<NSLOT>;
  constexpr int TBM = C::TBM, STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // align by OFFSETTING the shared array (not by rebuilding a pointer from an integer): the compiler keeps the
  // shared address space and emits LDS / STS instead of generic LD / ST for everything derived from it
  uint8_t* smem = smem_raw + ((1024u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(smem_raw)) & 1023u)) & 1023u);
  float* s_red = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);  // LayerNorm: [pass][slot][64 rows]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + C::RED_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int n_tiles = p.n_tiles;
  const int total_tiles = n_tiles * p.st.S * (p.st.Lp / TBM);
  const int iters = p.passes * p.kb_total;  // ring iterations per tile: (pass, K block)

  pdl_launch_dependents();  // the next kernel's CTAs may take this SM as soon as this CTA has left it
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.a_hi[0]);
    tma_prefetch_desc(&p.w_hi);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], C::MMA_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  // everything above overlapped the tail of the previous kernel; activations, lengths and stop flags are only read
  // from here on
  pdl_wait();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    regs_dec<40>();
    if (warp == 0 && elect_one()) {
      int g = 0;  // global k-block counter across tiles (ring position)
      TileWalk<TBM> walk(total_tiles, n_tiles);
      TileInfo ti;
      while (walk.next(p, ti)) {
        for (int it = 0; it < iters; ++it, ++g) {
          const int stage = g % STAGES, round = g / STAGES;
          mbar_wait(&empty[stage], (round & 1) ^ 1, p.dbg, 17, it);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          const int pass = it / p.kb_total, kb = it % p.kb_total;
          // pass order (x3): A_lo*W_hi, A_hi*W_lo, A_hi*W_hi ; (bf16): A_hi*W_hi
          const bool a_lo = (p.passes == 3) && pass == 0;
          const bool w_lo = (p.passes == 3) && pass == 1;
          int seg = kb >= p.kb0 ? 1 : 0;
          int kc = (seg ? kb - p.kb0 : kb) * BK;
          int arow = (int)ti.grow0;
          if (p.conv_cb) {  // convolution tap: shifted rows of the padded image, channel block kb % conv_cb
            const int tap = kb / p.conv_cb;
            arow += (tap / 3 - 1) * p.conv_w2 + (tap % 3 - 1);
            kc = (kb % p.conv_cb) * BK;
            seg = 0;
          }
          mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
          tma_load_2d(sa, a_lo ? &p.a_lo[seg] : &p.a_hi[seg], kc, arow, &full[stage]);
#pragma unroll
          for (int sl_ = 0; sl_ < NSLOT; ++sl_)
            tma_load_3d(sa + C::A_TILE_BYTES + sl_ * W_TILE_BYTES, w_lo ? &p.w_lo : &p.w_hi, kb * BK,
                        (ti.n_tile * NSLOT + sl_) * BN, ti.sel, &full[stage]);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA warpgroups: main loop, then epilogue
  regs_inc<232>();
  const int wg = warp / 4 - 1;   // MMA warpgroup 0 / 1
  const int wq = warp % 4;       // warp inside it: accumulator rows 16 wq .. +15
  const int tq = lane & 3, tr = lane >> 2;
  const uint32_t a_off = NSLOT == 1 ? wg * 64 * 128 : 0;                                   // this warpgroup's 64 A rows
  const uint32_t b_off = C::A_TILE_BYTES + (NSLOT == 2 ? wg * W_TILE_BYTES : 0);          // and its W slot
  const int mma_n = p.mma_n ? p.mma_n : BN;
  const int rl_a = (NSLOT == 1 ? wg * 64 : 0) + wq * 16 + tr;  // tile row of accumulator registers 4 j, 4 j + 1 (+8: 4 j + 2, 4 j + 3)
  auto release = [&](int stage) {  // this warp's MMAs have finished reading the stage
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
  };
  int g = 0;
  float acc[128];
  TileWalk<TBM> walk(total_tiles, n_tiles);
  TileInfo ti;
  while (walk.next(p, ti)) {
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int it = 0; it < iters; ++it, ++g) {
      const int stage = g % STAGES;
      mbar_wait(&full[stage], (g / STAGES) & 1, p.dbg, 18, it);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
      const uint64_t ad = make_sdesc_sw128(sa + a_off), bd = make_sdesc_sw128(sa + b_off);
      fence_regs(acc);
      wgmma_fence();
      if (mma_n == 256) {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_bf16_n256(acc, ad + 2 * k, bd + 2 * k, 1u);
      } else if (mma_n == 128) {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_bf16_n128(acc, ad + 2 * k, bd + 2 * k, 1u);
      } else {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_bf16_n64(acc, ad + 2 * k, bd + 2 * k, 1u);
      }
      wgmma_commit();
      fence_regs(acc);
      wgmma_wait<1>();  // the previous stage's MMAs are done: hand it back to the producer
      if (prev >= 0) release(prev);
      prev = stage;
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (prev >= 0) release(prev);

    if (EPI == TEPI_LN_GELU) {
      // ---------------------------------------------------------------- LayerNorm(512) + GELU
      // Every row of the tile lies in one quad of lanes per warpgroup (256 columns each): quad shuffles give the
      // warpgroup's share, shared memory merges the two slots.  Two-pass statistics (mean, then squared deviations).
      const float* bias = p.bias + wg * BN;
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * tq));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          acc[4 * j + 2 * hr] += bb.x; acc[4 * j + 2 * hr + 1] += bb.y;
          sum[hr] += acc[4 * j + 2 * hr] + acc[4 * j + 2 * hr + 1];
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 1);
        sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 2);
        if (tq == 0) s_red[wg * 64 + rl_a + 8 * hr] = sum[hr];
      }
      mma_bar();
      float mean[2], sq[2] = {0.f, 0.f};
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) mean[hr] = (s_red[rl_a + 8 * hr] + s_red[64 + rl_a + 8 * hr]) * (1.f / LG_FFN);
#pragma unroll
      for (int j = 0; j < 32; ++j)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const float d0 = acc[4 * j + 2 * hr] - mean[hr], d1 = acc[4 * j + 2 * hr + 1] - mean[hr];
          sq[hr] = fmaf(d0, d0, fmaf(d1, d1, sq[hr]));
        }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        sq[hr] += __shfl_xor_sync(0xffffffffu, sq[hr], 1);
        sq[hr] += __shfl_xor_sync(0xffffffffu, sq[hr], 2);
        if (tq == 0) s_red[128 + wg * 64 + rl_a + 8 * hr] = sq[hr];
      }
      mma_bar();
      float rstd[2];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr)
        rstd[hr] = rsqrtf((s_red[128 + rl_a + 8 * hr] + s_red[192 + rl_a + 8 * hr]) * (1.f / LG_FFN) + 1e-5f);
      const bool haslo = p.out_l != nullptr;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long grow = ti.grow0 + rl_a + 8 * hr;
        __nv_bfloat16* oh = p.out_h + grow * p.ldb + wg * BN;
        __nv_bfloat16* ol = haslo ? p.out_l + grow * p.ldb + wg * BN : nullptr;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int c = 8 * j + 2 * tq;
          const float2 gg = __ldg(reinterpret_cast<const float2*>(p.ln_g + wg * BN + c));
          const float2 be = __ldg(reinterpret_cast<const float2*>(p.ln_b + wg * BN + c));
          const float a = gelu_erf(fmaf((acc[4 * j + 2 * hr] - mean[hr]) * rstd[hr], gg.x, be.x));
          const float b = gelu_erf(fmaf((acc[4 * j + 2 * hr + 1] - mean[hr]) * rstd[hr], gg.y, be.y));
          const uint32_t hi = pack_bf16x2(a, b);
          *reinterpret_cast<uint32_t*>(oh + c) = hi;
          if (haslo) *reinterpret_cast<uint32_t*>(ol + c) = pack_bf16x2_lo(a, b, hi);
        }
      }
      continue;
    }

    if (EPI == TEPI_LSE || EPI == TEPI_ARGMAX) {
      // ---------------------------------------------------------------- assignment sweeps (lightglue.py:265-277, 302-305)
      // on a 128 x 256 tile of S = p_s p_partner^T; partials per 128-column slot, reduced over the quad of lanes that
      // holds a row
      const int lens = p.st.len[ti.sel];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int rl = rl_a + 8 * hr;
        const long grow = ti.grow0 + rl;
        const bool live = ti.r0 + rl < ti.len;
        const float rterm = (EPI == TEPI_ARGMAX && live) ? p.term[grow] : 0.f;
        const bool write_mat = EPI == TEPI_ARGMAX && p.logmat != nullptr && ti.s < p.st.B && live;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int col0 = ti.n_tile * BN + half * 128;
          const int ncols = lens - col0;  // live columns of this slot
          const int slot = ti.n_tile * 2 + half;
          if (EPI == TEPI_LSE) {
            constexpr float L2E = 1.4426950408889634f;
            float m = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (8 * jj + 2 * tq + e < ncols) m = fmaxf(m, acc[4 * (16 * half + jj) + 2 * hr + e]);
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            float se = 0.f;
            if (m != -INFINITY) {
              const float mb = -m * L2E;
#pragma unroll
              for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  if (8 * jj + 2 * tq + e < ncols) se += ex2_approx(fmaf(acc[4 * (16 * half + jj) + 2 * hr + e], L2E, mb));
            }
            se += __shfl_xor_sync(0xffffffffu, se, 1);
            se += __shfl_xor_sync(0xffffffffu, se, 2);
            if (live && tq == 0) reinterpret_cast<float2*>(p.part)[grow * p.part_stride + slot] = make_float2(m, se);
          } else {
            // score = 2 S + term_s[i] + term_partner[j]; the row term does not move the arg-max
            const float* ct = p.term + (long)ti.sel * p.st.Lp + col0;
            float* mo = write_mat ? p.logmat + ((long)ti.s * (p.mat_m + 1) + ti.r0 + rl) * (p.mat_n + 1) + col0 : nullptr;
            float best = -INFINITY;
            int arg = 0;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * jj + 2 * tq + e;
                if (c < ncols) {
                  const float sc = fmaf(2.f, acc[4 * (16 * half + jj) + 2 * hr + e], __ldg(ct + c));
                  if (mo) mo[c] = sc + rterm;
                  if (sc > best) { best = sc; arg = col0 + c; }  // ascending columns: first max wins
                }
              }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
              const float ob = __shfl_xor_sync(0xffffffffu, best, o);
              const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
              if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
            }
            if (live && tq == 0) {
              p.part[grow * p.part_stride + slot] = best + rterm;
              p.part_arg[grow * p.part_stride + slot] = arg;
            }
          }
        }
      }
      continue;
    }

    // ------------------------------------------------------------------ element-wise epilogues
    const float* bias = p.bias + (p.w_select == 1 ? (long)ti.sel * p.bias_sel_stride : 0) + ti.n_tile * BN;
    // which output a QKV tile feeds: packed channel order [q | k | v] (self) or [qk | v] (cross)
    const int which = ti.n_tile;
    const bool qkv_v = EPI == TEPI_QKV && (p.rope ? which == 2 : which == 1);
    const bool use_rope = EPI == TEPI_QKV && p.rope && !qkv_v;
    const bool f32out = EPI == TEPI_RESID || EPI == TEPI_F32;
    const bool has16 = EPI == TEPI_CONV || EPI == TEPI_RESID || (EPI == TEPI_F32 && p.out_h != nullptr);
    const bool haslo = has16 && p.out_l != nullptr;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int rl = rl_a + 8 * hr;
      const int r = ti.r0 + rl;
      const long grow = ti.grow0 + rl;
      const bool live = r < ti.len;
      bool inside = true;
      if (EPI == TEPI_CONV) {  // the padding pixels of the NHWC image stay zero for the next layer's taps
        const long pp = grow % p.conv_plane;
        const int yy = (int)(pp / p.conv_w2), xx = (int)(pp % p.conv_w2);
        inside = grow < p.conv_rows && yy >= 1 && yy <= p.conv_h && xx >= 1 && xx <= p.conv_w;
      }
      // RoPE cos / sin of this row, loaded ahead of its stores (the compiler does not move a load above a store it cannot
      // prove independent, so a load per column would pay its full latency every time); frequency index d / 2 =
      // 4 (j % 8) + tq, the same for every head
      float rc[8], rs[8];
      if (use_rope) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          rc[jj] = __ldg(p.cs + grow * 64 + 4 * jj + tq);
          rs[jj] = __ldg(p.cs + grow * 64 + 32 + 4 * jj + tq);
        }
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int tcol = 8 * j + 2 * tq;        // column inside the tile (even)
        const int col = ti.n_tile * BN + tcol;  // output channel
        if (EPI == TEPI_CONV && col >= p.ldb) continue;  // Cout < 256: the weight rows beyond it are zero padding
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + tcol));
        float v0 = acc[4 * j + 2 * hr] + bb.x, v1 = acc[4 * j + 2 * hr + 1] + bb.y;
        if (EPI == TEPI_QKV) {
          const int hh = tcol / LG_HDIM, d = tcol % LG_HDIM;
          if (qkv_v) {
            // V is stored transposed [S, H, 64, Lp] (K-major B operand of P*V)
            if (live) {
              __half* dst = p.vt + (((long)ti.s * LG_HEADS + hh) * LG_HDIM + d) * p.st.Lp + r;
              dst[0] = __float2half_rn(v0);
              dst[p.st.Lp] = __float2half_rn(v1);
            }
            continue;
          }
          if (use_rope) {  // rotary embedding on q / k (lightglue.py:58-65, 168-169); freq index = d / 2
            const float c = rc[j % 8], s = rs[j % 8];
            const float a = v0, b = v1;
            v0 = a * c - b * s;
            v1 = b * c + a * s;
          }
          __half* dst = (which == 0 ? p.q : p.k) + (((long)ti.s * LG_HEADS + hh) * p.st.Lp + r) * LG_HDIM + d;
          *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(v0, v1);
          continue;
        }
        if (p.scale != 1.f) { v0 *= p.scale; v1 *= p.scale; }
        if (EPI == TEPI_CONV) {
          v0 = inside ? ((p.relu && v0 < 0.f) ? 0.f : v0) : 0.f;
          v1 = inside ? ((p.relu && v1 < 0.f) ? 0.f : v1) : 0.f;
        }
        if (EPI == TEPI_RESID) {  // x + ffn(...) (lightglue.py:172 / 228-229)
          const float2 xr = *reinterpret_cast<const float2*>(p.out_f32 + grow * p.ldo + col);
          v0 += xr.x; v1 += xr.y;
        }
        if (f32out && col < p.ldo) *reinterpret_cast<float2*>(p.out_f32 + grow * p.ldo + col) = make_float2(v0, v1);
        if (has16 && col < p.ldb) {
          const uint32_t hi = pack_bf16x2(v0, v1);
          *reinterpret_cast<uint32_t*>(p.out_h + grow * p.ldb + col) = hi;
          if (haslo) *reinterpret_cast<uint32_t*>(p.out_l + grow * p.ldb + col) = pack_bf16x2_lo(v0, v1, hi);
        }
      }
    }
  }
}

// fp32 -> bf16 hi (/ lo) for rows < len
__global__ void __launch_bounds__(256) shadow_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                                     __nv_bfloat16* __restrict__ lo, int cols, SeqState st) {
  const int row = blockIdx.x;
  const int s = row / st.Lp, r = row % st.Lp;
  if (r >= st.len[s]) return;
  for (int c = threadIdx.x * 4; c < cols; c += 1024) {
    const float4 t = *reinterpret_cast<const float4*>(x + (long)row * cols + c);
    const float v[4] = {t.x, t.y, t.z, t.w};
    uint2 h, l;
    h.x = pack_bf16x2(v[0], v[1]); h.y = pack_bf16x2(v[2], v[3]);
    l.x = pack_bf16x2_lo(v[0], v[1], h.x); l.y = pack_bf16x2_lo(v[2], v[3], h.y);
    *reinterpret_cast<uint2*>(hi + (long)row * cols + c) = h;
    if (lo) *reinterpret_cast<uint2*>(lo + (long)row * cols + c) = l;
  }
}

__global__ void split_weights_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                     size_t n) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = w[i];
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// ------------------------------------------------------------------------------------------------
// host: the GEMM entry point, tensor maps, launches
// ------------------------------------------------------------------------------------------------
// cuTensorMapEncodeTiled is fetched through the runtime (no link-time dependency on libcuda).
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeFn)p;
  }
  return fn;
}

template <int NSLOT, int EPI>
int launch_linear_t(const TcLinParams& p, cudaStream_t stream) {
  using C = LinCfg<NSLOT>;
  const int num_sms = lg_num_sms();
  const int total = p.n_tiles * p.st.S * (p.st.Lp / C::TBM);
  const int grid = total < num_sms ? total : num_sms;
  return tc_launch(tc_linear_kernel<NSLOT, EPI>, dim3(grid), C::THREADS, C::SMEM, p, stream);
}
int launch_linear(const TcLinParams& p, cudaStream_t stream) {
  switch (p.epi) {
    case TEPI_QKV: return launch_linear_t<1, TEPI_QKV>(p, stream);
    case TEPI_LN_GELU: return launch_linear_t<2, TEPI_LN_GELU>(p, stream);
    case TEPI_RESID: return launch_linear_t<1, TEPI_RESID>(p, stream);
    case TEPI_F32: return launch_linear_t<1, TEPI_F32>(p, stream);
    case TEPI_CONV: return launch_linear_t<1, TEPI_CONV>(p, stream);
    case TEPI_LSE: return launch_linear_t<1, TEPI_LSE>(p, stream);
    case TEPI_ARGMAX: return launch_linear_t<1, TEPI_ARGMAX>(p, stream);
  }
  return lg_set_error("launch_linear: bad epilogue");
}

// Operands of one GEMM.  A = [A0 | A1] along K, each [st.S * st.Lp rows, k] bf16 row-major; W = nsel matrices [nout, K]
// bf16 (K = k0 + k1, or 9 k0 for a 3x3 convolution), sel_stride elements apart.  The lo images are read in bf16x3 only.
struct TcOperands {
  const __nv_bfloat16 *a0h, *a0l; int k0;
  const __nv_bfloat16 *a1h, *a1l; int k1;  // k1 = 0: one segment
  const __nv_bfloat16 *wh, *wl; int nout;
  int nsel; size_t sel_stride;
};

// The one host entry point of tc_linear_kernel: p carries the epilogue fields (and w_select / conv_* / mma_n where they
// apply); this adds the tensor maps, the K-block and pass counts, and launches n_tiles column tiles per row tile.
int tc_gemm(TcEngine& e, const SeqState& st, const TcOperands& d, int n_tiles, TcLinParams& p, cudaStream_t stream) {
  const uint64_t rows = (uint64_t)st.S * st.Lp;
  const uint32_t tbm = p.epi == TEPI_LN_GELU ? LinCfg<2>::TBM : LinCfg<1>::TBM;
  const uint64_t K = p.conv_cb ? 9 * d.k0 : d.k0 + d.k1, nout = d.nout, nsel = d.nsel;
  const uint64_t sel_bytes = (nsel > 1 ? d.sel_stride : nout * K) * 2;
  auto amap = [&](CUtensorMap* out, const void* a, uint64_t k) {  // box 64 x the tile height
    return tc_tmap(e, {a, 2, {k, rows}, {k * 2}, {BK, tbm}}, out);
  };
  auto wmap = [&](CUtensorMap* out, const void* w) { return tc_tmap(e, {w, 3, {K, nout, nsel}, {K * 2, sel_bytes}, {BK, BN, 1}}, out); };
  // maps the kernel does not read repeat a map it does (segment 1 of a one-segment A, every lo map in bf16)
  int r;
  if ((r = amap(&p.a_hi[0], d.a0h, d.k0))) return r;
  p.a_hi[1] = p.a_hi[0];
  if (d.k1 && (r = amap(&p.a_hi[1], d.a1h, d.k1))) return r;
  p.a_lo[0] = p.a_hi[0]; p.a_lo[1] = p.a_hi[1];
  if (e.x3) {
    if ((r = amap(&p.a_lo[0], d.a0l, d.k0))) return r;
    p.a_lo[1] = p.a_lo[0];
    if (d.k1 && (r = amap(&p.a_lo[1], d.a1l, d.k1))) return r;
  }
  if ((r = wmap(&p.w_hi, d.wh))) return r;
  p.w_lo = p.w_hi;
  if (e.x3 && (r = wmap(&p.w_lo, d.wl))) return r;
  p.kb_total = (int)(K / BK);
  p.kb0 = d.k1 ? d.k0 / BK : p.kb_total;
  p.passes = e.x3 ? 3 : 1;
  p.n_tiles = n_tiles;
  p.st = st;
  p.dbg = e.dbg;
  return launch_linear(p, stream);
}

// a matcher GEMM: one launch of the handle's count
int run_linear(LgHandle* h, const SeqState& st, const TcOperands& d, int n_tiles, TcLinParams& p, cudaStream_t stream) {
  h->launches += 1;
  return tc_gemm(h->tc, st, d, n_tiles, p, stream);
}
}  // namespace

struct TcMapCache {
  std::map<TmapArgs, CUtensorMap> m;
};

int tc_tmap(TcEngine& e, const TmapArgs& a, CUtensorMap* out) {
  auto& m = e.maps->m;
  auto it = m.find(a);
  if (it != m.end()) { *out = it->second; return 0; }
  if (m.size() > 4096) m.clear();
  EncodeFn enc = get_encode();
  if (!enc) return lg_set_error("cuTensorMapEncodeTiled unavailable");
  const cuuint32_t estr[3] = {1, 1, 1};
  if (enc(out, a.dtype, a.rank, const_cast<void*>(a.base), a.dims.data(), a.strides.data(), a.box.data(), estr,
          CU_TENSOR_MAP_INTERLEAVE_NONE, a.swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return lg_set_error("cuTensorMapEncodeTiled failed");
  m.emplace(a, *out);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// entry points used by lg_api.cu
// ------------------------------------------------------------------------------------------------

// ------------------------------------------------------------------------------------------------
// Assignment tail on the tensor cores (matches-only variant: the log-assignment matrix is never written)
// ------------------------------------------------------------------------------------------------
// launches: sweep 1 (LSE partials), z + term, sweep 2 (arg-max partials, optionally the matrix), [dustbin], tail
int tc_assign_sweeps(LgHandle* h, const TcBuffers& b, const SeqState& st, const AssignArgs& a, float* part, int* part_arg,
                     float* term, cudaStream_t stream) {
  float* logmat = a.log_assignment;
  const int M = a.M, N = a.N;
  const int ntc = (st.Lp + BN - 1) / BN;
  // A = p of every sequence, W = p of its partner sequence (w_select 2)
  const TcOperands ops{b.msgh, b.msgl, LG_DIM, nullptr, nullptr, 0, b.msgh, b.msgl, st.Lp, st.S, (size_t)st.Lp * LG_DIM};
  for (int sweep = 0; sweep < 2; ++sweep) {
    TcLinParams p{};
    p.epi = sweep == 0 ? TEPI_LSE : TEPI_ARGMAX;
    p.scale = 1.f; p.bias = h->wpk;  // unused
    p.part = part; p.part_arg = part_arg; p.part_stride = 2 * ntc; p.term = term;
    p.logmat = sweep == 1 ? logmat : nullptr; p.mat_m = M; p.mat_n = N;
    p.w_select = 2;
    int r;
    {
      Timer tm(h, LG_K_ASSIGN_MATRIX, stream, sweep == 1 && logmat != nullptr);  // the matrix-writing sweep on its own
      if ((r = run_linear(h, st, ops, ntc, p, stream))) return r;
    }
    if (sweep == 0) {
      if ((r = misc_assign_term(a, st, part, 2 * ntc, BN / 2, term, stream))) return r;
      h->launches += 1;
    }
  }
  if (logmat) { if (int rd = misc_assign_dustbin(a, st, stream)) return rd; h->launches += 1; }
  int r = misc_assign_tail(a, st, part, part_arg, 2 * ntc, BN / 2, stream);
  h->launches += 1;
  return r;
}

unsigned int tc_debug_timeout_code(const TcEngine& e, unsigned int* words32) {
  unsigned int v[32] = {0};
  if (!e.dbg) return 0;
  if (cudaMemcpy(v, e.dbg, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return 0xffffffffu;
  unsigned int first = 0;
  for (int i = 0; i < 32; ++i) {
    if (words32) words32[i] = v[i];
    if (v[i] && !first) first = (unsigned)i << 24 | (v[i] & 0x80ffffffu);
  }
  if (first) cudaMemset(e.dbg, 0, sizeof(v));
  return first;
}

int tc_engine_create(TcEngine* e, const float* w, size_t n, bool x3, cudaStream_t stream) {
  e->x3 = x3;
  cudaError_t err = cudaMalloc(&e->w_hi, n * sizeof(__nv_bfloat16));
  if (err != cudaSuccess) return lg_set_cuda_error(err, __FILE__, __LINE__);
  err = cudaMalloc(&e->w_lo, n * sizeof(__nv_bfloat16));
  if (err != cudaSuccess) return lg_set_cuda_error(err, __FILE__, __LINE__);
  split_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(w, e->w_hi, e->w_lo, n);
  LG_CHECK_LAUNCH();
  e->maps = new TcMapCache();
  err = cudaMalloc(&e->dbg, 32 * sizeof(unsigned int));
  if (err != cudaSuccess) return lg_set_cuda_error(err, __FILE__, __LINE__);
  cudaMemsetAsync(e->dbg, 0, 32 * sizeof(unsigned int), stream);
  if (!get_encode()) return lg_set_error("cuTensorMapEncodeTiled unavailable (driver too old?)");
  return 0;
}

void tc_engine_destroy(TcEngine* e) {
  if (e->w_hi) cudaFree(e->w_hi);
  if (e->w_lo) cudaFree(e->w_lo);
  delete e->maps;
  if (e->dbg) cudaFree(e->dbg);
  *e = TcEngine{};
}

void tc_carve(size_t* off, char* base, size_t S, int Lp, const LgHandle* h, TcBuffers* b) {
  const size_t R = S * Lp;
  const bool x3 = h->cfg.precision == LG_PREC_BF16X3;
  auto take = [&](size_t bytes) -> void* {
    *off = (*off + 1023) & ~(size_t)1023;
    void* p = base ? base + *off : nullptr;
    *off += bytes;
    return p;
  };
  b->xh = (__nv_bfloat16*)take(R * 256 * 2);
  b->xl = x3 ? (__nv_bfloat16*)take(R * 256 * 2) : nullptr;
  b->ctxh = (__nv_bfloat16*)take(R * 256 * 2);
  b->ctxl = x3 ? (__nv_bfloat16*)take(R * 256 * 2) : nullptr;
  b->msgh = (__nv_bfloat16*)take(R * 256 * 2);
  b->msgl = x3 ? (__nv_bfloat16*)take(R * 256 * 2) : nullptr;
  b->hh = (__nv_bfloat16*)take(R * 512 * 2);
  b->hl = x3 ? (__nv_bfloat16*)take(R * 512 * 2) : nullptr;
  b->q = (__half*)take(R * 256 * 2);
  b->k = (__half*)take(R * 256 * 2);
  b->vt = (__half*)take(R * 256 * 2);
}

int tc_refresh_shadow(LgHandle* h, const TcBuffers& b, const float* x, const SeqState& st, cudaStream_t stream) {
  shadow_kernel<<<st.S * st.Lp, 256, 0, stream>>>(x, b.xh, b.xl, LG_DIM, st);
  LG_CHECK_LAUNCH();
  return 0;
}

int tc_input_proj(LgHandle* h, const TcBuffers& b, const SeqState& st, const float* desc_packed, float* x, cudaStream_t stream) {
  const int d = h->cfg.input_dim;
  if (d % BK != 0) return lg_set_error("tensor-core input_proj needs input_dim % 64 == 0");
  shadow_kernel<<<st.S * st.Lp, 256, 0, stream>>>(desc_packed, b.hh, b.hl, d, st);
  LG_CHECK_LAUNCH();
  h->launches += 1;
  TcLinParams p{};
  p.epi = TEPI_F32; p.scale = 1.f; p.bias = h->wpk + h->o_inb;
  p.out_f32 = x; p.ldo = LG_DIM; p.out_h = b.xh; p.out_l = b.xl; p.ldb = LG_DIM;
  const TcOperands ops{b.hh, b.hl, d, nullptr, nullptr, 0, h->tc.w_hi + h->o_inw, h->tc.w_lo + h->o_inw, LG_DIM, 1, 0};
  return run_linear(h, st, ops, 1, p, stream);
}

int tc_final_proj(LgHandle* h, const TcBuffers& b, const SeqState& st, float* p_out, cudaStream_t stream) {
  TcLinParams p{};
  p.epi = TEPI_F32; p.scale = 0.25f;  // / 256^(1/4) (lightglue.py:291)
  p.w_select = 1;  // final_proj of the layer each pair stopped at
  p.bias = h->wpk + h->o_assign + AO_FB; p.bias_sel_stride = ASSIGN_BLOB_PAD;
  p.out_f32 = p_out; p.ldo = LG_DIM; p.out_h = b.msgh; p.out_l = b.msgl; p.ldb = LG_DIM;  // bf16 images feed the sweeps
  const size_t w = h->o_assign + AO_FW;
  const TcOperands ops{b.xh, b.xl, LG_DIM, nullptr, nullptr, 0, h->tc.w_hi + w, h->tc.w_lo + w, LG_DIM, h->cfg.n_layers,
                       ASSIGN_BLOB_PAD};
  return run_linear(h, st, ops, 1, p, stream);
}

int tc_conv(TcEngine& e, const SeqState& st, const __nv_bfloat16* in_h, const __nv_bfloat16* in_l, int cin, int taps, size_t w_off,
            const float* bias, int relu, int B, int H, int W, __nv_bfloat16* out_h, __nv_bfloat16* out_l, int cout, float* out_f32,
            int ldo, cudaStream_t stream) {
  if (cin % BK != 0 || (taps != 1 && taps != 9)) return lg_set_error("tc_conv: Cin must be a multiple of 64, 1x1 or 3x3");
  TcLinParams p{};
  p.epi = out_f32 ? TEPI_F32 : TEPI_CONV;
  p.scale = 1.f; p.bias = bias; p.relu = relu;
  p.out_f32 = out_f32; p.ldo = ldo; p.out_h = out_h; p.out_l = e.x3 ? out_l : nullptr; p.ldb = cout;
  const int mma_n = cout <= 64 ? 64 : cout <= 128 ? 128 : BN;  // no MMA columns for the zero rows of a narrow layer
  p.mma_n = mma_n == BN ? 0 : mma_n;
  p.conv_cb = taps == 9 ? cin / BK : 0;
  p.conv_w2 = W + 2; p.conv_h = H; p.conv_w = W;
  p.conv_plane = (long)(H + 2) * (W + 2); p.conv_rows = (long)B * p.conv_plane;
  const TcOperands ops{in_h, in_l, cin, nullptr, nullptr, 0, e.w_hi + w_off, e.w_lo + w_off, BN, 1, 0};
  return tc_gemm(e, st, ops, 1, p, stream);
}

int tc_block(LgHandle* h, const TcBuffers& b, const SeqState& st, int layer, int blk, float* x, const float* cs,
             cudaStream_t stream) {
  const BlockOff& o = blk == 0 ? h->bself : h->bcross;
  const size_t base = h->o_layers + (size_t)layer * h->layer_stride + (blk == 0 ? 0 : h->bself.total);
  const float* bw = h->wpk + base;
  const __nv_bfloat16 *wh = h->tc.w_hi + base, *wl = h->tc.w_lo + base;
  // Tile order against the 50 MB L2: every kernel of the chain reads what its predecessor wrote, and only the part written
  // LAST is still resident.  QKV and ffn.0 walk their tile lists backwards, ffn.3 (and the attention grid) forwards: ffn.3
  // starts on the hidden tiles ffn.0 finished with, the next QKV on the x images ffn.3 finished with, attention on the
  // q / k / v of the sequences QKV wrote last, ffn.0 on the context of the sequences attention wrote last.
  {  // QKV (+RoPE) / [to_qk | to_v] projection
    Timer t(h, LG_K_LINEAR, stream);
    Timer t2(h, LG_K_QKV, stream);
    TcLinParams p{};
    p.epi = TEPI_QKV; p.rope = blk == 0; p.scale = 1.f; p.bias = bw + o.bp; p.reverse = 1;
    p.q = b.q; p.k = b.k; p.vt = b.vt; p.cs = cs;
    const int nout = blk == 0 ? 3 * LG_DIM : 2 * LG_DIM;
    const TcOperands ops{b.xh, b.xl, LG_DIM, nullptr, nullptr, 0, wh + o.wp, wl + o.wp, nout, 1, 0};
    int r = run_linear(h, st, ops, nout / BN, p, stream);
    if (r) return r;
  }
  {
    Timer t(h, LG_K_ATTENTION, stream);
    int r = tc_attention(h, b, st, blk == 0 ? 0 : st.B, blk == 0 ? b.k : b.q, stream);
    if (r) return r;
  }
  Timer t(h, LG_K_LINEAR, stream);
  {  // ffn.0 on cat([x, msg]) + LayerNorm + GELU -> h; the output projection is folded into the weights (W1f, b1f:
     // lg_handle.h), so the GEMM reads cat([x, ctx]) and `msg` is never formed
    TcLinParams p{};
    p.epi = TEPI_LN_GELU; p.scale = 1.f; p.bias = bw + o.b1f; p.ln_g = bw + o.g; p.ln_b = bw + o.be;
    p.reverse = 1;
    p.out_h = b.hh; p.out_l = b.hl; p.ldb = LG_FFN;
    const TcOperands ops{b.xh, b.xl, LG_DIM, b.ctxh, b.ctxl, LG_DIM, wh + o.w1f, wl + o.w1f, LG_FFN, 1, 0};
    Timer t2(h, LG_K_FFN0, stream);
    int r = run_linear(h, st, ops, 1, p, stream);  // one 512-column tile: the whole LayerNorm row
    if (r) return r;
  }
  {  // ffn.3 + residual -> x (fp32 master + bf16 shadows)
    TcLinParams p{};
    p.epi = TEPI_RESID; p.scale = 1.f; p.bias = bw + o.b2; p.out_f32 = x; p.ldo = LG_DIM;
    p.out_h = b.xh; p.out_l = b.xl; p.ldb = LG_DIM;
    const TcOperands ops{b.hh, b.hl, LG_FFN, nullptr, nullptr, 0, wh + o.w2, wl + o.w2, LG_DIM, 1, 0};
    Timer t2(h, LG_K_FFN3, stream);
    int r = run_linear(h, st, ops, 1, p, stream);
    if (r) return r;
  }
  return 0;
}
