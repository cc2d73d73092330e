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
//   assignment's similarity sweeps, the nearest-neighbour matcher's top-2 sweep, bias + ReLU for the convolutions.
// Tiles: 128 rows x 256 columns, MMA warpgroup g owns rows 64 g .. +63.  The LayerNorm variant runs in clusters of two
// CTAs: a cluster owns a 128-row tile of all 512 columns, CTA rank r columns 256 r .. +255, and the two CTAs exchange
// their row partial sums through distributed shared memory.
// Threads: 384 = producer warpgroup (warp 0 issues the TMA loads; the warpgroup hands its registers to the others)
// + 2 MMA warpgroups.
#include <map>

#include "lg_handle.h"
#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BN = 256, BK = 64;
constexpr int W_TILE_BYTES = BN * BK * 2;  // 32 KB

enum { TEPI_QKV = 0, TEPI_LN_GELU = 2, TEPI_RESID = 3, TEPI_F32 = 4, TEPI_LSE = 5, TEPI_ARGMAX = 6, TEPI_CONV = 7, TEPI_TOP2 = 8 };
// the guided nearest-neighbour sweeps: TEPI_TOP2 over the columns that pass a homography (H) or epipolar (F) gate
enum { TEPI_TOP2_H = 9, TEPI_TOP2_F = 10 };

struct TcLinParams {
  CUtensorMap a_hi[2], a_lo[2];  // A segment 0 / 1, box 64 x tile rows
  CUtensorMap w_hi, w_lo;        // 3-D: (K, Nout, select), box 64 x 256 rows
  int kb0, kb_total, passes, n_tiles;
  int epi, rope;
  SeqState st;
  int w_select;                  // 1: third TMA coordinate / bias offset = stop_layer[pair] - 1
                                 // 2: third TMA coordinate = partner sequence (similarity sweeps of the assignment)
  float* part; int* part_arg; int part_stride;  // TEPI_LSE: (max, sumexp) pairs; TEPI_ARGMAX: best / arg; TEPI_TOP2:
                                                // (s1, s2) pairs / j1, [S*Lp, part_stride]
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
  // k x k convolution (k = 3: SuperPoint encoder, k = 5: DISK) as a GEMM over a zero-padded NHWC image [rows = B (H+2q)
  // (W+2q), Cin] with a border of q = k / 2 pixels: K block kb = (tap, 64-channel block); the A tile of a tap is the same
  // matrix shifted by (dy (W+2q) + dx) rows, dy, dx in [-q, q] (TMA fills the rows outside the tensor with zeros).
  // conv_cb = Cin / 64 (0: not a convolution).  TEPI_CONV zeroes the padding pixels again on the way out (conv_w2 = W + 2q,
  // conv_plane = (H+2q)(W+2q), conv_rows = B conv_plane) and applies ReLU.
  int conv_cb, conv_k, conv_pad, conv_w2, conv_h, conv_w, relu;
  long conv_plane, conv_rows;
  // stride-2 3x3 convolution by phase split (conv_pstride > 0): A holds the four polyphase images of the padded input,
  // phase (py, px) = padded pixels (2i + py, 2j + px) at the output's padded position (i + 1, j + 1), phase 2 py + px
  // starting at row (2 py + px) conv_pstride; tap (dy, dx) reads phase (dy & 1, dx & 1) shifted by (dy >> 1) conv_w2 +
  // (dx >> 1) rows.  The A map then spans 4 conv_pstride rows (conv_arows), more than the output's.
  int conv_pstride;
  long conv_arows;
  int mma_n;  // N of the MMAs when fewer than 256 output columns exist (64 / 128; 0 = 256): the weight rows beyond are zero
  // TEPI_QKV: the TMA store map of vt ([S H 64, Lp], box 64 rows x 64 d); TEPI_RESID: out_f32 (box 16 x 64), the map the
  // producer prefetches the residual x to L2 with
  CUtensorMap out_map;
  // TEPI_TOP2_H / F (appended, so the parameter offsets of the other epilogues stay put): gate records, field f of row
  // r at gate_rec[f * S Lp + r] (H: 2 fields, F: 6), gate_on[pair] != 0 for a guided pair, and the squared threshold
  const float* gate_rec; const int* gate_on; float gate_t2;
};

constexpr int TBM = 128;  // rows per tile

template <int EPI>
struct LinCfg {
  static constexpr bool LN = EPI == TEPI_LN_GELU;
  static constexpr int CLUSTER = LN ? 2 : 1;  // CTAs per 128-row tile: the LayerNorm needs all 512 columns of a row
  static constexpr int A_TILE_BYTES = TBM * BK * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + W_TILE_BYTES;
  static constexpr int THREADS = 384;
  static constexpr int MMA_WARPS = 8;
  // QKV: one staged vt box of 64 rows x 64 d (8 KB), two per MMA warpgroup; the guided top-2 sweeps: the tile's column
  // gate records (6 fields x 256 floats); every other epilogue stores from registers
  static constexpr int STG_BOX = 8192;
  static constexpr int STG_BYTES = EPI == TEPI_QKV ? 2 * 2 * STG_BOX
                                   : (EPI == TEPI_TOP2_H || EPI == TEPI_TOP2_F) ? 6 * BN * 4
                                                                                : 0;
  static constexpr int PAR_BYTES = (LN ? 3 : 1) * BN * 4;  // the tile's bias / LayerNorm bias, gamma, beta
  static constexpr int RED_BYTES = LN ? 2 * TBM * 4 : 0;  // LayerNorm: [pass][row] the peer CTA's row partial sums
  static constexpr int FIXED_BYTES = STG_BYTES + PAR_BYTES + RED_BYTES + 1024 + 256;  // + alignment slack + barriers
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
// Transpose of a 32-column chunk of one accumulator row inside the quad of lanes that holds it.  On entry lane q (=
// lane % 4) holds in v[i] the W words of its column pair 8 i + 2 q, +1 (i = 0 .. 3: the chunk's four 8-column groups);
// on return it holds in v[i] the words of the column pair 8 q + 2 i, +1, so 8 consecutive columns, which it writes with
// 16-byte stores.  Two butterfly exchanges (lanes q ^ 2, then q ^ 1) of two pairs each, then a reorder by source lane;
// words are only moved, never changed.
template <int W>
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4][W], int q) {
  const bool b1 = (q & 2) != 0, b0 = (q & 1) != 0;
  uint32_t s[2][2][W];  // [source: this lane, lane q ^ 2][e]: the column pair of group 2 b1 + e
#pragma unroll
  for (int e = 0; e < 2; ++e)
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const uint32_t give = b1 ? v[e][w] : v[2 + e][w];
      s[0][e][w] = b1 ? v[2 + e][w] : v[e][w];
      s[1][e][w] = __shfl_xor_sync(0xffffffffu, give, 2);
    }
  uint32_t t[4][W];  // the column pair of group q from lane q ^ d
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const uint32_t give = b0 ? s[h][0][w] : s[h][1][w];
      t[2 * h][w] = b0 ? s[h][1][w] : s[h][0][w];
      t[2 * h + 1][w] = __shfl_xor_sync(0xffffffffu, give, 1);
    }
#pragma unroll
  for (int i = 0; i < 4; ++i)  // v[i] = t[i ^ q]
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const uint32_t a = b0 ? t[i ^ 1][w] : t[i][w], b = b0 ? t[i ^ 3][w] : t[i ^ 2][w];
      v[i][w] = b1 ? b : a;
    }
}
__device__ __forceinline__ void st_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  *reinterpret_cast<uint4*>(p) = make_uint4(a, b, c, d);
}
__device__ __forceinline__ void mma_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // the two MMA warpgroups
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }  // one of them

struct TileInfo {
  int s, r0, n_tile, sel, len;
  long grow0;
};
// decode tile t (n-tile fastest, so neighbouring CTAs share A tiles in L2); returns false for tiles with nothing to do
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

// Persistent tile schedule: CTA c walks tiles c, c + grid, ... (skipping tiles with nothing to do).  In clusters of CL
// CTAs (n_tiles == CL), cluster c walks the row tiles c, c + grid / CL, ... and CTA rank r takes column tile r of each.
template <int CL>
struct TileWalk {
  int cur, step, end, n_tiles, rank;
  __device__ TileWalk(int total_tiles, int n_tiles_, int rank_)
      : cur(blockIdx.x / CL), step(gridDim.x / CL), end(total_tiles / CL), n_tiles(n_tiles_), rank(rank_) {}
  __device__ bool next(const TcLinParams& p, TileInfo& ti) {
    while (cur < end) {
      const int id = (p.reverse ? end - 1 - cur : cur) * CL + rank;
      cur += step;
      if (decode_tile(p, id, n_tiles, ti)) return true;
    }
    return false;
  }
};

template <int EPI>
__global__ void __launch_bounds__(LinCfg<EPI>::THREADS, 1) tc_linear_kernel(const __grid_constant__ TcLinParams p) {
  using C = LinCfg<EPI>;
  constexpr int STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES, STG_BOX = C::STG_BOX;
  constexpr bool LN = C::LN;
  // element-wise epilogues: each lane stores its results from registers (vt: through staged TMA stores)
  constexpr bool ELEMWISE = EPI == TEPI_QKV || EPI == TEPI_RESID || EPI == TEPI_F32 || EPI == TEPI_CONV || LN;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // align by OFFSETTING the shared array (not by rebuilding a pointer from an integer): the compiler keeps the
  // shared address space and emits LDS / STS instead of generic LD / ST for everything derived from it.  The offset is
  // the same in both CTAs of a cluster, so a shared address maps to the same variable in the peer (mapa).
  uint8_t* smem = smem_raw + ((1024u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(smem_raw)) & 1023u)) & 1023u);
  uint8_t* s_stg = smem + STAGES * STAGE_BYTES;                        // QKV: [MMA warpgroup][2 vt boxes of STG_BOX bytes]
  float* s_par = reinterpret_cast<float*>(s_stg + C::STG_BYTES);      // tile bias [256] / LayerNorm b, gamma, beta [3][256]
  float* s_red = reinterpret_cast<float*>(s_stg + C::STG_BYTES + C::PAR_BYTES);  // LayerNorm: [pass][128 rows]
  uint64_t* full = reinterpret_cast<uint64_t*>(s_stg + C::STG_BYTES + C::PAR_BYTES + C::RED_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* lnbar = empty + STAGES;  // LayerNorm: [MMA warpgroup][pass] the peer's partial sums have landed in s_red

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int n_tiles = p.n_tiles;
  const int total_tiles = n_tiles * p.st.S * (p.st.Lp / TBM);
  const int iters = p.passes * p.kb_total;  // ring iterations per tile: (pass, K block)
  const uint32_t rank = C::CLUSTER > 1 ? cluster_ctarank() : 0;

  pdl_launch_dependents();  // the next kernel's CTAs may take this SM as soon as this CTA has left it
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.a_hi[0]);
    tma_prefetch_desc(&p.w_hi);
    if (EPI == TEPI_QKV || EPI == TEPI_RESID) tma_prefetch_desc(&p.out_map);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], C::MMA_WARPS); }
    if (LN)  // one arrival per row-owning lane (lane % 4 == 0) of the peer's warpgroup
      for (int i = 0; i < 4; ++i) mbar_init(&lnbar[i], 32);
    fence_barrier_init();
  }
  // LayerNorm: the peer writes into this CTA's shared memory and arrives on its barriers only once both CTAs have
  // initialised theirs.  Every thread of every CTA reaches this barrier, whether or not its cluster gets a tile.
  if (C::CLUSTER > 1) cluster_sync_all();
  else __syncthreads();
  // everything above overlapped the tail of the previous kernel; activations, lengths and stop flags are only read
  // from here on
  pdl_wait();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    regs_dec<40>();
    if (warp == 0 && elect_one()) {
      int g = 0;  // global k-block counter across tiles (ring position)
      TileWalk<C::CLUSTER> walk(total_tiles, n_tiles, rank);
      TileInfo ti;
      while (walk.next(p, ti)) {
        if (EPI == TEPI_RESID)  // the epilogue's residual (x does not fit in L2) comes from HBM while the MMAs run
          for (int c = 0; c < 2 * BN / 16; ++c)
            tma_prefetch_l2_2d(&p.out_map, ti.n_tile * BN + (c % 16) * 16, (int)ti.grow0 + (c / 16) * 64);
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
            if (p.conv_pstride) {
              const int dy = tap / 3, dx = tap % 3;
              arow += ((dy & 1) * 2 + (dx & 1)) * p.conv_pstride + (dy >> 1) * p.conv_w2 + (dx >> 1);
            } else {
              arow += (tap / p.conv_k - p.conv_pad) * p.conv_w2 + (tap % p.conv_k - p.conv_pad);
            }
            kc = (kb % p.conv_cb) * BK;
            seg = 0;
          }
          mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
          tma_load_2d(sa, a_lo ? &p.a_lo[seg] : &p.a_hi[seg], kc, arow, &full[stage]);
          tma_load_3d(sa + C::A_TILE_BYTES, w_lo ? &p.w_lo : &p.w_hi, kb * BK, ti.n_tile * BN, ti.sel, &full[stage]);
        }
      }
    }
    if (C::CLUSTER > 1) {  // the exit barrier (below): the peer may still write into this CTA's shared memory
      __syncwarp();
      cluster_sync_all();
    }
    return;
  }

  // -------------------------------------------------------------------- MMA warpgroups: main loop, then epilogue
  regs_inc<232>();
  const int wg = warp / 4 - 1;   // MMA warpgroup 0 / 1
  const int wq = warp % 4;       // warp inside it: accumulator rows 16 wq .. +15
  const int tq = lane & 3, tr = lane >> 2;
  const uint32_t a_off = wg * 64 * 128;  // this warpgroup's 64 A rows
  const uint32_t b_off = C::A_TILE_BYTES;
  const int mma_n = p.mma_n ? p.mma_n : BN;
  const int rl_a = wg * 64 + wq * 16 + tr;  // tile row of accumulator registers 4 j, 4 j + 1 (+8: 4 j + 2, 4 j + 3)
  auto release = [&](int stage) {  // this warp's MMAs have finished reading the stage
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
  };
  const int mt = threadIdx.x - 128;                // 0 .. 255 over the MMA warpgroups
  const bool issuer = (threadIdx.x & 127) == 0;   // issues this warpgroup's vt TMA stores
  const int rw = wq * 16 + tr;                      // warpgroup row of registers 4 j, 4 j + 1 (+8: 4 j + 2, 4 j + 3)
  uint8_t* stg = s_stg + wg * 2 * STG_BOX;
  uint32_t u = 0;  // vt boxes this warpgroup has staged: box u uses buffer u & 1
  // output columns the element-wise epilogues write
  const int ocols = EPI == TEPI_QKV ? n_tiles * BN
                    : EPI == TEPI_CONV ? p.ldb
                                       : max(p.ldo, p.out_h != nullptr ? p.ldb : 0);
  if (LN) {  // bias, gamma, beta of this CTA's 256 LayerNorm columns: the same for every tile
    const int col = rank * BN + mt;
    s_par[mt] = p.bias[col]; s_par[BN + mt] = p.ln_g[col]; s_par[2 * BN + mt] = p.ln_b[col];
    mma_bar();
  }
  int g = 0;
  uint32_t lt = 0;  // tiles this CTA has finished: the phase of the LayerNorm exchange barriers
  float acc[128];
  TileWalk<C::CLUSTER> walk(total_tiles, n_tiles, rank);
  TileInfo ti;
  while (walk.next(p, ti)) {
    float bias_r = 0.f;  // bias of column mt of this tile, moved to shared memory after the main loop
    if (ELEMWISE && !LN) {
      const int col = ti.n_tile * BN + mt;
      if (col < ocols) bias_r = __ldg(p.bias + (p.w_select == 1 ? (long)ti.sel * p.bias_sel_stride : 0) + col);
    }
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
    if (ELEMWISE && !LN) {  // both warpgroups are done with the previous tile's bias
      mma_bar();
      s_par[mt] = bias_r;
      mma_bar();
    }

    float mean[2] = {0.f, 0.f}, rstd[2] = {0.f, 0.f};  // LayerNorm statistics of rows rl_a, rl_a + 8
    if (LN) {
      // ---------------------------------------------------------------- LayerNorm(512) statistics
      // Two-pass statistics (mean, then squared deviations) over the 512 columns of a row: this CTA's 256 (the quad of
      // lanes that holds the row sums them with two shuffles), plus the peer CTA's.  The quad's lane 0 stores its sum
      // into the peer's s_red[pass][row] through distributed shared memory, arrives on the peer's lnbar[wg][pass]
      // (release at cluster scope), waits on its own (acquire at cluster scope), reads the peer's sum and hands it to
      // its quad.  s_red has a single buffer per pass.  That is safe because the peer overwrites s_red[pass][row] for
      // tile t + 1 only after lane 0 of this quad has read it for tile t:
      //   pass 0 of t + 1 is written after the peer's wait for this lane's pass-1 arrival of tile t,
      //   pass 1 of t + 1 is written after the peer's wait for this lane's pass-0 arrival of tile t + 1,
      // and this lane makes each of those arrivals after its read, in program order.  The same chain keeps each
      // barrier at most one phase ahead of the lanes that wait on it.
      auto exchange = [&](float (&v)[2], int pass) {  // v: this CTA's partial -> slot 0 + slot 1
        float o[2] = {0.f, 0.f};
        if (tq == 0) {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) st_cluster_f32(mapa(s_red + pass * TBM + rl_a + 8 * hr, rank ^ 1), v[hr]);
          mbar_arrive_cluster(mapa(&lnbar[2 * wg + pass], rank ^ 1));
          mbar_wait<true>(&lnbar[2 * wg + pass], lt & 1, p.dbg, 20 + pass, lt);
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) o[hr] = s_red[pass * TBM + rl_a + 8 * hr];
        }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          o[hr] = __shfl_sync(0xffffffffu, o[hr], lane & ~3);
          v[hr] = rank == 0 ? v[hr] + o[hr] : o[hr] + v[hr];
        }
      };
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float2 bb = *reinterpret_cast<const float2*>(s_par + 8 * j + 2 * tq);
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
      }
      exchange(sum, 0);
      float sq[2] = {0.f, 0.f};
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) mean[hr] = sum[hr] * (1.f / LG_FFN);
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
      }
      exchange(sq, 1);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) rstd[hr] = rsqrtf(sq[hr] * (1.f / LG_FFN) + 1e-5f);
      ++lt;
    }

    constexpr bool GATED = EPI == TEPI_TOP2_H || EPI == TEPI_TOP2_F;
    constexpr int GATE_FIELDS = EPI == TEPI_TOP2_F ? 6 : 2;
    if (EPI == TEPI_TOP2 || GATED) {
      // ---------------------------------------------------------------- nearest-neighbour sweep (nn_api.cu)
      // per row and per 128-column slot of live partner columns: the best similarity s1, its column j1 (ascending
      // columns: the first maximum wins) and the best over the slot's other columns s2 (equal to s1 on a tie)
      const int lens = p.st.len[ti.sel];
      // Guided sweeps: only the columns whose gate passes enter the top-2.  The gate records of the tile's 256 partner
      // columns are staged in shared memory, one array per field (s_stg is sized for them in this epilogue); the
      // tile's own rows read theirs from global memory.  A pair that is not guided takes the ungated path: the flag is
      // uniform per tile, so both MMA warpgroups meet the same barriers.
      float* s_rec = reinterpret_cast<float*>(s_stg);  // [GATE_FIELDS][BN]
      const long rec_rows = (long)p.st.S * p.st.Lp;
      bool gate_on = false;
      if (GATED) {
        gate_on = p.gate_on[ti.s >= p.st.B ? ti.s - p.st.B : ti.s] != 0;
        if (gate_on) {
          const int col = ti.n_tile * BN + mt;
          mma_bar();  // both warpgroups are done with the previous tile's records
#pragma unroll
          for (int f = 0; f < GATE_FIELDS; ++f)
            s_rec[f * BN + mt] = col < p.st.Lp ? __ldg(p.gate_rec + f * rec_rows + (long)ti.sel * p.st.Lp + col) : 0.f;
          mma_bar();
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int rl = rl_a + 8 * hr;
        const long grow = ti.grow0 + rl;
        const bool live = ti.r0 + rl < ti.len;
        float rr[GATE_FIELDS];  // this row's gate record
#pragma unroll
        for (int f = 0; f < GATE_FIELDS; ++f) rr[f] = GATED && gate_on ? __ldg(p.gate_rec + f * rec_rows + grow) : 0.f;
        // include/nn_b200.h: step 5 of include/geometry_b200.h in fp32 with every operation rounded on its own.  Both
        // forms are symmetric in the two records, so the direction of the sweep does not enter: H squares the
        // difference of the projected point and the point (b - a = -(a - b) exactly); F takes the fmaxf of the two
        // point-to-line terms, each record holding its point and its line in the other image.
        auto gate = [&](int cl) -> bool {
          const float* cr = s_rec + cl;
          float err;
          if constexpr (EPI != TEPI_TOP2_F) {
            const float dx = __fsub_rn(rr[0], cr[0]), dy = __fsub_rn(rr[1], cr[BN]);
            err = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
          } else {
            // record: x, y, a, b, c, s = 1 / (a^2 + b^2) with (a, b, c) the point's epipolar line
            auto term = [](float px, float py, float a, float b, float c, float s) {
              const float d = __fadd_rn(__fadd_rn(__fmul_rn(px, a), __fmul_rn(py, b)), c);
              return __fmul_rn(__fmul_rn(d, d), s);
            };
            err = fmaxf(term(cr[0], cr[BN], rr[2], rr[3], rr[4], rr[5]),
                        term(rr[0], rr[1], cr[2 * BN], cr[3 * BN], cr[4 * BN], cr[5 * BN]));
          }
          return err < p.gate_t2;  // NaN fails
        };
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int col0 = ti.n_tile * BN + half * 128;
          const int ncols = lens - col0;
          float b1 = -INFINITY, b2 = -INFINITY;
          int a1 = INT_MAX;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * jj + 2 * tq + e;
              const float v = acc[4 * (16 * half + jj) + 2 * hr + e];
              if (c < ncols && (!GATED || !gate_on || gate(half * 128 + c))) {
                if (v > b1) { b2 = b1; b1 = v; a1 = col0 + c; }
                else b2 = fmaxf(b2, v);
              }
            }
          // merge over the quad of lanes that holds the row: (value descending, index ascending)
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) {
            const float ob1 = __shfl_xor_sync(0xffffffffu, b1, o), ob2 = __shfl_xor_sync(0xffffffffu, b2, o);
            const int oa1 = __shfl_xor_sync(0xffffffffu, a1, o);
            if (ob1 > b1 || (ob1 == b1 && oa1 < a1)) { b2 = fmaxf(b1, ob2); b1 = ob1; a1 = oa1; }
            else b2 = fmaxf(b2, ob1);
          }
          if (live && tq == 0) {
            const long at = grow * p.part_stride + ti.n_tile * 2 + half;
            reinterpret_cast<float2*>(p.part)[at] = make_float2(b1, b2);
            p.part_arg[at] = a1;
          }
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

    // ------------------------------------------------------------------ element-wise epilogues, direct stores
    // Each lane applies the epilogue arithmetic to its accumulator pairs, element by element, the quad of lanes that
    // holds a row transposes each 32-column chunk (quad_transpose), and every lane then writes 8 consecutive columns of
    // its row with 16-byte stores: one warp store instruction covers 8 rows x 64 contiguous bytes, whole 32-byte sectors.
    // Rows need no bound: Lp is a multiple of the 128-row tile, so every tile lies inside the S Lp rows.  Chunk loops are
    // unrolled so that the accumulators stay in registers.
    const int row0 = (int)ti.grow0 + wg * 64;  // first row of this warpgroup
    if (EPI == TEPI_QKV) {
      // which output a QKV tile feeds: packed channel order [q | k | v] (self) or [qk | v] (cross)
      const int which = ti.n_tile;
      const bool qkv_v = p.rope ? which == 2 : which == 1;
      if (qkv_v) {
        // V is stored transposed [S, H, 64, Lp] (K-major B operand of P*V): each warpgroup writes a head at a time into a
        // shared-memory box [64 d][64 rows] (128-byte swizzle, as the store map declares) that its issuer thread stores
        // with TMA once every writer has fenced it; a box is rewritten only after the store that read it two boxes
        // earlier has finished reading.  Padding rows are written as zeros: attention multiplies them by P = 0, which
        // stays 0 whatever x held there.
#pragma unroll
        for (int hh = 0; hh < BN / LG_HDIM; ++hh) {
          if (issuer) bulk_wait_read<1>();
          wg_bar(wg);
          uint8_t* box = stg + (u & 1) * STG_BOX;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int row = rw + 8 * hr;
            const bool live = ti.r0 + wg * 64 + row < ti.len;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * hh + jj, d = 8 * jj + 2 * tq;
              const float2 bb = *reinterpret_cast<const float2*>(s_par + 8 * j + 2 * tq);
              float v0 = acc[4 * j + 2 * hr] + bb.x, v1 = acc[4 * j + 2 * hr + 1] + bb.y;
              if (!live) v0 = v1 = 0.f;
              *reinterpret_cast<__half*>(box + swz(d * 128 + row * 2, 0x70)) = __float2half_rn(v0);
              *reinterpret_cast<__half*>(box + swz((d + 1) * 128 + row * 2, 0x70)) = __float2half_rn(v1);
            }
          }
          fence_proxy_async();
          wg_bar(wg);
          if (issuer) {
            tma_store_2d(&p.out_map, box, ti.r0 + wg * 64, (ti.s * LG_HEADS + hh) * LG_HDIM);
            bulk_commit();
          }
          ++u;
        }
        continue;
      }
      // q / k: [S, H, Lp, 64] fp16, a row's 64 d of a head are 128 contiguous bytes.  RoPE cos / sin of the two rows,
      // loaded before the stores; frequency index d / 2 = 4 (j % 8) + tq, the same for every head
      float rc[2][8], rs[2][8];
      if (p.rope) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const long grow = ti.grow0 + rl_a + 8 * hr;
            rc[hr][jj] = __ldg(p.cs + grow * 64 + 4 * jj + tq);
            rs[hr][jj] = __ldg(p.cs + grow * 64 + 32 + 4 * jj + tq);
          }
      }
      __half* out = which == 0 ? p.q : p.k;
#pragma unroll
      for (int hh = 0; hh < BN / LG_HDIM; ++hh)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          __half* orow = out + ((long)(ti.s * LG_HEADS + hh) * p.st.Lp + ti.r0 + wg * 64 + rw + 8 * hr) * LG_HDIM;
#pragma unroll
          for (int ch = 0; ch < 2; ++ch) {  // 32 d of the head
            uint32_t w[4][1];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int jj = 4 * ch + i, j = 8 * hh + jj;
              const float2 bb = *reinterpret_cast<const float2*>(s_par + 8 * j + 2 * tq);
              float v0 = acc[4 * j + 2 * hr] + bb.x, v1 = acc[4 * j + 2 * hr + 1] + bb.y;
              if (p.rope) {  // rotary embedding on q / k (lightglue.py:58-65, 168-169); freq index = d / 2
                const float c = rc[hr][jj], s = rs[hr][jj];
                const float a = v0, b = v1;
                v0 = a * c - b * s;
                v1 = b * c + a * s;
              }
              const __half2 h2 = __floats2half2_rn(v0, v1);
              w[i][0] = *reinterpret_cast<const uint32_t*>(&h2);
            }
            quad_transpose(w, tq);
            st_v4(orow + 32 * ch + 8 * tq, w[0][0], w[1][0], w[2][0], w[3][0]);
          }
        }
      continue;
    }

    // bias (* scale) (+ ReLU) (+ residual) -> fp32 and / or bf16 hi (/ lo), or LayerNorm + GELU -> bf16 hi (/ lo).
    // Column bounds: fp32 columns < ldo (a multiple of 4), bf16 columns < ldb (a multiple of 8), both checked by tc_gemm,
    // so each 16-byte store is wholly inside or outside.
    const bool f32out = EPI == TEPI_RESID || EPI == TEPI_F32;
    const bool has16 = EPI == TEPI_CONV || EPI == TEPI_RESID || LN || (EPI == TEPI_F32 && p.out_h != nullptr);
    const bool haslo = has16 && p.out_l != nullptr;
    const int cbase = ti.n_tile * BN;
    const int nch = (min(BN, ocols - cbase) + 31) / 32;  // 32-column chunks with columns to write
    bool inside[2] = {true, true};
    if (EPI == TEPI_CONV) {  // the padding pixels of the NHWC image stay zero for the next layer's taps
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long grow = ti.grow0 + rl_a + 8 * hr;
        const long pp = grow % p.conv_plane;
        const int yy = (int)(pp / p.conv_w2), xx = (int)(pp % p.conv_w2);
        inside[hr] = grow < p.conv_rows && yy >= p.conv_pad && yy < p.conv_h + p.conv_pad && xx >= p.conv_pad &&
                     xx < p.conv_w + p.conv_pad;
      }
    }
    // TEPI_RESID: the residual x of this lane's 8 columns of both rows (L2-resident: the producer prefetched the tile's
    // x), loaded one chunk ahead of the chunk being stored
    float4 xc[2][2], xn[2][2];
    auto load_x = [&](int ch, float4 (&xv)[2][2]) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int col = cbase + 32 * ch + 8 * tq + 4 * h;
          xv[hr][h] = col < p.ldo ? *reinterpret_cast<const float4*>(p.out_f32 + (long)(row0 + rw + 8 * hr) * p.ldo + col)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    if (EPI == TEPI_RESID) load_x(0, xc);
#pragma unroll
    for (int ch = 0; ch < BN / 32; ++ch) {
      if (ch >= nch) break;
      if (EPI == TEPI_RESID && ch + 1 < nch) load_x(ch + 1, xn);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        uint32_t w[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int j = 4 * ch + i;  // accumulator column group
          float v0, v1;
          if (LN) {  // the bias is in acc already (statistics above)
            const float2 gg = *reinterpret_cast<const float2*>(s_par + BN + 8 * j + 2 * tq);
            const float2 be = *reinterpret_cast<const float2*>(s_par + 2 * BN + 8 * j + 2 * tq);
            v0 = gelu_erf(fmaf((acc[4 * j + 2 * hr] - mean[hr]) * rstd[hr], gg.x, be.x));
            v1 = gelu_erf(fmaf((acc[4 * j + 2 * hr + 1] - mean[hr]) * rstd[hr], gg.y, be.y));
          } else {
            const float2 bb = *reinterpret_cast<const float2*>(s_par + 8 * j + 2 * tq);
            v0 = acc[4 * j + 2 * hr] + bb.x; v1 = acc[4 * j + 2 * hr + 1] + bb.y;
            if (p.scale != 1.f) { v0 *= p.scale; v1 *= p.scale; }
          }
          if (EPI == TEPI_CONV) {
            v0 = inside[hr] ? ((p.relu && v0 < 0.f) ? 0.f : v0) : 0.f;
            v1 = inside[hr] ? ((p.relu && v1 < 0.f) ? 0.f : v1) : 0.f;
          }
          w[i][0] = __float_as_uint(v0); w[i][1] = __float_as_uint(v1);
        }
        quad_transpose(w, tq);  // lane tq: columns 32 ch + 8 tq .. +7 of the tile
        float v[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) { v[2 * i] = __uint_as_float(w[i][0]); v[2 * i + 1] = __uint_as_float(w[i][1]); }
        if (EPI == TEPI_RESID) {  // x + ffn(...) (lightglue.py:172 / 228-229)
          const float4 a = xc[hr][0], b = xc[hr][1];
          v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
        }
        const long grow = row0 + rw + 8 * hr;
        const int col = cbase + 32 * ch + 8 * tq;
        if (f32out) {
          // 8 fp32 columns are one 32-byte sector, two 16-byte stores: lanes tq and tq ^ 1 swap halves so that each
          // store instruction writes whole sectors.  Lane tq then holds columns 4 (tq & 1) .. +3 of the groups tq & ~1
          // (a) and tq | 1 (b).
          const bool odd = tq & 1;
          uint32_t a[4], b[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t got = __shfl_xor_sync(0xffffffffu, __float_as_uint(odd ? v[k] : v[4 + k]), 1);
            a[k] = odd ? got : __float_as_uint(v[k]);
            b[k] = odd ? __float_as_uint(v[4 + k]) : got;
          }
          const int ca = cbase + 32 * ch + 8 * (tq & ~1) + 4 * odd, cb = ca + 8;
          float* o = p.out_f32 + grow * p.ldo;
          if (ca < p.ldo) st_v4(o + ca, a[0], a[1], a[2], a[3]);
          if (cb < p.ldo) st_v4(o + cb, b[0], b[1], b[2], b[3]);
        }
        if (has16 && col < p.ldb) {
          uint32_t hi[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) hi[i] = pack_bf16x2(v[2 * i], v[2 * i + 1]);
          st_v4(p.out_h + grow * p.ldb + col, hi[0], hi[1], hi[2], hi[3]);
          if (haslo)
            st_v4(p.out_l + grow * p.ldb + col, pack_bf16x2_lo(v[0], v[1], hi[0]), pack_bf16x2_lo(v[2], v[3], hi[1]),
                  pack_bf16x2_lo(v[4], v[5], hi[2]), pack_bf16x2_lo(v[6], v[7], hi[3]));
        }
      }
      if (EPI == TEPI_RESID) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) { xc[hr][0] = xn[hr][0]; xc[hr][1] = xn[hr][1]; }
      }
    }
  }
  // the vt stores must be complete (not only read) when the grid ends: the next kernel's griddepcontrol.wait relies on
  // it.  The direct stores are plain global stores, which the grid's completion covers.
  if (EPI == TEPI_QKV && issuer) bulk_wait_all();
  if (C::CLUSTER > 1) {  // neither CTA of a cluster exits while the other may still write into its shared memory
    __syncwarp();
    cluster_sync_all();
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

template <int EPI>
int launch_linear_t(const TcLinParams& p, cudaStream_t stream) {
  using C = LinCfg<EPI>;
  const int total = p.n_tiles * p.st.S * (p.st.Lp / TBM);
  int slots = lg_num_sms();  // co-resident CTAs, or clusters: how the SMs of the device split into clusters varies
  if (C::CLUSTER > 1) {
    if (p.n_tiles != C::CLUSTER) return lg_set_error("launch_linear: a cluster kernel needs one column tile per CTA");
    if (int r = lg_max_clusters((const void*)tc_linear_kernel<EPI>, C::THREADS, C::SMEM, C::CLUSTER, &slots)) return r;
  }
  const int units = total / C::CLUSTER;
  const int grid = (units < slots ? units : slots) * C::CLUSTER;
  return tc_launch(tc_linear_kernel<EPI>, dim3(grid), C::THREADS, C::SMEM, p, stream, C::CLUSTER);
}
int launch_linear(const TcLinParams& p, cudaStream_t stream) {
  switch (p.epi) {
    case TEPI_QKV: return launch_linear_t<TEPI_QKV>(p, stream);
    case TEPI_LN_GELU: return launch_linear_t<TEPI_LN_GELU>(p, stream);
    case TEPI_RESID: return launch_linear_t<TEPI_RESID>(p, stream);
    case TEPI_F32: return launch_linear_t<TEPI_F32>(p, stream);
    case TEPI_CONV: return launch_linear_t<TEPI_CONV>(p, stream);
    case TEPI_LSE: return launch_linear_t<TEPI_LSE>(p, stream);
    case TEPI_ARGMAX: return launch_linear_t<TEPI_ARGMAX>(p, stream);
    case TEPI_TOP2: return launch_linear_t<TEPI_TOP2>(p, stream);
    case TEPI_TOP2_H: return launch_linear_t<TEPI_TOP2_H>(p, stream);
    case TEPI_TOP2_F: return launch_linear_t<TEPI_TOP2_F>(p, stream);
  }
  return lg_set_error("launch_linear: bad epilogue");
}

// Operands of one GEMM.  A = [A0 | A1] along K, each [st.S * st.Lp rows, k] bf16 row-major; W = nsel matrices [nout, K]
// bf16 (K = k0 + k1, or k^2 k0 for a k x k convolution), sel_stride elements apart.  The lo images are read in bf16x3 only.
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
  const uint64_t K = p.conv_cb ? (uint64_t)p.conv_k * p.conv_k * d.k0 : d.k0 + d.k1, nout = d.nout, nsel = d.nsel;
  const uint64_t sel_bytes = (nsel > 1 ? d.sel_stride : nout * K) * 2;
  const uint64_t arows = p.conv_arows ? (uint64_t)p.conv_arows : rows;
  auto amap = [&](CUtensorMap* out, const void* a, uint64_t k) {  // box 64 x the tile height
    return tc_tmap(e, {a, 2, {k, arows}, {k * 2}, {BK, TBM}}, out);
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
  if (p.epi == TEPI_QKV) {  // the vt store map (64-row boxes)
    const uint64_t sh = (uint64_t)st.S * LG_HEADS;
    if ((r = tc_tmap(e, {p.vt, 2, {(uint64_t)st.Lp, sh * LG_HDIM}, {(uint64_t)st.Lp * 2}, {64, LG_HDIM}}, &p.out_map)))
      return r;
  } else if (p.epi == TEPI_RESID || p.epi == TEPI_F32 || p.epi == TEPI_CONV || p.epi == TEPI_LN_GELU) {
    // the epilogue writes 16-byte vectors: 4 fp32 or 8 bf16 columns, at row starts on 16-byte boundaries
    auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (p.out_f32 && (p.ldo % 4 != 0 || !aligned(p.out_f32)))
      return lg_set_error("tc_gemm: an fp32 output needs ldo % 4 == 0 and a 16-byte aligned base");
    if ((p.out_h || p.out_l) && (p.ldb % 8 != 0 || !aligned(p.out_h) || !aligned(p.out_l)))
      return lg_set_error("tc_gemm: a bf16 output needs ldb % 8 == 0 and 16-byte aligned bases");
    if (p.epi == TEPI_RESID) {  // the producer prefetches each tile's residual x to L2 through this map
      const uint64_t ldo = p.ldo;
      if ((r = tc_tmap(e, {p.out_f32, 2, {ldo, rows}, {ldo * 4}, {16, 64}, CU_TENSOR_MAP_SWIZZLE_64B,
                           CU_TENSOR_MAP_DATA_TYPE_FLOAT32}, &p.out_map)))
        return r;
    }
  }
  p.kb_total = (int)(K / BK);
  p.kb0 = d.k1 ? d.k0 / BK : p.kb_total;
  p.passes = e.x3 ? 3 : 1;
  p.n_tiles = n_tiles;
  p.st = st;
  p.dbg = e.dbg;
  return launch_linear(p, stream);
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
      if ((r = tc_gemm(h->tc, st, ops, ntc, p, stream))) return r;
    }
    if (sweep == 0 && (r = misc_assign_term(a, st, part, 2 * ntc, BN / 2, term, stream))) return r;
  }
  if (logmat) LG_RC(misc_assign_dustbin(a, st, stream));
  return misc_assign_tail(a, st, part, part_arg, 2 * ntc, BN / 2, stream);
}

// Nearest-neighbour sweep: S = d_s d_partner^T of every sequence in split-bf16 (hi / lo [st.S * st.Lp, dim]), per row the
// top-2 partials of every 128-column slot into part (float2) / part_arg, [st.S * st.Lp, pstride]
int tc_nn_sweep(TcEngine& e, const SeqState& st, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int dim, float* part,
                int* part_arg, int pstride, cudaStream_t stream, const TcNnGate* gate) {
  if (dim % BK != 0) return lg_set_error("tc_nn_sweep: the descriptor size must be a multiple of 64");
  const int ntc = (st.Lp + BN - 1) / BN;
  if (pstride < 2 * ntc) return lg_set_error("tc_nn_sweep: slot stride too small");
  const TcOperands ops{hi, lo, dim, nullptr, nullptr, 0, hi, lo, st.Lp, st.S, (size_t)st.Lp * dim};
  TcLinParams p{};
  p.epi = TEPI_TOP2; p.scale = 1.f;
  p.part = part; p.part_arg = part_arg; p.part_stride = pstride;
  p.w_select = 2;
  if (gate) {
    p.epi = gate->fundamental ? TEPI_TOP2_F : TEPI_TOP2_H;
    p.gate_rec = gate->rec; p.gate_on = gate->on; p.gate_t2 = gate->t2;
  }
  return tc_gemm(e, st, ops, ntc, p, stream);
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
  cudaError_t err;
  if (n) {  // n = 0: an engine without weights (both operands are activations)
    err = cudaMalloc(&e->w_hi, n * sizeof(__nv_bfloat16));
    if (err != cudaSuccess) return lg_set_cuda_error(err, __FILE__, __LINE__);
    err = cudaMalloc(&e->w_lo, n * sizeof(__nv_bfloat16));
    if (err != cudaSuccess) return lg_set_cuda_error(err, __FILE__, __LINE__);
    split_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(w, e->w_hi, e->w_lo, n);
    LG_CHECK_LAUNCH();
  }
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

void tc_carve(WsBump& w, size_t S, int Lp, const LgHandle* h, TcBuffers* b) {
  const size_t R = S * Lp;
  const bool x3 = h->cfg.precision == LG_PREC_BF16X3;
  constexpr size_t A = 1024;  // every buffer on a 1024-byte boundary
  b->xh = w.take<__nv_bfloat16>(R * 256, A);
  b->xl = x3 ? w.take<__nv_bfloat16>(R * 256, A) : nullptr;
  b->ctxh = w.take<__nv_bfloat16>(R * 256, A);
  b->ctxl = x3 ? w.take<__nv_bfloat16>(R * 256, A) : nullptr;
  b->msgh = w.take<__nv_bfloat16>(R * 256, A);
  b->msgl = x3 ? w.take<__nv_bfloat16>(R * 256, A) : nullptr;
  b->hh = w.take<__nv_bfloat16>(R * 512, A);
  b->hl = x3 ? w.take<__nv_bfloat16>(R * 512, A) : nullptr;
  b->q = w.take<__half>(R * 256, A);
  b->k = w.take<__half>(R * 256, A);
  b->vt = w.take<__half>(R * 256, A);
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
  TcLinParams p{};
  p.epi = TEPI_F32; p.scale = 1.f; p.bias = h->wpk + h->o_inb;
  p.out_f32 = x; p.ldo = LG_DIM; p.out_h = b.xh; p.out_l = b.xl; p.ldb = LG_DIM;
  const TcOperands ops{b.hh, b.hl, d, nullptr, nullptr, 0, h->tc.w_hi + h->o_inw, h->tc.w_lo + h->o_inw, LG_DIM, 1, 0};
  return tc_gemm(h->tc, st, ops, 1, p, stream);
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
  return tc_gemm(h->tc, st, ops, 1, p, stream);
}

namespace {
int conv_launch(TcEngine& e, const SeqState& st, const __nv_bfloat16* in_h, const __nv_bfloat16* in_l, int cin, int taps,
                size_t w_off, const float* bias, int relu, int B, int H, int W, __nv_bfloat16* out_h, __nv_bfloat16* out_l, int cout,
                float* out_f32, int ldo, int pstride, cudaStream_t stream) {
  TcLinParams p{};
  p.conv_pstride = pstride;
  p.conv_arows = pstride ? 4L * pstride : 0;
  p.epi = out_f32 ? TEPI_F32 : TEPI_CONV;
  p.scale = 1.f; p.bias = bias; p.relu = relu;
  p.out_f32 = out_f32; p.ldo = ldo; p.out_h = out_h; p.out_l = e.x3 ? out_l : nullptr; p.ldb = cout;
  const int mma_n = cout <= 64 ? 64 : cout <= 128 ? 128 : BN;  // no MMA columns for the zero rows of a narrow layer
  p.mma_n = mma_n == BN ? 0 : mma_n;
  p.conv_cb = taps > 1 ? cin / BK : 0;
  p.conv_k = taps == 25 ? 5 : 3;
  p.conv_pad = p.conv_k / 2;  // 1x1: the 3x3 layout (SuperPoint's heads read the padded maps of their 3x3 inputs)
  p.conv_w2 = W + 2 * p.conv_pad; p.conv_h = H; p.conv_w = W;
  p.conv_plane = (long)(H + 2 * p.conv_pad) * p.conv_w2; p.conv_rows = (long)B * p.conv_plane;
  const TcOperands ops{in_h, in_l, cin, nullptr, nullptr, 0, e.w_hi + w_off, e.w_lo + w_off, BN, 1, 0};
  return tc_gemm(e, st, ops, 1, p, stream);
}
}  // namespace

int tc_conv(TcConvWeights& cw, const SeqState& st, const TcConvArgs& a, cudaStream_t stream) {
  if (a.cin % BK != 0 || (a.taps != 1 && a.taps != 9 && a.taps != 25))
    return lg_set_error("tc_conv: Cin must be a multiple of 64, 1x1, 3x3 or 5x5");
  if (a.pstride < 0 || (a.pstride > 0 && a.taps != 9))
    return lg_set_error("tc_conv: a stride-2 convolution is 3x3 and its phase stride positive");
  return conv_launch(cw.tc, st, a.in_h, a.in_l, a.cin, a.taps, cw.w_off[a.region], cw.wpk + cw.b_off[a.region], a.relu, a.B, a.H,
                     a.W, a.out_h, a.out_l, a.cout, a.out_f32, a.ldo, a.pstride, stream);
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
    int r = tc_gemm(h->tc, st, ops, nout / BN, p, stream);
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
    int r = tc_gemm(h->tc, st, ops, LG_FFN / BN, p, stream);  // one 2-CTA cluster per 128 rows: the whole LayerNorm row
    if (r) return r;
  }
  {  // ffn.3 + residual -> x (fp32 master + bf16 shadows)
    TcLinParams p{};
    p.epi = TEPI_RESID; p.scale = 1.f; p.bias = bw + o.b2; p.out_f32 = x; p.ldo = LG_DIM;
    p.out_h = b.xh; p.out_l = b.xl; p.ldb = LG_DIM;
    const TcOperands ops{b.hh, b.hl, LG_FFN, nullptr, nullptr, 0, wh + o.w2, wl + o.w2, LG_DIM, 1, 0};
    Timer t2(h, LG_K_FFN3, stream);
    int r = tc_gemm(h->tc, st, ops, 1, p, stream);
    if (r) return r;
  }
  return 0;
}
