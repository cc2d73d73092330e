// wgmma flash attention for the tensor-core path (lightglue.py:113-137: softmax(q k^T / 8) v, no mask).
//
// One CTA owns 128 query rows of one (sequence, head) and sweeps the key/value sequence in blocks of 64:
//   S = Q K_j^T            wgmma m64n64k16, Q and K in shared memory (TMA, 128B swizzle), S in registers
//   P = exp2(c S - c m)    online softmax in registers (running row maximum m, rows reduced over quads of lanes)
//   O = alpha O + P V_j    wgmma m64n64k16, A = P as fp16 from registers, B = V^T tile in shared memory
// The denominator is summed per thread and reduced once at the end; one division per row.
// Warp roles (384 threads = 3 warpgroups): warpgroup 0 = TMA producer (warp 0; the warpgroup hands its registers to
// the others), warpgroups 1 and 2 = query rows 0-63 / 64-127 of the CTA.  ~80 KB of shared memory, so two CTAs are
// resident per SM and one CTA's exponentials overlap the other's MMAs.
#include "lg_handle.h"
#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int QT = 128;          // query rows per CTA
constexpr int KB = 64;           // keys per block
constexpr int KV_STAGES = 4;
constexpr int Q_TILE_BYTES = QT * 64 * 2;                // 16 KB
constexpr int K_TILE_BYTES = KB * 64 * 2;                // 8 KB
constexpr int V_TILE_BYTES = 64 * KB * 2;                // [64 d rows][64 keys], 8 KB
constexpr int STAGE_BYTES = K_TILE_BYTES + V_TILE_BYTES;  // 16 KB
constexpr int SMEM_BYTES = Q_TILE_BYTES + KV_STAGES * STAGE_BYTES + 1024 + 256;
constexpr float SCALE_LOG2 = 0.125f * 1.4426950408889634f;  // dh^-0.5 * log2(e)

struct AttnParams {
  CUtensorMap q_map;   // (64, Lp, S*H)   box (64, 128, 1)
  CUtensorMap k_map;   // (64, Lp, S*H)   box (64, 64, 1)
  CUtensorMap vt_map;  // (Lp, 64, S*H)   box (64, 64, 1)
  __nv_bfloat16* ctxh; __nv_bfloat16* ctxl;
  int kv_shift;
  SeqState st;
  unsigned int* dbg;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {  // a -> low half
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(384, 2) tc_attention_kernel(const __grid_constant__ AttnParams p) {
  pdl_launch_dependents();
  pdl_wait();  // the sequence lengths read right below belong to the dependency chain
  const int s = blockIdx.z, h = blockIdx.y, r0 = blockIdx.x * QT;
  const int len_q = p.st.len[s];
  if (r0 >= len_q || lg_pair_stopped(p.st, s)) return;
  const int skv = (s + p.kv_shift) % p.st.S;
  const int len_kv = p.st.len[skv];
  const int nkv = (len_kv + KB - 1) / KB;
  const int nwg = len_q - r0 > 64 ? 2 : 1;  // MMA warpgroups with live query rows

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(smem_raw)) & 1023u)) & 1023u);
  uint8_t* sq = smem;                   // 16 KB
  uint8_t* skvb = smem + Q_TILE_BYTES;  // KV_STAGES x 16 KB
  uint64_t* q_full = reinterpret_cast<uint64_t*>(skvb + KV_STAGES * STAGE_BYTES);
  uint64_t* kv_full = q_full + 1;
  uint64_t* kv_empty = kv_full + KV_STAGES;

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.q_map);
    tma_prefetch_desc(&p.k_map);
    tma_prefetch_desc(&p.vt_map);
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 4 * nwg); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_dec<24>();
    if (warp == 0 && nkv > 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, Q_TILE_BYTES);
      tma_load_3d(sq, &p.q_map, 0, r0, s * LG_HEADS + h, q_full);
      for (int j = 0; j < nkv; ++j) {
        const int stage = j % KV_STAGES, round = j / KV_STAGES;
        mbar_wait(&kv_empty[stage], (round & 1) ^ 1, p.dbg, 1, j);
        uint8_t* dst = skvb + stage * STAGE_BYTES;
        mbar_arrive_expect_tx(&kv_full[stage], STAGE_BYTES);
        tma_load_3d(dst, &p.k_map, 0, j * KB, skv * LG_HEADS + h, &kv_full[stage]);
        tma_load_3d(dst + K_TILE_BYTES, &p.vt_map, j * KB, 0, skv * LG_HEADS + h, &kv_full[stage]);
      }
    }
    return;
  }
  regs_inc<104>();
  const int wg = warp / 4 - 1;
  if (wg >= nwg) return;
  const int tq = lane & 3, tr = lane >> 2;
  const int ra = r0 + wg * 64 + (warp % 4) * 16 + tr;  // query row of accumulator registers 4 j, 4 j + 1 (+8: 4 j + 2, 4 j + 3)
  if (nkv == 0) {  // no keys: the context is zero
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      if (ra + 8 * hr >= len_q) continue;
      const long off = ((long)s * p.st.Lp + ra + 8 * hr) * LG_DIM + h * LG_HDIM;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(p.ctxh + off + 8 * j + 2 * tq) = 0u;
        if (p.ctxl) *reinterpret_cast<uint32_t*>(p.ctxl + off + 8 * j + 2 * tq) = 0u;
      }
    }
    return;
  }

  const uint64_t qdesc = make_sdesc_sw128(smem_u32(sq + wg * 64 * 128));
  const uint64_t kdesc0 = make_sdesc_sw128(smem_u32(skvb));
  const uint64_t vdesc0 = make_sdesc_sw128(smem_u32(skvb + K_TILE_BYTES));
  float o[32], sv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  mbar_wait(q_full, 0, p.dbg, 2);
  for (int j = 0; j < nkv; ++j) {
    const int stage = j % KV_STAGES;
    mbar_wait(&kv_full[stage], (j / KV_STAGES) & 1, p.dbg, 3, j);
    const uint64_t kdesc = kdesc0 + (uint64_t)(stage * (STAGE_BYTES >> 4));
    const uint64_t vdesc = vdesc0 + (uint64_t)(stage * (STAGE_BYTES >> 4));
    fence_regs(sv);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_f16_n64_ss(sv, qdesc + 2 * k, kdesc + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sv);
    const int valid = len_kv - j * KB;
    if (valid < KB) {  // keys past the end of the sequence do not exist
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * jj + 2 * tq + (e & 1) >= valid) sv[4 * jj + e] = -INFINITY;
    }
    // online softmax; the row maximum of the block is reduced over the quad of lanes holding the row
    uint32_t pa[16];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = m[hr];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * hr], sv[4 * jj + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float alpha = ex2((m[hr] - mx) * SCALE_LOG2);  // 0 in the first block (m = -inf)
      m[hr] = mx;
      const float nmc = -mx * SCALE_LOG2;
      float bs = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float e0 = ex2(fmaf(sv[4 * jj + 2 * hr], SCALE_LOG2, nmc));
        const float e1 = ex2(fmaf(sv[4 * jj + 2 * hr + 1], SCALE_LOG2, nmc));
        bs += e0 + e1;
        // A fragment of key slice jj / 2: registers {row a, cols 0-7}, {row b, 0-7}, {row a, 8-15}, {row b, 8-15}
        pa[4 * (jj / 2) + 2 * (jj & 1) + hr] = pack_half2(e0, e1);
      }
      l[hr] = l[hr] * alpha + bs;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) { o[4 * jj + 2 * hr] *= alpha; o[4 * jj + 2 * hr + 1] *= alpha; }
    }
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint32_t a4[4] = {pa[4 * ks], pa[4 * ks + 1], pa[4 * ks + 2], pa[4 * ks + 3]};
      wgmma_f16_n64_rs(o, a4, vdesc + 2 * ks);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[stage]);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float lt = l[hr];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = lt > 0.f ? 1.f / lt : 0.f;
    const int r = ra + 8 * hr;
    if (r >= len_q) continue;
    const long off = ((long)s * p.st.Lp + r) * LG_DIM + h * LG_HDIM;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float a = o[4 * jj + 2 * hr] * inv, b = o[4 * jj + 2 * hr + 1] * inv;
      const uint32_t hi = pack_bf16x2(a, b);
      *reinterpret_cast<uint32_t*>(p.ctxh + off + 8 * jj + 2 * tq) = hi;
      if (p.ctxl) *reinterpret_cast<uint32_t*>(p.ctxl + off + 8 * jj + 2 * tq) = pack_bf16x2_lo(a, b, hi);
    }
  }
}

}  // namespace

int tc_attention(LgHandle* h, const TcBuffers& b, const SeqState& st, int kv_shift, const __half* kbuf, cudaStream_t stream) {
  const uint64_t SH = (uint64_t)st.S * LG_HEADS, Lp = st.Lp;
  AttnParams p;
  int r;
  if ((r = tc_tmap(h->tc, {b.q, 3, {64, Lp, SH}, {128, Lp * 128}, {64, QT, 1}}, &p.q_map))) return r;
  if ((r = tc_tmap(h->tc, {kbuf, 3, {64, Lp, SH}, {128, Lp * 128}, {64, KB, 1}}, &p.k_map))) return r;
  if ((r = tc_tmap(h->tc, {b.vt, 3, {Lp, 64, SH}, {Lp * 2, 64 * Lp * 2}, {64, 64, 1}}, &p.vt_map))) return r;
  p.ctxh = b.ctxh; p.ctxl = b.ctxl; p.kv_shift = kv_shift; p.st = st; p.dbg = h->tc.dbg;
  return tc_launch(tc_attention_kernel, dim3(st.Lp / QT, LG_HEADS, st.S), 384, SMEM_BYTES, p, stream);
}
