// Tensor-core (wgmma / TMA) path: LG_PREC_BF16 and LG_PREC_BF16X3.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "lg_internal.h"
#include "ws_bump.h"

struct LgHandle;
struct TcMapCache;

// What the tensor-core GEMMs need from their owner (the matcher's handle, SuperPoint's SpTc); all zero = none
struct TcEngine {
  bool x3;             // LG_PREC_BF16X3: three passes over K (hi / lo split operands)
  __nv_bfloat16* w_hi; // bf16 hi / lo images of the owner's packed fp32 weights (same element offsets)
  __nv_bfloat16* w_lo;
  TcMapCache* maps;    // tensor maps of the linears and attention, keyed by every encode argument
  unsigned int* dbg;   // device words: site code of the first pipeline wait that timed out (0 = none)
};
// splits the n floats of the device array w into the engine's bf16 images; on failure the caller still destroys `e`
int tc_engine_create(TcEngine* e, const float* w, size_t n, bool x3, cudaStream_t stream);
void tc_engine_destroy(TcEngine* e);
// 0, or the site code of the first mbarrier wait that timed out since the last call (synchronises)
unsigned int tc_debug_timeout_code(const TcEngine& e, unsigned int* words32);
// per-forward activation buffers carved from the workspace (lo = null in LG_PREC_BF16)
struct TcBuffers {
  __nv_bfloat16 *xh, *xl;      // [S*Lp, 256] shadows of the fp32 residual stream
  __nv_bfloat16 *ctxh, *ctxl;  // [S*Lp, 256] attention output, heads concatenated h-major
  __nv_bfloat16 *msgh, *msgl;  // [S*Lp, 256] out_proj / to_out output
  __nv_bfloat16 *hh, *hl;      // [S*Lp, 512] LayerNorm+GELU output
  __half *q, *k;               // [S, H, Lp, 64] fp16 (attention operands, as lightglue.py:119)
  __half* vt;                  // [S, H, 64, Lp] fp16, V transposed
};

void tc_carve(WsBump& b, size_t S, int Lp, const LgHandle* h, TcBuffers* out);
// x fp32 [S, Lp, 256] -> bf16 (hi / lo) shadow copies the linears consume
int tc_refresh_shadow(LgHandle* h, const TcBuffers& b, const float* x, const SeqState& st, cudaStream_t stream);
int tc_input_proj(LgHandle* h, const TcBuffers& b, const SeqState& st, const float* desc_packed, float* x, cudaStream_t stream);
int tc_block(LgHandle* h, const TcBuffers& b, const SeqState& st, int layer, int blk, float* x, const float* cs,
             cudaStream_t stream);
int tc_final_proj(LgHandle* h, const TcBuffers& b, const SeqState& st, float* p_out, cudaStream_t stream);
// Similarity sweeps of the assignment on the tensor cores: S = p p_partner^T in both directions, row LSE
// (sweep 1) and row arg-max of the score (sweep 2); p (bf16 hi/lo) is read from b.msgh / b.msgl.
int tc_assign_sweeps(LgHandle* h, const TcBuffers& b, const SeqState& st, const AssignArgs& a, float* part, int* part_arg,
                     float* term, cudaStream_t stream);
// softmax(q k^T / 8) v per (sequence, head): q from b.q, keys from kbuf, values from b.vt; key/value
// sequence = (s + kv_shift) % S; writes b.ctxh (/ b.ctxl)
int tc_attention(LgHandle* h, const TcBuffers& b, const SeqState& st, int kv_shift, const __half* kbuf, cudaStream_t stream);
// k x k convolution (k = 1: `taps` = 1, k = 3: `taps` = 9, zero padding 1) + bias (+ ReLU) as a tensor-core GEMM over a
// zero-padded NHWC image stored as a [st.S * st.Lp rows, Cin] matrix, row = padded pixel b (H+2)(W+2) + y (W+2) + x
// (SuperPoint encoder, superpoint.py:137-153).  Weights: [256 rows (Cout, zero padded), taps * Cin] at e.w_hi/w_lo +
// w_off; bias padded to 256.  Output: the same padded layout with `cout` channels as bf16 hi (/ lo), padding pixels
// zeroed -- or, if out_f32 is given, fp32 [rows, ldo] without ReLU / zeroing (the 1x1 heads).
int tc_conv(TcEngine& e, const SeqState& st, const __nv_bfloat16* in_h, const __nv_bfloat16* in_l, int cin, int taps, size_t w_off,
            const float* bias, int relu, int B, int H, int W, __nv_bfloat16* out_h, __nv_bfloat16* out_l, int cout, float* out_f32,
            int ldo, cudaStream_t stream);
