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

// What the tensor-core GEMMs need from their owner (the matcher's handle, a TcConvWeights, the nearest-neighbour
// matcher's handle); all zero = none
struct TcEngine {
  bool x3;             // LG_PREC_BF16X3: three passes over K (hi / lo split operands)
  __nv_bfloat16* w_hi; // bf16 hi / lo images of the owner's packed fp32 weights (same element offsets)
  __nv_bfloat16* w_lo;
  TcMapCache* maps;    // tensor maps of the linears and attention, keyed by every encode argument
  unsigned int* dbg;   // device words: site code of the first pipeline wait that timed out (0 = none)
};
// splits the n floats of the device array w into the engine's bf16 images (n = 0: no weights); on failure the caller
// still destroys `e`
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
// Nearest-neighbour sweep on the tensor cores (split-bf16, e.x3): S = d_s d_partner^T in both directions from the bf16
// hi / lo images [st.S * st.Lp, dim]; per live row and 128-column slot of live partner columns, (s1, s2) into part
// (float2) and j1 into part_arg, [st.S * st.Lp, pstride] with pstride >= 2 ceil(Lp / 256) (k_tc_linear.cu, TEPI_TOP2).
// With a gate (guided matching, include/nn_b200.h) only the columns (row record, column record) passes enter the top-2
// of a pair with on[pair] != 0 (TEPI_TOP2_H / TEPI_TOP2_F).
struct TcNnGate {
  bool fundamental;  // records: H (u, v) / F (x, y, a, b, c, s), field f of row r at rec[f * st.S * st.Lp + r]
  const float* rec;
  const int* on;     // [st.B] 0: the pair is matched ungated
  float t2;          // a column passes when err < t2
};
int tc_nn_sweep(TcEngine& e, const SeqState& st, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int dim, float* part,
                int* part_arg, int pstride, cudaStream_t stream, const TcNnGate* gate = nullptr);
// softmax(q k^T / 8) v per (sequence, head): q from b.q, keys from kbuf, values from b.vt; key/value
// sequence = (s + kv_shift) % S; writes b.ctxh (/ b.ctxl)
int tc_attention(LgHandle* h, const TcBuffers& b, const SeqState& st, int kv_shift, const __half* kbuf, cudaStream_t stream);

// ---------------------------------------------------------------- convolution owners: SuperPoint, DISK, HardNet
// fp32 -> split-bf16 operand: hi = bf16(v), lo = bf16(v - hi)
__device__ __forceinline__ void tc_split(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Row plan of a tc_conv operand: `used` rows stored as two "sequences" of Lp rows (the GEMM kernel walks 128-row tiles
// per sequence), Lp the smallest multiple of LG_TILE (at least one) that holds half of them.
struct TcRows { int Lp; long rows; };
TcRows tc_rows(long used);
// Its SeqState, read from four device words: len[2] (live rows of each sequence), stop_layer (0), unused.
inline SeqState tc_rows_state(const TcRows& r, const int* words) { return SeqState{2, 1, r.Lp, words, words + 2}; }
// The words of n matrices ([n][4], every row live) with one copy (n <= 8)
int tc_rows_words(const TcRows* r, int n, int* words, cudaStream_t stream);

// One region of packed convolution weights: [rows, K], column tap * cpad + ci, from a source [cout, cin, taps]
// (nn.Conv2d) whose output channels co0 .. co0 + ncopy - 1 become rows 0 .. ncopy - 1, and a bias [rows]; zero past cin,
// taps and ncopy.  The bias is copied from b, or, with bn_var set, an eval BatchNorm (eps 1e-5) is folded in, in double:
// w rs and -bn_mean rs, rs = 1 / sqrt(bn_var + 1e-5).
struct TcConvRegion {
  const float *w, *b;
  const float *bn_mean, *bn_var;
  int cin, cpad, taps, rows, K;
  int co0, ncopy;
};
#define TC_CONV_MAX_REGIONS 12
// The packed fp32 weights of a convolution owner and the bf16x3 engine over their bf16 images.  Every region starts on
// a 64-float boundary: the bf16 images are TMA bases (16 bytes) and fp32 regions may be read as float4.
struct TcConvWeights {
  float* wpk;
  size_t w_off[TC_CONV_MAX_REGIONS], b_off[TC_CONV_MAX_REGIONS];  // float offsets of each region's weights and bias
  TcEngine tc;
};
// Packs the n regions on `stream`; the sources are read there, so they must stay alive until the stream has run it.
int tc_conv_weights_create(TcConvWeights** out, const TcConvRegion* reg, int n, cudaStream_t stream);
void tc_conv_weights_destroy(TcConvWeights* cw);

// k x k convolution (k = 1: `taps` = 1 and k = 3: `taps` = 9, zero padding q = 1; k = 5: `taps` = 25, q = 2) + bias
// (+ ReLU) as a tensor-core GEMM over a zero-padded NHWC image stored as a [st.S * st.Lp rows, Cin] matrix, row = padded
// pixel b (H+2q)(W+2q) + y (W+2q) + x (SuperPoint encoder, superpoint.py:137-153; DISK's U-Net; HardNet).  Weights and
// bias: region `region` of the TcConvWeights, [256 rows (Cout, zero padded), taps * Cin].  Output: the same padded layout
// with `cout` channels as bf16 hi (/ lo), padding pixels zeroed -- or, if out_f32 is given, fp32 [rows, ldo] without
// ReLU / zeroing (SuperPoint's 1x1 heads, DISK's convolutions: their padding rows hold garbage).  With taps = 1 it is a
// plain GEMM [rows, Cin] x [Cout, Cin]^T (the descriptor heads on gathered rows; B, H, W unused).
// pstride > 0: 3x3 convolution with stride 2 and zero padding 1 (HardNet) -> the padded layout at the OUTPUT size H x W.
// in_h / in_l then hold the four polyphase images of the padded input, each in the output's padded frame (W + 2 columns),
// phase 2 py + px (padded input pixel (2i + py, 2j + px) at frame position (i + 1, j + 1)) starting at row
// (2 py + px) pstride: tap (dy, dx) reads phase (dy & 1, dx & 1) shifted by (dy >> 1) (W + 2) + (dx >> 1) rows.
struct TcConvArgs {
  const __nv_bfloat16 *in_h, *in_l;
  int cin, taps, pstride, region, relu;  // pstride 0: stride 1
  int B, H, W;
  __nv_bfloat16 *out_h, *out_l;
  int cout;
  float* out_f32;
  int ldo;
};
int tc_conv(TcConvWeights& cw, const SeqState& st, const TcConvArgs& a, cudaStream_t stream);
