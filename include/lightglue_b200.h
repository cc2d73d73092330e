/*
 * lightglue_b200.h -- C ABI of the H100-native LightGlue matcher forward path.
 *
 * The reference (cvg/LightGlue) is pure Python: it has no FFI / plugin interface, its boundary is
 * the Python class `LightGlue` (lightglue/lightglue.py:321-662).  This header is the C-ABI a
 * binding for that class calls; `lightglue_b200/matcher.py` is exactly such a binding (ctypes) and
 * keeps the reference's constructor / forward / output-dict contract.  Every entry point below
 * names the reference code it replaces.
 *
 * Conventions
 *   - plain C types only: device pointers, sizes, a cudaStream_t passed as void*;
 *   - every function returns 0 on success, non-zero on failure; lg_last_error() gives the text;
 *   - nothing here synchronises the host with the device and nothing allocates after lg_create
 *     (the caller owns inputs, outputs and the workspace; the handle owns only its packed weights);
 *   - all tensors are dense row-major; "B" pairs, image0 has M keypoints, image1 has N.
 */
#ifndef LIGHTGLUE_B200_H_
#define LIGHTGLUE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LG_ABI_VERSION 3

#if defined(__GNUC__)
#define LG_API __attribute__((visibility("default")))
#else
#define LG_API
#endif

/* Arithmetic the linear layers / similarity run in (softmax, LayerNorm, residual stream and all
 * reductions are always fp32). */
enum {
  LG_PREC_FP32 = 0,   /* fp32 CUDA-core path: reference-grade, used for index-exact parity      */
  LG_PREC_BF16 = 1,   /* wgmma tensor cores, bf16 operands (fp16 inside attention), fp32 accum   */
  LG_PREC_BF16X3 = 2  /* wgmma, split-bf16 (hi+lo, 3 MMAs) linears: ~fp32 accuracy              */
};

/* Mirrors LightGlue.default_conf (lightglue.py:322-335). */
typedef struct LgConfig {
  int32_t abi_version;        /* LG_ABI_VERSION */
  int32_t input_dim;          /* conf.input_dim: 256 (SuperPoint) / 128 (DISK, ALIKED, SIFT...)  */
  int32_t pos_dim;            /* 2, or 4 when conf.add_scale_ori (lightglue.py:394-396)          */
  int32_t n_layers;           /* conf.n_layers (9)                                               */
  int32_t precision;          /* LG_PREC_*                                                       */
  float depth_confidence;     /* conf.depth_confidence, <= 0 disables early exit                 */
  float width_confidence;     /* conf.width_confidence, <= 0 disables point pruning              */
  float filter_threshold;     /* conf.filter_threshold                                           */
} LgConfig;

/* One forward call == LightGlue._forward (lightglue.py:483-629). */
typedef struct LgInputs {
  int32_t B, M, N;
  const float* kpts0;   /* [B, M, 2] pixel (x, y)                                  (487)         */
  const float* kpts1;   /* [B, N, 2]                                                             */
  const float* desc0;   /* [B, M, input_dim]                                       (502)         */
  const float* desc1;   /* [B, N, input_dim]                                                     */
  const float* size0;   /* [B, 2] (w, h) or NULL -> bbox normalisation             (35-36, 491)  */
  const float* size1;
  const float* scales0; /* [B, M] / [B, N], only when pos_dim == 4                 (495-501)     */
  const float* oris0;
  const float* scales1;
  const float* oris1;
  int32_t pruning_threshold; /* pruning_min_kpts(device): prune an image only while it has more
                                keypoints than this                                 (551, 658-662) */
  /* Ragged batches (SURVEY 8f2; the reference pads + masks instead, lightglue.py:46-55, 256-262, 512-520):
   * optional DEVICE arrays [B]; pair b uses only the first lens0[b] rows of kpts0/desc0 (<= M) and the
   * first lens1[b] rows of kpts1/desc1 (<= N).  NULL = every pair uses M / N.  Rows past the length are
   * never read; their outputs are matches -1, scores 0, prune 0.  A pair with a zero length is
   * answered like the reference's empty-input branch (568-588): nothing matched, stop = 1. */
  const int32_t* lens0;
  const int32_t* lens1;
} LgInputs;

typedef struct LgOutputs {
  int64_t* matches0;        /* [B, M]  -1 = unmatched                               (606-609)     */
  int64_t* matches1;        /* [B, N]                                                             */
  float* matching_scores0;  /* [B, M]                                               (610-613)     */
  float* matching_scores1;  /* [B, N]                                                             */
  int32_t* stop;            /* [B] last executed layer + 1, per pair                (583, 624)    */
  int32_t* prune0;          /* [B, M] pruning counters (535-536, 558); may be NULL                */
  int32_t* prune1;          /* [B, N]                                                             */
  int32_t* n_matches;       /* [B]                                                                */
  int64_t* matches;         /* [B, min(M,N), 2] packed (i0, i1), ascending i0; first n_matches[b]
                               rows valid                                           (593-602)     */
  float* match_scores;      /* [B, min(M,N)]                                                      */
  float* log_assignment;    /* optional [B, M+1, N+1] log-assignment matrix (MatchAssignment.forward,
                               lightglue.py:265-277, 287-296); NULL = do not materialise it.  Only
                               valid when pruning/early exit are off (dense indexing).            */
} LgOutputs;

typedef struct LgHandle LgHandle;

/* Number of floats in the weight blob for (input_dim, pos_dim, n_layers).  Blob = the reference
 * state_dict tensors (lightglue.py:388-413), fp32, concatenated in this order:
 *   posenc.Wr.weight [32, pos_dim]
 *   input_proj.weight [256, input_dim], input_proj.bias [256]        (only if input_dim != 256)
 *   for l in 0..L-1:
 *     self_attn : Wqkv.w [768,256] Wqkv.b [768] out_proj.w [256,256] out_proj.b [256]
 *                 ffn.0.w [512,512] ffn.0.b [512] ffn.1.w [512] ffn.1.b [512] ffn.3.w [256,512] ffn.3.b [256]
 *     cross_attn: to_qk.w [256,256] to_qk.b [256] to_v.w [256,256] to_v.b [256] to_out.w [256,256] to_out.b [256]
 *                 ffn.0.w ffn.0.b ffn.1.w ffn.1.b ffn.3.w ffn.3.b        (shapes as above)
 *   for l in 0..L-1: log_assignment.l.matchability.w [256] .b [1]  final_proj.w [256,256] .b [256]
 *   for l in 0..L-2: token_confidence.l.token.0.w [256] .b [1]
 */
LG_API size_t lg_weight_blob_floats(int32_t input_dim, int32_t pos_dim, int32_t n_layers);

/* Replaces LightGlue.__init__'s module construction + load_state_dict (lightglue.py:376-437):
 * packs the fp32 DEVICE blob into the layouts the kernels want (row permutation of Wqkv, bf16
 * hi/lo copies) on `stream`.  The blob may be freed once the stream has drained. */
LG_API int lg_create(const LgConfig* cfg, const float* weights_dev, size_t n_floats, void* stream, LgHandle** out);
LG_API int lg_destroy(LgHandle* h);

/* Bytes of scratch lg_forward needs for a (B, M, N) problem.  The workspace must be zero-filled
 * once after allocation (padding rows are never written and must stay finite). */
LG_API size_t lg_workspace_bytes(const LgHandle* h, int32_t B, int32_t M, int32_t N);

/* Replaces LightGlue._forward (lightglue.py:483-629): keypoint normalisation (31-43), positional
 * encoding (68-81), n_layers x (SelfBlock 140-172, CrossBlock 175-230), token confidence / early
 * exit (84-94, 645-656), point pruning (636-643, 551-566), MatchAssignment (280-296),
 * filter_matches (302-318) and the output assembly (593-614).  Asynchronous on `stream`.
 * Early exit / pruning are evaluated per pair (identical to the reference for B == 1, which is the
 * only batch size for which the reference's adaptive bookkeeping is well defined). */
LG_API int lg_forward(LgHandle* h, const LgInputs* in, const LgOutputs* out, void* workspace, size_t workspace_bytes,
               void* stream);

/* Stand-alone MatchAssignment.forward + filter_matches on dense descriptors (lightglue.py:287-296,
 * 302-318) using layer `layer`'s head: x0 [B, M, 256], x1 [B, N, 256] fp32 device.  For unit
 * tests and for the HBM-roofline measurement of the materialising variant. */
LG_API int lg_assign(LgHandle* h, int32_t layer, int32_t B, int32_t M, int32_t N, const float* x0, const float* x1,
              const LgOutputs* out, void* workspace, size_t workspace_bytes, void* stream);

/* Kernel-level entry point (unit tests / ncu): Attention.forward (lightglue.py:97-137) on heads that are
 * already projected and rotated, through the attention kernel lg_forward uses in this handle's precision
 * mode.  q0, k0, v0 [B, 4, M, 64] and q1, k1, v1 [B, 4, N, 64] fp32 device (the reference's [B, H, N, dh]
 * layout, 166-167 / 207).  cross == 0: ctx0 = softmax(q0 k0^T / 8) v0, ctx1 likewise for image 1
 * (SelfBlock, 170); cross != 0: ctx0 = softmax(q0 k1^T / 8) v1 and ctx1 = softmax(q1 k0^T / 8) v0
 * (CrossBlock, 210-214).  ctx0 [B, M, 256], ctx1 [B, N, 256] fp32, heads concatenated h-major (171 / 208).
 * The tensor-core modes round q, k, v to fp16 like the reference's flash path (116-121). */
LG_API int lg_attention(LgHandle* h, int32_t B, int32_t M, int32_t N, int32_t cross, const float* q0, const float* k0,
                 const float* v0, const float* q1, const float* k1, const float* v1, float* ctx0, float* ctx1,
                 void* workspace, size_t workspace_bytes, void* stream);

/* Block-level parity hook (SURVEY 4.1: per-layer comparison against the reference's hooks on
 * `transformers[i]`, lightglue.py:541): while `buf` is non-NULL every lg_forward on this handle copies the fp32
 * residual stream after each transformer layer i into buf[i][s][r][256], s < 2B sequences (image0 of pair s, then
 * image1 of pair s - B), r < lg_padded_length(M, N) rows (rows past a sequence's length are unspecified; with point
 * pruning rows are in the compacted order).  `floats` = capacity of buf; NULL switches the capture off. */
LG_API int lg_debug_capture_layers(LgHandle* h, float* buf, size_t floats);
LG_API int32_t lg_padded_length(int32_t M, int32_t N);

/* Number of kernel launches issued by the last lg_forward / lg_assign on this handle. */
LG_API int64_t lg_last_launch_count(const LgHandle* h);

/* Timing hooks for bench.py: lg_forward records a CUDA-event pair around every launch of the
 * named kernel class when enabled; lg_kernel_time_ms returns the summed milliseconds and launch
 * count since the last reset (synchronises on those events only). */
enum { LG_K_ATTENTION = 0, LG_K_LINEAR = 1, LG_K_ASSIGN = 2, LG_K_OTHER = 3, LG_K_ASSIGN_MATRIX = 4,
       /* sub-classes of LG_K_LINEAR (tensor-core modes): */ LG_K_QKV = 5, LG_K_FFN0 = 6, LG_K_FFN3 = 7,
       /* whole materialising assignment stage (final_proj + sweeps + dustbin) */ LG_K_ASSIGN_STAGE = 8, LG_K_CLASSES = 9 };
LG_API int lg_timing_enable(LgHandle* h, int32_t enable);
LG_API int lg_kernel_time_ms(LgHandle* h, int32_t kernel_class, double* ms, int64_t* launches);

/* Debug aid: 0, or a code identifying the first in-kernel pipeline wait that timed out since the last
 * call (the kernels give up instead of hanging); `words32` (optional, 32 entries) receives the
 * per-site codes.  Synchronises the device. */
LG_API uint32_t lg_debug_timeout_code(LgHandle* h, uint32_t* words32);

LG_API const char* lg_last_error(void);
LG_API const char* lg_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* LIGHTGLUE_B200_H_ */
