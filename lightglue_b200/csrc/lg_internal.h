// Internal declarations shared by the translation units of liblightglue_b200.so.
// Sequence model: a batch of B pairs is 2B token sequences.  Sequence s < B is image0 of pair s,
// sequence s >= B is image1 of pair s - B.  Every per-token buffer is [S, Lp, C] with Lp = the
// common padded length (multiple of 128), so 128-row tiles never straddle sequences.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define LG_DIM 256
#define LG_HEADS 4
#define LG_HDIM 64
#define LG_FFN 512
#define LG_TILE 128

// Error returns of the C-ABI code: a failed CUDA call records its error and returns it (LG_CU; LG_CHECK_LAUNCH after a
// kernel launch), a non-zero return code is passed on (LG_RC).
#define LG_CU(x)                                                                 \
  do {                                                                           \
    cudaError_t e__ = (x);                                                       \
    if (e__ != cudaSuccess) return lg_set_cuda_error(e__, __FILE__, __LINE__);   \
  } while (0)
#define LG_CHECK_LAUNCH() LG_CU(cudaGetLastError())
#define LG_RC(x)         \
  do {                   \
    int r__ = (x);       \
    if (r__) return r__; \
  } while (0)

int lg_set_cuda_error(cudaError_t e, const char* file, int line);
int lg_set_error(const char* msg);
// Per-DEVICE one-time kernel setup (function attributes are per device: a process may drive several GPUs).
// Opts `func` in to `bytes` of dynamic shared memory on the current device the first time it is seen there.
int lg_func_smem_once(const void* func, int bytes);
// SM count of the current device (queried once per device).
int lg_num_sms();

// Device-side view of the adaptive state; all arrays live in the workspace.
struct SeqState {
  int S, B, Lp;
  const int* len;         // [S] current number of live points per sequence
  const int* stop_layer;  // [B] 0 while the pair is still running, else (last executed layer + 1)
};

__device__ __forceinline__ bool lg_pair_stopped(const SeqState& st, int s) {
  return st.stop_layer[s >= st.B ? s - st.B : s] != 0;
}

// ----------------------------------------------------------------------------------------------
// fp32 CUDA-core path (k_simt.cu)
// ----------------------------------------------------------------------------------------------
enum { EPI_STORE = 0, EPI_RESID = 1, EPI_QKV_ROPE = 2, EPI_QK_V = 3 };

struct GemmArgs {
  // A = [A0 | A1] along K (concat for the FFN input, lightglue.py:172/228); rows are [S*Lp]
  const float* A0; int lda0; int K0;
  const float* A1; int lda1;
  const float* W; const float* bias;  // W [Nout, K] row-major (nn.Linear layout)
  long w_sel_stride, b_sel_stride;    // > 0: W += (stop_layer[pair] - 1) * stride  (per-pair head select)
  int K, Nout;
  int epi; float scale;
  float* out; int ldo;                // EPI_STORE / EPI_RESID
  float* q; float* k; float* v;       // EPI_QKV_ROPE / EPI_QK_V: [S, H, Lp, 64]
  const float* cs;                    // [S, Lp, 64] cos(32) | sin(32)
};
int simt_gemm(const GemmArgs& a, const SeqState& st, cudaStream_t stream);
// softmax(q k^T / 8) v for every (sequence, head); key/value sequence = (s + kv_shift) % S.
int simt_attention(const float* q, const float* k, const float* v, float* ctx /*[S,Lp,256]*/, int kv_shift,
                   const SeqState& st, cudaStream_t stream);
int simt_layernorm_gelu(float* h /*[S*Lp,512] in place*/, const float* gamma, const float* beta, const SeqState& st,
                        cudaStream_t stream);

// ----------------------------------------------------------------------------------------------
// shared non-GEMM kernels (k_misc.cu)
// ----------------------------------------------------------------------------------------------
struct PosencArgs {
  const float* kpts0; const float* kpts1;      // [B,M,2], [B,N,2]
  const float* size0; const float* size1;      // [B,2] or null
  const float* scales0; const float* oris0; const float* scales1; const float* oris1;
  const float* wr;                              // [32, pos_dim]
  int pos_dim, B, M, N, Lp;
  float* cs;                                    // [S, Lp, 64]
  const int* lens0; const int* lens1;           // [B] valid rows per pair, or null (= M / N)
};
int misc_posenc(const PosencArgs& a, cudaStream_t stream);
// descriptors [B,M,d] / [B,N,d] -> padded [S, Lp, d] fp32
// (+ optionally the bf16 hi / lo images of the same rows, [S * Lp, d], for the tensor-core linears)
int misc_pack_desc(const float* d0, const float* d1, float* out, int B, int M, int N, int Lp, int d, const int* lens0,
                   const int* lens1, cudaStream_t stream, void* hi = nullptr, void* lo = nullptr);
// len[s] = lens[s] (or M / N), ind[s][r] = r, prune[s][r] = 1 for live rows, below = 0, stop_layer = 0 -- or 1 for a
// pair with an empty image (answered like lightglue.py:568-588: no layer runs, nothing matches)
int misc_init_state(int* len, int* ind, int* prune, int* stop_layer, int* below, int n_below, int B, int M, int N, int Lp,
                    const int* lens0, const int* lens1, cudaStream_t stream);

struct AdaptArgs {
  const float* x;                   // [S, Lp, 256] fp32 residual stream
  const float* tok_w; const float* tok_b;      // token_confidence[i] (null: early exit off)
  const float* mat_w; const float* mat_b;      // log_assignment[i].matchability (null: pruning off)
  float thr;                        // confidence_thresholds[i]
  float depth_conf, width_conf;
  int layer, M, N, pruning_threshold;
  const int* lens0; const int* lens1;  // [B] original lengths of a ragged batch, or null (= M / N)
  unsigned char* keep;              // [S, Lp]
  int* below;                       // [B] (this layer's slot)
  int* stop_layer;                  // [B] (written)
  const int* len_in; int* len_out;  // [S]
  int* pos;                         // [S, Lp] destination row of each kept row
  int* did_prune;                   // [S]
};
int misc_adapt_score(const AdaptArgs& a, const SeqState& st, cudaStream_t stream);
int misc_adapt_decide(const AdaptArgs& a, const SeqState& st, cudaStream_t stream);
struct GatherArgs {
  const float* x_in; float* x_out;      // [S, Lp, 256]
  const float* cs_in; float* cs_out;    // [S, Lp, 64]
  const int* ind_in; int* ind_out;      // [S, Lp]
  int* prune;                           // [S, Lp] by original index
  const unsigned char* keep; const int* pos; const int* did_prune;
  const int* len_in;
  const int* len_out; int* stop_layer; int layer;  // an image pruned to 0 points ends its pair (lightglue.py:539-540)
};
int misc_adapt_gather(const GatherArgs& a, const SeqState& st, cudaStream_t stream);
int misc_finalize_stop(int* stop_layer, int B, int n_layers, cudaStream_t stream);

// lg_attention plumbing: [B, H, n, 64] fp32 heads -> the attention kernels' operand layouts, and back.
// fp32 mode: qf/kf/vf fp32 [S, H, Lp, 64].  Tensor-core modes: qh/kh fp16 [S, H, Lp, 64], vth fp16 [S, H, 64, Lp].
struct AttnIoArgs {
  const float *q0, *k0, *v0, *q1, *k1, *v1;
  int B, M, N, Lp;
  float *qf, *kf, *vf;
  void *qh, *kh, *vth;          // __half*
  const float* ctxf;            // fp32 mode: [S, Lp, 256]
  const void *ctxh, *ctxl;      // tensor-core modes: bf16 hi (/ lo) [S*Lp, 256]
  float *out0, *out1;           // [B, M, 256], [B, N, 256]
};
int misc_attn_pack(const AttnIoArgs& a, cudaStream_t stream);
int misc_attn_unpack(const AttnIoArgs& a, cudaStream_t stream);

// Assignment tail (lightglue.py:265-318) on projected descriptors p [S, Lp, 256] (already / 256^0.25)
struct AssignArgs {
  const float* p;        // [S, Lp, 256]
  const float* x;        // [S, Lp, 256] (matchability input)
  const float* mat_w; const float* mat_b; long mat_sel_stride;  // per-pair head select via stop_layer
  float* z;              // [S, Lp] matchability logits
  float* rowpart; float* colpart;  // [S(pair side), Lp, nt, 2] partial (max, sumexp) per 64-wide tile
  float* rowlse; float* collse;    // [B, Lp]
  float* rowbest; int* rowarg; float* colbest; int* colarg;  // [B, Lp, nt] then reduced into [.., 0]
  int nt;                // number of 64-wide tiles along Lp
  float filter_threshold;
  // compact-index results
  int* m0c; int* m1c; float* ms0c; float* ms1c;   // [B, Lp]
  // final outputs
  const int* ind;        // [S, Lp]
  int M, N;
  int64_t* matches0; int64_t* matches1; float* mscores0; float* mscores1;
  int* n_matches; int64_t* matches; float* match_scores; int cap;  // cap = min(M, N)
  float* log_assignment; // optional [B, M+1, N+1]
};
int misc_assign(const AssignArgs& a, const SeqState& st, cudaStream_t stream, int64_t* launches);
// companions of the tensor-core sweeps: z + LSE combine (after sweep 1), slot reduce + filter + outputs (after sweep 2)
int misc_assign_term(const AssignArgs& a, const SeqState& st, const float* part, int pstride, int slot_cols, float* term,
                     cudaStream_t stream);
int misc_assign_dustbin(const AssignArgs& a, const SeqState& st, cudaStream_t stream);
int misc_assign_tail(const AssignArgs& a, const SeqState& st, const float* part, const int* part_arg, int pstride, int slot_cols,
                     cudaStream_t stream);
int misc_export_stop_prune(const int* stop_layer, const int* prune, int* stop_out, int* prune0, int* prune1, int B, int M,
                           int N, int Lp, cudaStream_t stream);

// packed assignment / token heads inside LgHandle::wpk (floats)
#define AO_FW 0                                   // final_proj.weight [256,256]
#define AO_FB (LG_DIM * LG_DIM)                   // final_proj.bias [256]
#define AO_MW (AO_FB + LG_DIM)                    // matchability.weight [256]
#define AO_MB (AO_MW + LG_DIM)                    // matchability.bias [1]
#define ASSIGN_BLOB_PAD (AO_MB + 64)
#define TOKEN_BLOB_PAD (LG_DIM + 64)              // token.0.weight [256] | bias [1]
