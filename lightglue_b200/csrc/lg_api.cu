// C-ABI of liblightglue_b200.so: handle / weight packing / workspace carving / forward orchestration.
// See include/lightglue_b200.h for the contract and the reference lines each entry point replaces.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <new>
#include <vector>

#include "../../include/lightglue_b200.h"
#include "lg_internal.h"
#include "lg_handle.h"
#include "lg_tc.h"

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
thread_local int64_t lg_launches;
int lg_set_error(const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return 1;
}
int lg_set_cuda_error(cudaError_t e, const char* file, int line) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s:%d", (int)e, cudaGetErrorString(e), file, line);
  return 2;
}

extern "C" const char* lg_last_error(void) { return g_err; }

// ------------------------------------------------------------------------------------------------
// per-device one-time setup
// ------------------------------------------------------------------------------------------------
#include <map>
#include <mutex>
namespace {
std::mutex g_dev_mu;
std::map<std::pair<int, const void*>, int> g_smem_done;  // (device, kernel) -> bytes opted in
std::map<int, int> g_sms;
std::map<std::pair<int, const void*>, int> g_clusters;  // (device, kernel) -> co-resident clusters
}  // namespace
int lg_func_smem_once(const void* func, int bytes) {
  int dev = 0;
  LG_CU(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = g_smem_done.find({dev, func});
  if (it != g_smem_done.end() && it->second >= bytes) return 0;
  LG_CU(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  g_smem_done[{dev, func}] = bytes;
  return 0;
}
int lg_num_sms() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = g_sms.find(dev);
  if (it != g_sms.end()) return it->second;
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  g_sms[dev] = n;
  return n;
}
int lg_max_clusters(const void* func, int threads, int smem, int cluster, int* out) {
  if (int r = lg_func_smem_once(func, smem)) return r;
  int dev = 0;
  LG_CU(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = g_clusters.find({dev, func});
  if (it != g_clusters.end()) { *out = it->second; return 0; }
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cluster); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem;
  cfg.attrs = at; cfg.numAttrs = 1;
  int n = 0;
  LG_CU(cudaOccupancyMaxActiveClusters(&n, func, &cfg));
  if (n <= 0) return lg_set_error("lg_max_clusters: the kernel's clusters do not fit on this device");
  g_clusters[{dev, func}] = n;
  *out = n;
  return 0;
}
extern "C" const char* lg_build_info(void) {
#define LG_STR2(x) #x
#define LG_STR(x) LG_STR2(x)
  return "lightglue_b200 abi=" LG_STR(LG_ABI_VERSION) " arch=sm_90a (" __DATE__ " " __TIME__ ")";
}

// ------------------------------------------------------------------------------------------------
// weight blob layout (reference order, see header) and packed layout (kernel order)
// ------------------------------------------------------------------------------------------------
namespace {
constexpr size_t D = LG_DIM, F = LG_FFN;
constexpr size_t SELF_BLOB = 3 * D * D + 3 * D + D * D + D + F * F + F + F + F + D * F + D;
constexpr size_t CROSS_BLOB = 3 * (D * D + D) + F * F + F + F + F + D * F + D;
constexpr size_t ASSIGN_BLOB = D + 1 + D * D + D;
constexpr size_t TOKEN_BLOB = D + 1;
}  // namespace

extern "C" size_t lg_weight_blob_floats(int32_t input_dim, int32_t pos_dim, int32_t n_layers) {
  size_t n = 32 * (size_t)pos_dim;
  if (input_dim != (int)D) n += D * (size_t)input_dim + D;
  n += (size_t)n_layers * (SELF_BLOB + CROSS_BLOB + ASSIGN_BLOB);
  n += (size_t)(n_layers - 1) * TOKEN_BLOB;
  return n;
}

// Wqkv rows: reference channel c = h*192 + d*3 + which (lightglue.py:166)  ->  packed row which*256 + h*64 + d
__global__ void permute_qkv_kernel(const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ wo,
                                   float* __restrict__ bo) {
  const int prow = blockIdx.x;  // packed row
  const int which = prow / 256, h = (prow % 256) / 64, d = prow % 64;
  const int src = h * 192 + d * 3 + which;
  for (int c = threadIdx.x; c < 256; c += blockDim.x) wo[(size_t)prow * 256 + c] = w[(size_t)src * 256 + c];
  if (threadIdx.x == 0) bo[prow] = b[src];
}

// W1f = [W1[:, :256] | W1[:, 256:] Wo], b1f = b1 + W1[:, 256:] bo, accumulated in double (see lg_handle.h)
__global__ void fold_out_proj_kernel(const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ wo,
                                     const float* __restrict__ bo, float* __restrict__ w1f, float* __restrict__ b1f) {
  const int n = blockIdx.x;  // ffn.0 output channel
  const float* row = w1 + (size_t)n * LG_FFN;
  for (int c = threadIdx.x; c < LG_DIM; c += blockDim.x) {
    w1f[(size_t)n * LG_FFN + c] = row[c];
    double acc = 0.0;
    for (int j = 0; j < LG_DIM; ++j) acc += (double)row[LG_DIM + j] * (double)wo[(size_t)j * LG_DIM + c];
    w1f[(size_t)n * LG_FFN + LG_DIM + c] = (float)acc;
  }
  if (threadIdx.x == 0) {
    double acc = (double)b1[n];
    for (int j = 0; j < LG_DIM; ++j) acc += (double)row[LG_DIM + j] * (double)bo[j];
    b1f[n] = (float)acc;
  }
}

extern "C" int lg_create(const LgConfig* cfg, const float* blob, size_t n_floats, void* stream_, LgHandle** out) {
  if (!cfg || !blob || !out) return lg_set_error("lg_create: null argument");
  if (cfg->abi_version != LG_ABI_VERSION) return lg_set_error("lg_create: ABI version mismatch");
  if (cfg->n_layers < 1 || cfg->n_layers > 64) return lg_set_error("lg_create: n_layers out of range");
  if (cfg->pos_dim != 2 && cfg->pos_dim != 4) return lg_set_error("lg_create: pos_dim must be 2 or 4");
  if (cfg->input_dim < 4 || cfg->input_dim % 16 != 0 || cfg->input_dim > 512)
    return lg_set_error("lg_create: input_dim must be a multiple of 16 in [16, 512]");
  if (cfg->precision < LG_PREC_FP32 || cfg->precision > LG_PREC_BF16X3) return lg_set_error("lg_create: bad precision");
  if (n_floats != lg_weight_blob_floats(cfg->input_dim, cfg->pos_dim, cfg->n_layers))
    return lg_set_error("lg_create: weight blob has the wrong size");
  cudaStream_t stream = (cudaStream_t)stream_;
  LgHandle* h = new (std::nothrow) LgHandle();
  if (!h) return lg_set_error("lg_create: out of host memory");
  struct Guard {  // every failure path below releases the handle and what it owns
    LgHandle* h;
    ~Guard() { if (h) lg_destroy(h); }
  } guard{h};
  h->wpk = nullptr;
  memset(&h->tc, 0, sizeof(h->tc));
  h->cfg = *cfg;
  h->timing = false;
  h->dbg_layers = nullptr; h->dbg_layers_floats = 0;
  for (int i = 0; i < LG_K_CLASSES; ++i) h->ev_used[i] = 0;
  LG_CU(cudaGetDevice(&h->device));
  const int L = cfg->n_layers;
  h->bself = block_off(3 * D);
  h->bcross = block_off(2 * D);
  h->layer_stride = h->bself.total + h->bcross.total;
  size_t c = 0;
  h->o_wr = c; c += 32 * (size_t)cfg->pos_dim;
  c = (c + 63) / 64 * 64;
  h->o_inw = c; c += D * (size_t)cfg->input_dim;
  h->o_inb = c; c += D;
  h->o_layers = c; c += (size_t)L * h->layer_stride;
  h->o_assign = c; c += (size_t)L * ASSIGN_BLOB_PAD;
  h->o_token = c; c += (size_t)L * TOKEN_BLOB_PAD;
  h->wpk_floats = c;
  LG_CU(cudaMalloc(&h->wpk, c * sizeof(float)));
  LG_CU(cudaMemsetAsync(h->wpk, 0, c * sizeof(float), stream));
  auto cp = [&](size_t dst, const float* src, size_t n) {
    return cudaMemcpyAsync(h->wpk + dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, stream);
  };
  const float* p = blob;
  LG_CU(cp(h->o_wr, p, 32 * (size_t)cfg->pos_dim)); p += 32 * (size_t)cfg->pos_dim;
  if (cfg->input_dim != (int)D) {
    LG_CU(cp(h->o_inw, p, D * (size_t)cfg->input_dim)); p += D * (size_t)cfg->input_dim;
    LG_CU(cp(h->o_inb, p, D)); p += D;
  }
  for (int l = 0; l < L; ++l) {
    float* base = h->wpk + h->o_layers + (size_t)l * h->layer_stride;
    // self block
    permute_qkv_kernel<<<768, 128, 0, stream>>>(p, p + 3 * D * D, base + h->bself.wp, base + h->bself.bp);
    LG_CHECK_LAUNCH();
    p += 3 * D * D + 3 * D;
    size_t bo = h->o_layers + (size_t)l * h->layer_stride;
    LG_CU(cp(bo + h->bself.wo, p, D * D)); p += D * D;
    LG_CU(cp(bo + h->bself.bo, p, D)); p += D;
    LG_CU(cp(bo + h->bself.w1, p, F * F)); p += F * F;
    LG_CU(cp(bo + h->bself.b1, p, F)); p += F;
    LG_CU(cp(bo + h->bself.g, p, F)); p += F;
    LG_CU(cp(bo + h->bself.be, p, F)); p += F;
    LG_CU(cp(bo + h->bself.w2, p, D * F)); p += D * F;
    LG_CU(cp(bo + h->bself.b2, p, D)); p += D;
    // cross block: [to_qk ; to_v] stacked into one [512, 256] projection
    bo += h->bself.total;
    LG_CU(cp(bo + h->bcross.wp, p, D * D)); p += D * D;
    LG_CU(cp(bo + h->bcross.bp, p, D)); p += D;
    LG_CU(cp(bo + h->bcross.wp + D * D, p, D * D)); p += D * D;
    LG_CU(cp(bo + h->bcross.bp + D, p, D)); p += D;
    LG_CU(cp(bo + h->bcross.wo, p, D * D)); p += D * D;
    LG_CU(cp(bo + h->bcross.bo, p, D)); p += D;
    LG_CU(cp(bo + h->bcross.w1, p, F * F)); p += F * F;
    LG_CU(cp(bo + h->bcross.b1, p, F)); p += F;
    LG_CU(cp(bo + h->bcross.g, p, F)); p += F;
    LG_CU(cp(bo + h->bcross.be, p, F)); p += F;
    LG_CU(cp(bo + h->bcross.w2, p, D * F)); p += D * F;
    LG_CU(cp(bo + h->bcross.b2, p, D)); p += D;
    for (int blk = 0; blk < 2; ++blk) {
      const BlockOff& o = blk == 0 ? h->bself : h->bcross;
      float* bw = base + (blk == 0 ? 0 : h->bself.total);
      fold_out_proj_kernel<<<(unsigned)F, 256, 0, stream>>>(bw + o.w1, bw + o.b1, bw + o.wo, bw + o.bo, bw + o.w1f, bw + o.b1f);
      LG_CHECK_LAUNCH();
    }
  }
  for (int l = 0; l < L; ++l) {  // packed: final_proj.w [256,256] | final_proj.b [256] | matchability.w [256] | .b [1] (+pad)
    const size_t dst = h->o_assign + (size_t)l * ASSIGN_BLOB_PAD;
    LG_CU(cp(dst + AO_MW, p, D)); p += D;
    LG_CU(cp(dst + AO_MB, p, 1)); p += 1;
    LG_CU(cp(dst + AO_FW, p, D * D)); p += D * D;
    LG_CU(cp(dst + AO_FB, p, D)); p += D;
  }
  for (int l = 0; l < L - 1; ++l) {
    const size_t dst = h->o_token + (size_t)l * TOKEN_BLOB_PAD;
    LG_CU(cp(dst, p, D)); p += D;
    LG_CU(cp(dst + D, p, 1)); p += 1;
  }
  if ((size_t)(p - blob) != n_floats) return lg_set_error("lg_create: internal blob walk mismatch");
  for (int i = 0; i < L; ++i) {
    double t = 0.8 + 0.1 * exp(-4.0 * i / L);
    t = t < 0 ? 0 : (t > 1 ? 1 : t);
    h->thr[i] = (float)t;
  }
  if (cfg->precision != LG_PREC_FP32) {
    int r = tc_engine_create(&h->tc, h->wpk, h->wpk_floats, cfg->precision == LG_PREC_BF16X3, stream);
    if (r) return r;
  }
  guard.h = nullptr;
  *out = h;
  return 0;
}

extern "C" int lg_destroy(LgHandle* h) {
  if (!h) return 0;
  if (h->wpk) cudaFree(h->wpk);
  tc_engine_destroy(&h->tc);
  for (int i = 0; i < LG_K_CLASSES; ++i)
    for (cudaEvent_t e : h->ev[i]) cudaEventDestroy(e);
  delete h;
  return 0;
}

extern "C" uint32_t lg_debug_timeout_code(LgHandle* h, uint32_t* words32) { return h ? tc_debug_timeout_code(h->tc, words32) : 0; }

extern "C" int64_t lg_last_launch_count(const LgHandle* h) { return h ? h->launches : 0; }

extern "C" int lg_debug_capture_layers(LgHandle* h, float* buf, size_t floats) {
  if (!h) return lg_set_error("null handle");
  h->dbg_layers = buf;
  h->dbg_layers_floats = buf ? floats : 0;
  return 0;
}
extern "C" int32_t lg_padded_length(int32_t M, int32_t N) {
  const int mx = M > N ? M : N;
  return ((mx > 0 ? mx : 1) + LG_TILE - 1) / LG_TILE * LG_TILE;
}

extern "C" int lg_timing_enable(LgHandle* h, int32_t enable) {
  if (!h) return lg_set_error("null handle");
  h->timing = enable != 0;
  for (int i = 0; i < LG_K_CLASSES; ++i) h->ev_used[i] = 0;
  return 0;
}

extern "C" int lg_kernel_time_ms(LgHandle* h, int32_t kc, double* ms, int64_t* launches) {
  if (!h || kc < 0 || kc >= LG_K_CLASSES) return lg_set_error("lg_kernel_time_ms: bad argument");
  double tot = 0;
  for (size_t i = 0; i + 1 < h->ev_used[kc]; i += 2) {
    LG_CU(cudaEventSynchronize(h->ev[kc][i + 1]));
    float t = 0;
    LG_CU(cudaEventElapsedTime(&t, h->ev[kc][i], h->ev[kc][i + 1]));
    tot += t;
  }
  if (ms) *ms = tot;
  if (launches) *launches = (int64_t)(h->ev_used[kc] / 2);
  h->ev_used[kc] = 0;
  return 0;
}

namespace {
// ---------------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------------
struct Workspace {
  int Lp, nt;
  float *xa, *xb, *csa, *csb, *q, *k, *v, *ctx, *msg, *hbuf, *z, *term;
  float *rowpart, *colpart, *rowlse, *collse, *rowbest, *colbest, *ms0c, *ms1c;
  int *rowarg, *colarg, *m0c, *m1c, *tc_parg;
  float* tc_part;
  int *lena, *lenb, *inda, *indb, *prune, *stop_layer, *below, *pos, *did_prune;
  unsigned char* keep;
  TcBuffers tc;
  size_t bytes;
};

int round_up(int x, int m) { return (x + m - 1) / m * m; }

void carve(const LgHandle* h, int B, int M, int N, char* base, Workspace* w) {
  WsBump b{base, 0};
  const int mx = M > N ? M : N;
  const int Lp = round_up(mx > 0 ? mx : 1, LG_TILE);
  const size_t S = 2 * (size_t)B, R = S * Lp;
  const bool prune = h->cfg.width_confidence > 0;
  const bool fp32 = h->cfg.precision == LG_PREC_FP32;
  w->Lp = Lp;
  w->nt = Lp / 64;
  w->xa = b.take<float>(R * D);
  w->xb = prune ? b.take<float>(R * D) : nullptr;
  w->csa = b.take<float>(R * 64);
  w->csb = prune ? b.take<float>(R * 64) : nullptr;
  if (fp32) {
    w->q = b.take<float>(R * D);
    w->k = b.take<float>(R * D);
    w->v = b.take<float>(R * D);
    w->ctx = b.take<float>(R * D);
    w->msg = b.take<float>(R * D);
    w->hbuf = b.take<float>(R * F);
    memset(&w->tc, 0, sizeof(w->tc));
  } else {
    w->q = w->k = w->v = w->msg = nullptr;
    w->ctx = b.take<float>(R * D);   // projected descriptors for the assignment sweeps (fp32)
    w->hbuf = b.take<float>(R * (size_t)(h->cfg.input_dim > (int)D ? h->cfg.input_dim : (int)D));
    tc_carve(b, S, Lp, h, &w->tc);
  }
  w->z = b.take<float>(R);
  w->term = b.take<float>(R);
  {  // tensor-core assignment sweeps: one (max, sumexp) / (best, arg) slot per 128 columns of the partner
    const size_t slots = fp32 ? 0 : 2 * (size_t)((Lp + 255) / 256);
    w->tc_part = b.take<float>(R * slots * 2);
    w->tc_parg = b.take<int>(R * slots);
  }
  const size_t P = (size_t)B * Lp;
  w->rowpart = b.take<float>(P * w->nt * 2);
  w->colpart = b.take<float>(P * w->nt * 2);
  w->rowlse = b.take<float>(P);
  w->collse = b.take<float>(P);
  w->rowbest = b.take<float>(P * w->nt);
  w->colbest = b.take<float>(P * w->nt);
  w->rowarg = b.take<int>(P * w->nt);
  w->colarg = b.take<int>(P * w->nt);
  w->m0c = b.take<int>(P);
  w->m1c = b.take<int>(P);
  w->ms0c = b.take<float>(P);
  w->ms1c = b.take<float>(P);
  w->lena = b.take<int>(S);
  w->lenb = b.take<int>(S);
  w->inda = b.take<int>(R);
  w->indb = prune ? b.take<int>(R) : nullptr;
  w->prune = b.take<int>(R);
  w->stop_layer = b.take<int>(B);
  w->below = b.take<int>((size_t)h->cfg.n_layers * B);
  w->pos = b.take<int>(R);
  w->did_prune = b.take<int>(S);
  w->keep = b.take<unsigned char>(R);
  w->bytes = b.bytes();
}

__global__ void fill_empty_kernel(int64_t* m0, int64_t* m1, float* s0, float* s1, int* stop, int* p0, int* p1, int* nm,
                                  long n0, long n1, int B) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i < n0) { m0[i] = -1; s0[i] = 0.f; if (p0) p0[i] = 1; }
  if (i < n1) { m1[i] = -1; s1[i] = 0.f; if (p1) p1[i] = 1; }
  if (i < B) { if (stop) stop[i] = 1; if (nm) nm[i] = 0; }
}

// What lg_forward, lg_assign and lg_attention start from: the carved workspace, the sequence state and the launch count
// before their first launch (each reports the count's increase over the call).
struct Call {
  Workspace w;
  SeqState st;
  int64_t launches0;
};

// Carves the workspace and checks its size (the error starts with `who`), starts the launch count, and runs the first
// launch, misc_init_state (lens0 / lens1 null: M / N rows per pair).
int begin_call(LgHandle* h, const char* who, int B, int M, int N, const int* lens0, const int* lens1, void* workspace,
               size_t ws_bytes, cudaStream_t stream, Call* c) {
  Workspace& w = c->w;
  carve(h, B, M, N, (char*)workspace, &w);
  if (!workspace || ws_bytes < w.bytes) {
    char msg[64];
    snprintf(msg, sizeof(msg), "%s: workspace too small", who);
    return lg_set_error(msg);
  }
  c->launches0 = lg_launches;
  LG_RC(misc_init_state(w.lena, w.inda, w.prune, w.stop_layer, w.below, h->cfg.n_layers * B, B, M, N, w.Lp, lens0, lens1,
                        stream));
  c->st = SeqState{2 * B, B, w.Lp, w.lena, w.stop_layer};
  return 0;
}

// tc_block's counterpart on the CUDA cores (fp32): QKV, attention, out_proj, ffn.0, LayerNorm + GELU, ffn.3 + residual
int simt_block(LgHandle* h, const Workspace& w, const SeqState& st, int layer, int blk, float* x, const float* cs,
               cudaStream_t stream) {
  const BlockOff& o = blk == 0 ? h->bself : h->bcross;
  const float* bw = h->wpk + h->o_layers + (size_t)layer * h->layer_stride + (blk == 0 ? 0 : h->bself.total);
  GemmArgs g{};
  g.A0 = x; g.lda0 = D; g.K0 = D; g.K = D;
  g.W = bw + o.wp; g.bias = bw + o.bp; g.scale = 1.f;
  g.q = w.q; g.k = w.k; g.v = w.v; g.cs = cs;
  g.Nout = blk == 0 ? 3 * D : 2 * D;
  g.epi = blk == 0 ? EPI_QKV_ROPE : EPI_QK_V;
  { Timer t(h, LG_K_LINEAR, stream); LG_RC(simt_gemm(g, st, stream)); }
  {
    Timer t(h, LG_K_ATTENTION, stream);
    if (blk == 0) LG_RC(simt_attention(w.q, w.k, w.v, w.ctx, 0, st, stream));
    else LG_RC(simt_attention(w.q, w.q, w.v, w.ctx, st.B, st, stream));
  }
  Timer t(h, LG_K_LINEAR, stream);
  GemmArgs go{};  // out_proj / to_out
  go.A0 = w.ctx; go.lda0 = D; go.K0 = D; go.K = D; go.W = bw + o.wo; go.bias = bw + o.bo; go.Nout = D;
  go.epi = EPI_STORE; go.scale = 1.f; go.out = w.msg; go.ldo = D;
  LG_RC(simt_gemm(go, st, stream));
  GemmArgs g1{};  // ffn.0 on cat([x, msg])
  g1.A0 = x; g1.lda0 = D; g1.K0 = D; g1.A1 = w.msg; g1.lda1 = D; g1.K = F; g1.W = bw + o.w1; g1.bias = bw + o.b1;
  g1.Nout = F; g1.epi = EPI_STORE; g1.scale = 1.f; g1.out = w.hbuf; g1.ldo = F;
  LG_RC(simt_gemm(g1, st, stream));
  LG_RC(simt_layernorm_gelu(w.hbuf, bw + o.g, bw + o.be, st, stream));
  GemmArgs g2{};  // ffn.3 + residual
  g2.A0 = w.hbuf; g2.lda0 = F; g2.K0 = F; g2.K = F; g2.W = bw + o.w2; g2.bias = bw + o.b2; g2.Nout = D;
  g2.epi = EPI_RESID; g2.scale = 1.f; g2.out = x; g2.ldo = D;
  LG_RC(simt_gemm(g2, st, stream));
  return 0;
}
}  // namespace

extern "C" size_t lg_workspace_bytes(const LgHandle* h, int32_t B, int32_t M, int32_t N) {
  if (!h || B <= 0 || M < 0 || N < 0) return 0;
  Workspace w;
  carve(h, B, M, N, nullptr, &w);
  return w.bytes;
}

// the assignment tail shared by lg_forward and lg_assign
static int run_assign(LgHandle* h, const Workspace& w, const SeqState& st, const float* x, const int* ind, int M, int N,
                      const LgOutputs* out, cudaStream_t stream) {
  const float* abase = h->wpk + h->o_assign;
  // the whole materialising stage (final_proj + both sweeps + combines + dustbin + filter + output) as one interval
  Timer tstage(h, LG_K_ASSIGN_STAGE, stream, out->log_assignment != nullptr);
  {
    Timer t(h, LG_K_LINEAR, stream);
    if (h->cfg.precision == LG_PREC_FP32) {
      GemmArgs g{};
      g.A0 = x; g.lda0 = D; g.K0 = D; g.A1 = nullptr; g.lda1 = 0;
      g.W = abase + AO_FW; g.bias = abase + AO_FB;
      g.w_sel_stride = ASSIGN_BLOB_PAD; g.b_sel_stride = ASSIGN_BLOB_PAD;
      g.K = D; g.Nout = D; g.epi = EPI_STORE; g.scale = 0.25f;  // / 256^(1/4) (lightglue.py:291)
      g.out = w.ctx; g.ldo = D;
      LG_RC(simt_gemm(g, st, stream));
    } else {
      LG_RC(tc_final_proj(h, w.tc, st, w.ctx, stream));
    }
  }
  AssignArgs a{};
  a.p = w.ctx; a.x = x;
  a.mat_w = abase + AO_MW; a.mat_b = abase + AO_MB; a.mat_sel_stride = ASSIGN_BLOB_PAD;
  a.z = w.z; a.rowpart = w.rowpart; a.colpart = w.colpart; a.rowlse = w.rowlse; a.collse = w.collse;
  a.rowbest = w.rowbest; a.rowarg = w.rowarg; a.colbest = w.colbest; a.colarg = w.colarg; a.nt = w.nt;
  a.filter_threshold = h->cfg.filter_threshold;
  a.m0c = w.m0c; a.m1c = w.m1c; a.ms0c = w.ms0c; a.ms1c = w.ms1c;
  a.ind = ind; a.M = M; a.N = N;
  a.matches0 = out->matches0; a.matches1 = out->matches1; a.mscores0 = out->matching_scores0; a.mscores1 = out->matching_scores1;
  a.n_matches = out->n_matches; a.matches = out->matches; a.match_scores = out->match_scores; a.cap = M < N ? M : N;
  a.log_assignment = out->log_assignment;
  {
    Timer t(h, out->log_assignment ? LG_K_OTHER : LG_K_ASSIGN, stream);
    if (h->cfg.precision != LG_PREC_FP32 && st.Lp >= 256) {
      // both similarity sweeps on the tensor cores; the N x M matrix reaches HBM only if the caller asked for it
      LG_RC(tc_assign_sweeps(h, w.tc, st, a, w.tc_part, w.tc_parg, w.term, stream));
    } else {
      LG_RC(misc_assign(a, st, stream));
    }
  }
  return 0;
}

static int check_outputs(const LgOutputs* out) {
  if (!out || !out->matches0 || !out->matches1 || !out->matching_scores0 || !out->matching_scores1 || !out->n_matches ||
      !out->matches || !out->match_scores)
    return lg_set_error("LgOutputs: required output pointer is null");
  return 0;
}

extern "C" int lg_forward(LgHandle* h, const LgInputs* in, const LgOutputs* out, void* workspace, size_t ws_bytes,
                          void* stream_) {
  if (!h || !in || !out) return lg_set_error("lg_forward: null argument");
  const int B = in->B, M = in->M, N = in->N;
  if (B <= 0 || M < 0 || N < 0) return lg_set_error("lg_forward: bad shape");
  if (h->cfg.pos_dim == 4 && (M > 0 && N > 0) && (!in->scales0 || !in->oris0 || !in->scales1 || !in->oris1))
    return lg_set_error("lg_forward: scales/oris required when pos_dim == 4");
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool early = h->cfg.depth_confidence > 0, prune = h->cfg.width_confidence > 0;
  if (out->log_assignment && (early || prune)) return lg_set_error("lg_forward: log_assignment needs adaptivity off");
  if (M == 0 || N == 0) {  // lightglue.py:568-588: no keypoints -> nothing matched, stop = 1
    // (a zero-sized side may come with null pointers; the non-empty side's outputs must exist)
    if ((M > 0 && (!out->matches0 || !out->matching_scores0)) || (N > 0 && (!out->matches1 || !out->matching_scores1)))
      return lg_set_error("LgOutputs: required output pointer is null");
    const long n0 = (long)B * M, n1 = (long)B * N;
    long mx = n0 > n1 ? n0 : n1;
    if (mx < B) mx = B;
    const int64_t launches0 = lg_launches;
    fill_empty_kernel<<<(unsigned)((mx + 255) / 256), 256, 0, stream>>>(out->matches0, out->matches1, out->matching_scores0,
                                                                       out->matching_scores1, out->stop, out->prune0,
                                                                       out->prune1, out->n_matches, n0, n1, B);
    LG_CHECK_LAUNCH();
    h->launches = lg_launches - launches0;
    return 0;
  }
  LG_RC(check_outputs(out));
  if (!in->kpts0 || !in->kpts1 || !in->desc0 || !in->desc1) return lg_set_error("lg_forward: null input tensor");
  if (out->log_assignment && (in->lens0 || in->lens1))
    return lg_set_error("lg_forward: log_assignment is defined for dense batches only (no lens0/lens1)");
  Call c;
  LG_RC(begin_call(h, "lg_forward", B, M, N, in->lens0, in->lens1, workspace, ws_bytes, stream, &c));
  const Workspace& w = c.w;
  SeqState& st = c.st;
  const int L = h->cfg.n_layers, Lp = w.Lp;
  const bool fp32 = h->cfg.precision == LG_PREC_FP32;
  float *x = w.xa, *x_alt = w.xb, *cs = w.csa, *cs_alt = w.csb;
  int *len = w.lena, *len_alt = w.lenb, *ind = w.inda, *ind_alt = w.indb;

  {  // positional encoding, cached for all layers (lightglue.py:523-525)
    Timer t(h, LG_K_OTHER, stream);
    PosencArgs pa{in->kpts0, in->kpts1, in->size0, in->size1, in->scales0, in->oris0, in->scales1, in->oris1,
                  h->wpk + h->o_wr, h->cfg.pos_dim, B, M, N, Lp, cs, in->lens0, in->lens1};
    LG_RC(misc_posenc(pa, stream));
  }
  // descriptors -> residual stream (optionally through input_proj, lightglue.py:521-522)
  if (h->cfg.input_dim == (int)D) {
    LG_RC(misc_pack_desc(in->desc0, in->desc1, x, B, M, N, Lp, D, in->lens0, in->lens1, stream, fp32 ? nullptr : (void*)w.tc.xh,
                      fp32 ? nullptr : (void*)w.tc.xl));
  } else {
    LG_RC(misc_pack_desc(in->desc0, in->desc1, w.hbuf, B, M, N, Lp, h->cfg.input_dim, in->lens0, in->lens1, stream));
    Timer t(h, LG_K_LINEAR, stream);
    if (fp32) {
      GemmArgs g{};
      g.A0 = w.hbuf; g.lda0 = h->cfg.input_dim; g.K0 = h->cfg.input_dim;
      g.W = h->wpk + h->o_inw; g.bias = h->wpk + h->o_inb;
      g.K = h->cfg.input_dim; g.Nout = D; g.epi = EPI_STORE; g.scale = 1.f; g.out = x; g.ldo = D;
      LG_RC(simt_gemm(g, st, stream));
    } else {
      LG_RC(tc_input_proj(h, w.tc, st, w.hbuf, x, stream));
    }
  }

  for (int i = 0; i < L; ++i) {
    for (int blk = 0; blk < 2; ++blk)  // 0: SelfBlock (159-172), 1: CrossBlock (201-230)
      LG_RC(fp32 ? simt_block(h, w, st, i, blk, x, cs, stream) : tc_block(h, w.tc, st, i, blk, x, cs, stream));
    if (h->dbg_layers) {
      const size_t per = (size_t)2 * B * Lp * D;
      if ((size_t)(i + 1) * per > h->dbg_layers_floats) return lg_set_error("lg_debug_capture_layers: buffer too small");
      LG_CU(cudaMemcpyAsync(h->dbg_layers + (size_t)i * per, x, per * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
    if (i == L - 1) break;  // no early stopping or adaptive width at the last layer (544-545)
    if (!early && !prune) continue;
    Timer t(h, LG_K_OTHER, stream);
    AdaptArgs a{};
    a.x = x;
    const float* tk = h->wpk + h->o_token + (size_t)i * TOKEN_BLOB_PAD;
    const float* as = h->wpk + h->o_assign + (size_t)i * ASSIGN_BLOB_PAD;
    a.tok_w = early ? tk : nullptr; a.tok_b = early ? tk + D : nullptr;
    a.mat_w = prune ? as + AO_MW : nullptr; a.mat_b = prune ? as + AO_MB : nullptr;
    a.thr = h->thr[i]; a.depth_conf = h->cfg.depth_confidence; a.width_conf = h->cfg.width_confidence;
    a.layer = i; a.M = M; a.N = N; a.pruning_threshold = in->pruning_threshold;
    a.lens0 = in->lens0; a.lens1 = in->lens1;
    a.keep = w.keep; a.below = w.below + (size_t)i * B; a.stop_layer = w.stop_layer;
    a.len_in = len; a.len_out = prune ? len_alt : len; a.pos = w.pos; a.did_prune = w.did_prune;
    LG_RC(misc_adapt_score(a, st, stream));
    LG_RC(misc_adapt_decide(a, st, stream));
    if (prune) {
      GatherArgs ga{x, x_alt, cs, cs_alt, ind, ind_alt, w.prune, w.keep, w.pos, w.did_prune, len, len_alt, w.stop_layer, i};
      LG_RC(misc_adapt_gather(ga, st, stream));
      float* tf = x; x = x_alt; x_alt = tf;
      tf = cs; cs = cs_alt; cs_alt = tf;
      int* ti = ind; ind = ind_alt; ind_alt = ti;
      ti = len; len = len_alt; len_alt = ti;
      st.len = len;
      if (!fp32) LG_RC(tc_refresh_shadow(h, w.tc, x, st, stream));
    }
  }
  LG_RC(misc_finalize_stop(w.stop_layer, B, L, stream));
  LG_RC(run_assign(h, w, st, x, ind, M, N, out, stream));
  LG_RC(misc_export_stop_prune(w.stop_layer, w.prune, out->stop, out->prune0, out->prune1, B, M, N, Lp, stream));
  h->launches = lg_launches - c.launches0;
  return 0;
}

extern "C" int lg_assign(LgHandle* h, int32_t layer, int32_t B, int32_t M, int32_t N, const float* x0, const float* x1,
                         const LgOutputs* out, void* workspace, size_t ws_bytes, void* stream_) {
  if (!h || !x0 || !x1) return lg_set_error("lg_assign: null argument");
  LG_RC(check_outputs(out));
  if (B <= 0 || M <= 0 || N <= 0 || layer < 0 || layer >= h->cfg.n_layers) return lg_set_error("lg_assign: bad shape/layer");
  cudaStream_t stream = (cudaStream_t)stream_;
  Call c;
  LG_RC(begin_call(h, "lg_assign", B, M, N, nullptr, nullptr, workspace, ws_bytes, stream, &c));
  const Workspace& w = c.w;
  LG_RC(misc_finalize_stop(w.stop_layer, B, layer + 1, stream));  // selects log_assignment[layer] for every pair
  LG_RC(misc_pack_desc(x0, x1, w.xa, B, M, N, w.Lp, D, nullptr, nullptr, stream));
  if (h->cfg.precision != LG_PREC_FP32) LG_RC(tc_refresh_shadow(h, w.tc, w.xa, c.st, stream));
  LG_RC(run_assign(h, w, c.st, w.xa, w.inda, M, N, out, stream));
  h->launches = lg_launches - c.launches0;
  return 0;
}

extern "C" int lg_attention(LgHandle* h, int32_t B, int32_t M, int32_t N, int32_t cross, const float* q0, const float* k0,
                            const float* v0, const float* q1, const float* k1, const float* v1, float* ctx0, float* ctx1,
                            void* workspace, size_t ws_bytes, void* stream_) {
  if (!h || !q0 || !k0 || !v0 || !q1 || !k1 || !v1 || !ctx0 || !ctx1) return lg_set_error("lg_attention: null argument");
  if (B <= 0 || M <= 0 || N <= 0) return lg_set_error("lg_attention: bad shape");
  cudaStream_t stream = (cudaStream_t)stream_;
  Call c;
  LG_RC(begin_call(h, "lg_attention", B, M, N, nullptr, nullptr, workspace, ws_bytes, stream, &c));
  const Workspace& w = c.w;
  const bool fp32 = h->cfg.precision == LG_PREC_FP32;
  AttnIoArgs a{};
  a.q0 = q0; a.k0 = k0; a.v0 = v0; a.q1 = q1; a.k1 = k1; a.v1 = v1;
  a.B = B; a.M = M; a.N = N; a.Lp = w.Lp;
  if (fp32) { a.qf = w.q; a.kf = w.k; a.vf = w.v; a.ctxf = w.ctx; }
  else { a.qh = w.tc.q; a.kh = w.tc.k; a.vth = w.tc.vt; a.ctxh = w.tc.ctxh; a.ctxl = w.tc.ctxl; }
  a.out0 = ctx0; a.out1 = ctx1;
  LG_RC(misc_attn_pack(a, stream));
  {
    Timer t(h, LG_K_ATTENTION, stream);
    if (fp32) LG_RC(simt_attention(w.q, w.k, w.v, w.ctx, cross ? B : 0, c.st, stream));
    else LG_RC(tc_attention(h, w.tc, c.st, cross ? B : 0, w.tc.k, stream));
  }
  LG_RC(misc_attn_unpack(a, stream));
  h->launches = lg_launches - c.launches0;
  return 0;
}
