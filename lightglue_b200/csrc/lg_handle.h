// The handle behind the C ABI, shared by the orchestration (lg_api.cu) and the tensor-core path.
#pragma once
#include <vector>

#include "../../include/lightglue_b200.h"
#include "lg_internal.h"
#include "lg_tc.h"

// packed per-block fp32 layout (floats):
//   Wp [Np,256] | bp [Np] | Wo [256,256] | bo | W1 [512,512] | b1 | ln.g | ln.b | W2 [256,512] | b2 | W1f [512,512] | b1f
// W1f / b1f: ffn.0 with the attention output projection folded in (tensor-core path):
//   ffn.0(cat[x, out_proj(ctx)]) = W1[:, :256] x + (W1[:, 256:] Wo) ctx + (b1 + W1[:, 256:] bo)
// so the block runs cat[x, ctx] through ONE GEMM and `msg` never exists (lightglue.py:171-172, 227-229).
struct BlockOff {
  size_t wp, bp, wo, bo, w1, b1, g, be, w2, b2, w1f, b1f, total;
};
inline BlockOff block_off(size_t np) {
  BlockOff o;
  size_t c = 0;
  o.wp = c; c += np * LG_DIM;
  o.bp = c; c += np;
  o.wo = c; c += (size_t)LG_DIM * LG_DIM;
  o.bo = c; c += LG_DIM;
  o.w1 = c; c += (size_t)LG_FFN * LG_FFN;
  o.b1 = c; c += LG_FFN;
  o.g = c; c += LG_FFN;
  o.be = c; c += LG_FFN;
  o.w2 = c; c += (size_t)LG_DIM * LG_FFN;
  o.b2 = c; c += LG_DIM;
  o.w1f = c; c += (size_t)LG_FFN * LG_FFN;
  o.b1f = c; c += LG_FFN;
  o.total = c;
  return o;
}

struct LgHandle {
  LgConfig cfg;
  int device;
  float* wpk;  // packed fp32 weights (device)
  size_t wpk_floats;
  size_t o_wr, o_inw, o_inb, o_layers, o_assign, o_token;  // offsets into wpk
  BlockOff bself, bcross;
  size_t layer_stride;
  float thr[64];  // confidence_thresholds (lightglue.py:631-634)
  TcEngine tc;    // tensor-core path: bf16 hi/lo copies of wpk, tensor maps (all zero in fp32 mode)
  int64_t launches;
  float* dbg_layers; size_t dbg_layers_floats;  // lg_debug_capture_layers
  bool timing;
  std::vector<cudaEvent_t> ev[LG_K_CLASSES];
  size_t ev_used[LG_K_CLASSES];
};

// Records a CUDA-event pair on the launching stream around the launches in its scope (bench.py's
// per-kernel-class device times).  No-op unless lg_timing_enable(h, 1).
struct Timer {
  LgHandle* h; int kc; cudaStream_t s; bool on;
  // Timers of the SAME class must not nest (they share one cursor); `enable` = false makes this one inert.
  Timer(LgHandle* h_, int kc_, cudaStream_t s_, bool enable = true) : h(h_), kc(kc_), s(s_), on(h_->timing && enable) {
    if (!on) return;
    if (h->ev_used[kc] + 2 > 40000) { on = false; return; }
    while (h->ev[kc].size() < h->ev_used[kc] + 2) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
      h->ev[kc].push_back(e);
    }
    cudaEventRecord(h->ev[kc][h->ev_used[kc]], s);
  }
  ~Timer() {
    if (!on) return;
    cudaEventRecord(h->ev[kc][h->ev_used[kc] + 1], s);
    h->ev_used[kc] += 2;
  }
};
