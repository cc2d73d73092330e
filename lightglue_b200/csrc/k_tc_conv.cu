// Host plumbing of the tensor-core convolution owners (SuperPoint's backbone, DISK, HardNet; lg_tc.h): the row plan of
// their operands and their packed weights.  The convolution itself is tc_conv (k_tc_linear.cu).
#include <algorithm>
#include <new>

#include "lg_tc.h"

namespace {

// one block per row of the region: see TcConvRegion
__global__ void tc_conv_pack_kernel(const TcConvRegion g, float* __restrict__ wo, float* __restrict__ bo) {
  const int r = blockIdx.x, co = g.co0 + r;
  const bool live = r < g.ncopy;
  const double rs = live && g.bn_var ? 1.0 / sqrt((double)g.bn_var[co] + 1e-5) : 0.0;
  for (int idx = threadIdx.x; idx < g.K; idx += blockDim.x) {
    const int tap = idx / g.cpad, ci = idx % g.cpad;
    float v = 0.f;
    if (live && tap < g.taps && ci < g.cin) {
      const float s = g.w[((size_t)co * g.cin + ci) * g.taps + tap];
      v = g.bn_var ? (float)((double)s * rs) : s;
    }
    wo[(size_t)r * g.K + idx] = v;
  }
  if (threadIdx.x == 0) bo[r] = !live ? 0.f : g.bn_var ? (float)(-(double)g.bn_mean[co] * rs) : g.b[co];
}

size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }

}  // namespace

TcRows tc_rows(long used) {
  const int Lp = (int)std::max<long>(LG_TILE, ((used + 1) / 2 + LG_TILE - 1) / LG_TILE * LG_TILE);
  return TcRows{Lp, 2L * Lp};
}

int tc_rows_words(const TcRows* r, int n, int* words, cudaStream_t stream) {
  int host[4 * 8] = {0};
  if (n > 8) return lg_set_error("tc_rows_words: at most 8 matrices");
  for (int i = 0; i < n; ++i) { host[4 * i] = r[i].Lp; host[4 * i + 1] = r[i].Lp; }
  LG_CU(cudaMemcpyAsync(words, host, 4 * n * sizeof(int), cudaMemcpyHostToDevice, stream));
  return 0;
}

int tc_conv_weights_create(TcConvWeights** out, const TcConvRegion* reg, int n, cudaStream_t stream) {
  if (n > TC_CONV_MAX_REGIONS) return lg_set_error("tc_conv_weights_create: too many regions");
  TcConvWeights* cw = new (std::nothrow) TcConvWeights{};
  if (!cw) return lg_set_error("tc_conv_weights_create: out of host memory");
  struct Guard {
    TcConvWeights* cw;
    ~Guard() { tc_conv_weights_destroy(cw); }
  } guard{cw};
  size_t c = 0;
  for (int i = 0; i < n; ++i) {
    cw->w_off[i] = c; c = align64(c + (size_t)reg[i].rows * reg[i].K);
    cw->b_off[i] = c; c = align64(c + reg[i].rows);
  }
  LG_CU(cudaMalloc(&cw->wpk, c * sizeof(float)));
  LG_CU(cudaMemsetAsync(cw->wpk, 0, c * sizeof(float), stream));  // the alignment gaps
  for (int i = 0; i < n; ++i)
    tc_conv_pack_kernel<<<reg[i].rows, 256, 0, stream>>>(reg[i], cw->wpk + cw->w_off[i], cw->wpk + cw->b_off[i]);
  LG_CHECK_LAUNCH();
  LG_RC(tc_engine_create(&cw->tc, cw->wpk, c, true, stream));
  guard.cw = nullptr;
  *out = cw;
  return 0;
}

void tc_conv_weights_destroy(TcConvWeights* cw) {
  if (!cw) return;
  tc_engine_destroy(&cw->tc);
  cudaFree(cw->wpk);
  delete cw;
}
