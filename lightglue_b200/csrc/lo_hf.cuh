// The LO-RANSAC pieces shared by the homography (lo_homography_api.cu, header steps LH1-LH8) and the fundamental
// matrix (lo_fundamental_api.cu, LF1-LF8), both compiled with -fmad=false: the per-pair state, the workspace, and the
// hyp and score kernels of each chunk.  The LM and final kernels are each model's own.
#pragma once
#include <stdint.h>

#include "geo_hf.cuh"
#include "lo_common.cuh"

namespace {

struct LoHfPair {
  double model[9];           // the pair's model in pixels, scaled as step 4
  unsigned long long score;  // its LH3 / LF3 score
  int count;                 // its inliers
  int h;                     // the hypothesis that seeded it; -1: none yet
  int nlo;                   // local optimisations adopted
};

struct LoHfWs {
  LoHfPair* pair;           // [B]
  unsigned long long* acc;  // [B, GEO_CHUNK] count << 40 | score of the current chunk's hypotheses
};

size_t lohf_carve(char* base, int B, int M, GeoWs* w, LoHfWs* l) {
  WsBump b{base, carve(base, B, M, w)};
  l->pair = b.take<LoHfPair>(B);
  l->acc = b.take<unsigned long long>((size_t)B * GEO_CHUNK);
  return b.bytes();
}

struct LoHfArgs {
  GeoArgs g;
  LoHfWs l;
  int32_t* num_lo;
  int64_t* cost;
};

// Step 4's hypotheses of chunk c (a.g.kind and a.g.s pick H or F), one thread per sample
__global__ void __launch_bounds__(GEO_CHUNK, 1) lohf_hyp_kernel(LoHfArgs a, int c) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (c == 0 && t == 0) {
    LoHfPair& L = a.l.pair[b];
    L.score = 0;
    L.count = 0;
    L.h = -1;
    L.nlo = 0;
  }
  const GeoPair& P = a.g.w.pair[b];
  const int h = c * GEO_CHUNK + t;
  double m[9];
  const bool ok = P.stop == 0 && h < a.g.max_iters && geo_hypothesis(a.g, P, a.g.w.pts + (long)b * a.g.M, h, m);
  if (ok) {
    float* hm = a.g.w.hyp + ((long)b * GEO_CHUNK + t) * 9;
    for (int i = 0; i < 9; ++i) hm[i] = (float)m[i];
    a.l.acc[(long)b * GEO_CHUNK + t] = 0;
  }
  a.g.w.count[(long)b * GEO_CHUNK + t] = ok ? 0 : -1;
}

// The chunk's LH3 / LF3 scores: (B, splits) CTAs, each streams a slice of the pair's points through shared memory
template <int KIND>
__global__ void __launch_bounds__(GEO_CHUNK) lohf_score_kernel(LoHfArgs a) {
  const int b = blockIdx.x, split = blockIdx.y, t = threadIdx.x;
  const GeoPair& P = a.g.w.pair[b];
  if (P.stop) return;
  const int lo = (int)((long)P.n * split / gridDim.y), hi = (int)((long)P.n * (split + 1) / gridDim.y);
  const bool valid = a.g.w.count[(long)b * GEO_CHUNK + t] >= 0;
  float h[9];
  for (int i = 0; i < 9; ++i) h[i] = valid ? a.g.w.hyp[((long)b * GEO_CHUNK + t) * 9 + i] : 0.f;
  const float thr2 = a.g.thr2;
  const float w = (float)GEO_LO_QSCALE / thr2;
  const float4* pts = a.g.w.pts + (long)b * a.g.M;
  __shared__ float4 tile[TILE];
  unsigned long long k = 0;
  for (int base = lo; base < hi; base += TILE) {
    const int m = min(TILE, hi - base);
    __syncthreads();
    for (int i = t; i < m; i += GEO_CHUNK) tile[i] = pts[base + i];
    __syncthreads();
    if (valid)
      for (int i = 0; i < m; ++i) k += lo_term(geo_err(KIND, h, tile[i]), thr2, w);
  }
  if (k) atomicAdd(a.l.acc + (long)b * GEO_CHUNK + t, k);
}

}  // namespace
