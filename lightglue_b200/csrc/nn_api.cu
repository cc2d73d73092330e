// C ABI of the nearest-neighbour matcher (include/nn_b200.h): per group of pairs, the split into bf16 hi / lo images,
// the tensor-core top-2 sweep of both directions (k_tc_linear.cu, TEPI_TOP2) and one CTA per pair for the tests and
// the outputs.
#include <math.h>
#include <stdint.h>

#include <new>

#include "../../include/nn_b200.h"
#include "block_scan.cuh"
#include "lg_internal.h"
#include "lg_tc.h"
#include "ws_bump.h"

struct NnHandle {
  TcEngine tc;  // no weights: its tensor-map cache only
};

namespace {

constexpr int TAIL_THREADS = 1024;

// Sequence layout of one group of G pairs, as the matcher's: sequence s < G is image 0 of pair s, s >= G image 1 of pair
// s - G, each Lp rows.  Per row of a group: the bf16 images, the sweep's slot partials and the row's kept j / s1.
struct NnWs {
  int G, Lp, pstride;
  __nv_bfloat16 *hi, *lo;  // [2G Lp, D]
  float* part;             // [2G Lp, pstride] (s1, s2)
  int* parg;               // [2G Lp, pstride] j1
  int* jbest;              // [2G Lp] j1 when the row passes its tests, else -1
  float* sbest;            // [2G Lp] s1
  int* len;                // [2G] rows of each sequence
  int* stop;               // [G] zero: the sweep's per-pair stop words
};

size_t carve(char* base, int B, int M, int N, int D, NnWs* w) {
  const int mx = M > N ? M : N;
  w->Lp = ((mx > 0 ? mx : 1) + LG_TILE - 1) / LG_TILE * LG_TILE;
  const int gmax = NN_GROUP_ROWS / w->Lp > 1 ? NN_GROUP_ROWS / w->Lp : 1;
  const int groups = (B + gmax - 1) / gmax;
  w->G = groups > 0 ? (B + groups - 1) / groups : 0;  // balanced groups
  w->pstride = 2 * ((w->Lp + 255) / 256);
  const size_t R = 2 * (size_t)w->G * w->Lp;
  WsBump b{base, 0};
  w->hi = b.take<__nv_bfloat16>(R * D, 1024);
  w->lo = b.take<__nv_bfloat16>(R * D, 1024);
  w->part = b.take<float>(R * w->pstride * 2);
  w->parg = b.take<int>(R * w->pstride);
  w->jbest = b.take<int>(R);
  w->sbest = b.take<float>(R);
  w->len = b.take<int>(2 * (size_t)w->G);
  w->stop = b.take<int>(w->G);
  return b.bytes();
}

__device__ __forceinline__ int pair_len(const int* lens, int b, int cap) {
  if (!lens) return cap;
  const int v = lens[b];
  return v < 0 ? 0 : v > cap ? cap : v;
}

struct PackArgs {
  const float *d0, *d1;
  const int *lens0, *lens1;
  int b0, g, M, N, D, Lp;  // pairs b0 .. b0 + g - 1
  __nv_bfloat16 *hi, *lo;
  int *len, *stop;
};

// descriptors -> bf16 hi / lo rows of the group's sequences, zero past each length; the length and stop words
__global__ void __launch_bounds__(256) nn_pack_kernel(PackArgs a) {
  const int q = a.D / 4;
  const long total = 2L * a.g * a.Lp * q;
  const long tid = blockIdx.x * 256L + threadIdx.x;
  if (tid < 2 * a.g) {
    const bool im1 = tid >= a.g;
    const int pb = a.b0 + (int)(im1 ? tid - a.g : tid);
    a.len[tid] = pair_len(im1 ? a.lens1 : a.lens0, pb, im1 ? a.N : a.M);
    if (!im1) a.stop[tid] = 0;
  }
  for (long idx = tid; idx < total; idx += (long)gridDim.x * 256) {
    const long row = idx / q;
    const int c = (int)(idx % q) * 4;
    const int s = (int)(row / a.Lp), r = (int)(row % a.Lp);
    const bool im1 = s >= a.g;
    const int pb = a.b0 + (im1 ? s - a.g : s);
    const int cap = im1 ? a.N : a.M;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < pair_len(im1 ? a.lens1 : a.lens0, pb, cap))
      v = *reinterpret_cast<const float4*>((im1 ? a.d1 : a.d0) + ((long)pb * cap + r) * a.D + c);
    __nv_bfloat16 h[4], l[4];
    tc_split(v.x, h[0], l[0]); tc_split(v.y, h[1], l[1]); tc_split(v.z, h[2], l[2]); tc_split(v.w, h[3], l[3]);
    *reinterpret_cast<uint2*>(a.hi + row * a.D + c) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(a.lo + row * a.D + c) = *reinterpret_cast<const uint2*>(l);
  }
}

struct TailArgs {
  const float2* part; const int* parg; int pstride;
  int* jbest; float* sbest;
  const int* len;
  int g, Lp, M, N;
  float r2, t2;  // <= 0: test off
  int mutual;
  // outputs of the group's first pair
  int64_t *m0, *m1; float *ms0, *ms1; int* n_matches; int64_t* matches; float* mscores;
};

// One CTA per pair: merge the slots of every row of both sides into (j1, s1, s2) and apply the ratio and distance
// tests; then the mutual check, the outputs at every row, and the ordered `matches` list (ascending i).
__global__ void __launch_bounds__(TAIL_THREADS, 1) nn_tail_kernel(TailArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int m = a.len[b], n = a.len[a.g + b];
  const long row0 = (long)b * a.Lp, row1 = (long)(a.g + b) * a.Lp;
  for (int side = 0; side < 2; ++side) {
    const int rows = side ? n : m, cols = side ? m : n;
    const int nt = (cols + 127) / 128;  // slots with live columns
    for (int r = tid; r < rows; r += TAIL_THREADS) {
      const long row = (side ? row1 : row0) + r;
      const float2* pt = a.part + row * a.pstride;
      const int* pa = a.parg + row * a.pstride;
      float s1 = -INFINITY, s2 = -INFINITY;
      int j = -1;
      for (int t = 0; t < nt; ++t) {  // ascending slots: on a tie the earlier slot (lower j) keeps its place
        const float2 v = pt[t];
        if (v.x > s1) { s2 = fmaxf(s1, v.y); s1 = v.x; j = pa[t]; }
        else s2 = fmaxf(s2, v.x);
      }
      const float d1 = 2.f * (1.f - s1), d2 = 2.f * (1.f - s2);  // s2 = -inf: d2 = +inf
      const bool keep = (a.r2 <= 0.f || d1 <= a.r2 * d2) && (a.t2 <= 0.f || d1 <= a.t2);
      a.jbest[row] = keep && j >= 0 && j < cols ? j : -1;
      a.sbest[row] = s1;
    }
  }
  __syncthreads();
  for (int j = tid; j < a.N; j += TAIL_THREADS) {
    int i = j < n ? a.jbest[row1 + j] : -1;
    if (i >= 0 && a.mutual && a.jbest[row0 + i] != j) i = -1;
    a.m1[(long)b * a.N + j] = i;
    a.ms1[(long)b * a.N + j] = i >= 0 ? (a.sbest[row1 + j] + 1.f) * 0.5f : 0.f;
  }
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < a.M; base += TAIL_THREADS) {
    const int i = base + tid;
    int j = i < m ? a.jbest[row0 + i] : -1;
    if (j >= 0 && a.mutual && a.jbest[row1 + j] != i) j = -1;
    const float sc = j >= 0 ? (a.sbest[row0 + i] + 1.f) * 0.5f : 0.f;
    if (i < a.M) {
      a.m0[(long)b * a.M + i] = j;
      a.ms0[(long)b * a.M + i] = sc;
    }
    const int slot = block_scan_step(j >= 0, tid, warp_sums, &carry);
    if (j >= 0) {
      a.matches[((long)b * a.M + slot) * 2] = i;
      a.matches[((long)b * a.M + slot) * 2 + 1] = j;
      a.mscores[(long)b * a.M + slot] = sc;
    }
  }
  if (tid == 0) a.n_matches[b] = carry;
}

}  // namespace

extern "C" int nn_create(void* stream, NnHandle** out) {
  if (!out) return lg_set_error("nn_create: null argument");
  *out = nullptr;
  NnHandle* h = new (std::nothrow) NnHandle{};
  if (!h) return lg_set_error("nn_create: out of host memory");
  if (int r = tc_engine_create(&h->tc, nullptr, 0, true, (cudaStream_t)stream)) {
    tc_engine_destroy(&h->tc);
    delete h;
    return r;
  }
  *out = h;
  return 0;
}

extern "C" int nn_destroy(NnHandle* h) {
  if (!h) return 0;
  tc_engine_destroy(&h->tc);
  delete h;
  return 0;
}

static bool dim_ok(int D) { return D >= NN_MIN_DIM && D <= NN_MAX_DIM && D % 64 == 0; }

extern "C" size_t nn_workspace_bytes(int32_t B, int32_t M, int32_t N, int32_t D) {
  if (B < 0 || M < 0 || N < 0 || !dim_ok(D)) return 0;
  NnWs w;
  return carve(nullptr, B, M, N, D, &w);
}

extern "C" int nn_match(NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnOutputs* out, void* workspace,
                        size_t workspace_bytes, void* stream_) {
  if (!h || !cfg || !in || !out) return lg_set_error("nn_match: null argument");
  if (cfg->abi_version != NN_ABI_VERSION) return lg_set_error("nn_match: ABI version mismatch");
  const int B = in->B, M = in->M, N = in->N, D = cfg->dim;
  if (!dim_ok(D)) return lg_set_error("nn_match: dim must be a multiple of 64 in [64, 512]");
  if (B < 0 || M < 0 || N < 0) return lg_set_error("nn_match: negative size");
  if (!isfinite(cfg->ratio_thresh) || cfg->ratio_thresh > 1.f) return lg_set_error("nn_match: ratio_thresh must be <= 1");
  if (!isfinite(cfg->distance_thresh)) return lg_set_error("nn_match: distance_thresh must be finite");
  if (B == 0) return 0;
  if ((M > 0 && (!in->desc0 || !out->matches0 || !out->matching_scores0 || !out->matches || !out->match_scores)) ||
      (N > 0 && (!in->desc1 || !out->matches1 || !out->matching_scores1)) || !out->n_matches)
    return lg_set_error("nn_match: required pointer is null");
  if ((reinterpret_cast<uintptr_t>(in->desc0) | reinterpret_cast<uintptr_t>(in->desc1)) & 15)
    return lg_set_error("nn_match: descriptors must be 16-byte aligned");
  NnWs w;
  if (!workspace || workspace_bytes < carve(nullptr, B, M, N, D, &w)) return lg_set_error("nn_match: workspace too small");
  carve(static_cast<char*>(workspace), B, M, N, D, &w);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const double r = cfg->ratio_thresh, t = cfg->distance_thresh;
  TailArgs ta{};
  ta.part = reinterpret_cast<const float2*>(w.part); ta.parg = w.parg; ta.pstride = w.pstride;
  ta.jbest = w.jbest; ta.sbest = w.sbest; ta.len = w.len;
  ta.Lp = w.Lp; ta.M = M; ta.N = N;
  ta.r2 = r > 0 ? (float)(r * r) : 0.f;
  ta.t2 = t > 0 ? (float)(t * t) : 0.f;
  ta.mutual = cfg->mutual_check != 0;
  for (int b0 = 0; b0 < B; b0 += w.G) {
    const int g = B - b0 < w.G ? B - b0 : w.G;
    PackArgs pa{in->desc0, in->desc1, in->lens0, in->lens1, b0, g, M, N, D, w.Lp, w.hi, w.lo, w.len, w.stop};
    const long groups4 = 2L * g * w.Lp * (D / 4);
    const long blocks = (groups4 + 255) / 256;
    nn_pack_kernel<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256, 0, stream>>>(pa);
    LG_CHECK_LAUNCH();
    const SeqState st{2 * g, g, w.Lp, w.len, w.stop};
    LG_RC(tc_nn_sweep(h->tc, st, w.hi, w.lo, D, w.part, w.parg, w.pstride, stream));
    ta.g = g;
    ta.m0 = out->matches0 + (long)b0 * M; ta.ms0 = out->matching_scores0 + (long)b0 * M;
    ta.m1 = out->matches1 + (long)b0 * N; ta.ms1 = out->matching_scores1 + (long)b0 * N;
    ta.n_matches = out->n_matches + b0;
    ta.matches = out->matches + (long)b0 * M * 2; ta.mscores = out->match_scores + (long)b0 * M;
    nn_tail_kernel<<<g, TAIL_THREADS, 0, stream>>>(ta);
    LG_CHECK_LAUNCH();
  }
  return 0;
}
