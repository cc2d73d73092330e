// C ABI of the nearest-neighbour matcher (include/nn_b200.h): per group of pairs, the split into bf16 hi / lo images,
// the tensor-core top-2 sweep of both directions (k_tc_linear.cu, TEPI_TOP2) and one CTA per pair for the tests and
// the outputs.  Guided matching adds one launch per group that writes the gate records, and runs the sweep with the
// gated epilogue (TEPI_TOP2_H / TEPI_TOP2_F).
#include <math.h>
#include <stdint.h>
#include <stdio.h>

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
  float* rec;              // guided only: [GATE_FIELDS][2G Lp] the rows' gate records
  int* gate_on;            // guided only: [G] non-zero for a guided pair
};

constexpr int GATE_FIELDS = 6;  // F: x, y, a, b, c, s; H uses the first two

size_t carve(char* base, int B, int M, int N, int D, NnWs* w, bool guided = false) {
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
  w->rec = guided ? b.take<float>(R * GATE_FIELDS) : nullptr;
  w->gate_on = guided ? b.take<int>(w->G) : nullptr;
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

struct GateArgs {
  const double* model; const uint8_t* valid;
  const float *k0, *k1;
  int b0, g, M, N, Lp;  // pairs b0 .. b0 + g - 1
  int fundamental;
  float* rec; int* on;
};

// One thread per row of the group's sequences: the row's gate record, from step 5 of include/geometry_b200.h in fp32
// with every operation rounded on its own (this file is compiled with fused multiply-adds allowed), the model rounded
// to float.  H: an image-0 row stores its projected point ((h0 x + h1 y) + h2) w, ((h3 x + h4 y) + h5) w with
// w = 1 / ((h6 x + h7 y) + h8), an image-1 row its point.  F: a row stores its point, its epipolar line in the other
// image (F x0 row by row for image 0, F^T x1 for image 1) and 1 / (a^2 + b^2).  Rows past M / N store zeros.
__global__ void __launch_bounds__(256) nn_gate_record_kernel(GateArgs a) {
  const long rows = 2L * a.g * a.Lp;
  const long row = blockIdx.x * 256L + threadIdx.x;
  if (row < a.g) a.on[row] = a.valid ? a.valid[a.b0 + row] != 0 : 1;
  if (row >= rows) return;
  const int s = (int)(row / a.Lp), r = (int)(row % a.Lp);
  const bool im1 = s >= a.g;
  const int pb = a.b0 + (im1 ? s - a.g : s);
  const int cap = im1 ? a.N : a.M;
  float v[GATE_FIELDS] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (r < cap) {
    const float2 x = reinterpret_cast<const float2*>(im1 ? a.k1 : a.k0)[(long)pb * cap + r];
    float h[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = (float)a.model[(long)pb * 9 + k];
    // (u x + v y) + w, rounded step by step
    auto lin = [&](float u, float vv, float w) { return __fadd_rn(__fadd_rn(__fmul_rn(u, x.x), __fmul_rn(vv, x.y)), w); };
    v[0] = x.x; v[1] = x.y;
    if (!a.fundamental) {
      if (!im1) {
        const float w = __fdiv_rn(1.f, lin(h[6], h[7], h[8]));
        v[0] = __fmul_rn(lin(h[0], h[1], h[2]), w);
        v[1] = __fmul_rn(lin(h[3], h[4], h[5]), w);
      }
    } else {
      const float la = im1 ? lin(h[0], h[3], h[6]) : lin(h[0], h[1], h[2]);
      const float lb = im1 ? lin(h[1], h[4], h[7]) : lin(h[3], h[4], h[5]);
      const float lc = im1 ? lin(h[2], h[5], h[8]) : lin(h[6], h[7], h[8]);
      v[2] = la; v[3] = lb; v[4] = lc;
      v[5] = __fdiv_rn(1.f, __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb)));
    }
  }
  const int fields = a.fundamental ? GATE_FIELDS : 2;
  for (int f = 0; f < fields; ++f) a.rec[f * rows + row] = v[f];
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

extern "C" size_t nn_guided_workspace_bytes(int32_t B, int32_t M, int32_t N, int32_t D) {
  if (B < 0 || M < 0 || N < 0 || !dim_ok(D)) return 0;
  NnWs w;
  return carve(nullptr, B, M, N, D, &w, true);
}

extern "C" int64_t nn_workspace_layout(int32_t B, int32_t M, int32_t N, int32_t D, int32_t guided, int64_t* offsets,
                                       int64_t* bytes, int32_t* plan) {
  if (B < 1 || M < 0 || N < 0 || !dim_ok(D)) return 0;
  NnWs w;
  char* const base = reinterpret_cast<char*>(kLayoutBase);
  const size_t total = carve(base, B, M, N, D, &w, guided != 0);
  const size_t R = 2 * (size_t)w.G * w.Lp, G = (size_t)w.G, f = sizeof(float), i = sizeof(int), h = sizeof(__nv_bfloat16);
  const struct { const void* p; size_t n; } buf[NN_LAYOUT_BUFFERS] = {
      {w.hi, R * D * h}, {w.lo, R * D * h},       {w.part, R * w.pstride * 2 * f}, {w.parg, R * w.pstride * i},
      {w.jbest, R * i},  {w.sbest, R * f},        {w.len, 2 * G * i},              {w.stop, G * i},
      {w.rec, R * GATE_FIELDS * f}, {w.gate_on, G * i}};
  for (int k = 0; k < NN_LAYOUT_BUFFERS; ++k) {
    if (offsets) offsets[k] = buf[k].p ? (int64_t)((const char*)buf[k].p - base) : -1;
    if (bytes) bytes[k] = buf[k].p ? (int64_t)buf[k].n : 0;
  }
  if (plan) {
    plan[0] = w.G;
    plan[1] = w.Lp;
    plan[2] = w.pstride;
    plan[3] = (B + w.G - 1) / w.G;
  }
  return (int64_t)total;
}

static int nn_error(const char* entry, const char* what) {
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", entry, what);
  return lg_set_error(msg);
}

// nn_match and nn_match_guided (guide non-null): the argument checks, then per group the pack, [the gate records,] the
// sweep and the tail
static int nn_run(const char* entry, NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnGuide* guide,
                  const NnOutputs* out, void* workspace, size_t workspace_bytes, void* stream_) {
  const bool guided = guide != nullptr;
  if (!h || !cfg || !in || !out) return nn_error(entry, "null argument");
  if (cfg->abi_version != NN_ABI_VERSION) return nn_error(entry, "ABI version mismatch");
  const int B = in->B, M = in->M, N = in->N, D = cfg->dim;
  if (!dim_ok(D)) return nn_error(entry, "dim must be a multiple of 64 in [64, 512]");
  if (B < 0 || M < 0 || N < 0) return nn_error(entry, "negative size");
  if (!isfinite(cfg->ratio_thresh) || cfg->ratio_thresh > 1.f) return nn_error(entry, "ratio_thresh must be <= 1");
  if (!isfinite(cfg->distance_thresh)) return nn_error(entry, "distance_thresh must be finite");
  if (guided) {
    if (guide->kind != NN_GUIDE_H && guide->kind != NN_GUIDE_F) return nn_error(entry, "kind must be NN_GUIDE_H or NN_GUIDE_F");
    if (!(guide->max_error > 0.0) || !isfinite(guide->max_error)) return nn_error(entry, "max_error must be positive and finite");
  }
  if (B == 0) return 0;
  if ((M > 0 && (!in->desc0 || !out->matches0 || !out->matching_scores0 || !out->matches || !out->match_scores)) ||
      (N > 0 && (!in->desc1 || !out->matches1 || !out->matching_scores1)) || !out->n_matches)
    return nn_error(entry, "required pointer is null");
  if ((reinterpret_cast<uintptr_t>(in->desc0) | reinterpret_cast<uintptr_t>(in->desc1)) & 15)
    return nn_error(entry, "descriptors must be 16-byte aligned");
  if (guided) {
    if (!guide->model || (M > 0 && !guide->kpts0) || (N > 0 && !guide->kpts1))
      return nn_error(entry, "model or keypoint pointer is null");
    if ((reinterpret_cast<uintptr_t>(guide->model) | reinterpret_cast<uintptr_t>(guide->kpts0) |
         reinterpret_cast<uintptr_t>(guide->kpts1)) & 7)
      return nn_error(entry, "model and keypoints must be 8-byte aligned");
  }
  NnWs w;
  if (!workspace || workspace_bytes < carve(nullptr, B, M, N, D, &w, guided)) return nn_error(entry, "workspace too small");
  carve(static_cast<char*>(workspace), B, M, N, D, &w, guided);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const double r = cfg->ratio_thresh, t = cfg->distance_thresh;
  TailArgs ta{};
  ta.part = reinterpret_cast<const float2*>(w.part); ta.parg = w.parg; ta.pstride = w.pstride;
  ta.jbest = w.jbest; ta.sbest = w.sbest; ta.len = w.len;
  ta.Lp = w.Lp; ta.M = M; ta.N = N;
  ta.r2 = r > 0 ? (float)(r * r) : 0.f;
  ta.t2 = t > 0 ? (float)(t * t) : 0.f;
  ta.mutual = cfg->mutual_check != 0;
  TcNnGate gate{};
  if (guided) {
    gate.fundamental = guide->kind == NN_GUIDE_F;
    gate.rec = w.rec; gate.on = w.gate_on;
    gate.t2 = (float)(guide->max_error * guide->max_error);
  }
  for (int b0 = 0; b0 < B; b0 += w.G) {
    const int g = B - b0 < w.G ? B - b0 : w.G;
    PackArgs pa{in->desc0, in->desc1, in->lens0, in->lens1, b0, g, M, N, D, w.Lp, w.hi, w.lo, w.len, w.stop};
    const long groups4 = 2L * g * w.Lp * (D / 4);
    const long blocks = (groups4 + 255) / 256;
    nn_pack_kernel<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256, 0, stream>>>(pa);
    LG_CHECK_LAUNCH();
    if (guided) {
      const GateArgs ga{guide->model, guide->valid, guide->kpts0, guide->kpts1, b0, g, M, N, w.Lp, gate.fundamental,
                        w.rec, w.gate_on};
      nn_gate_record_kernel<<<(unsigned)((2L * g * w.Lp + 255) / 256), 256, 0, stream>>>(ga);
      LG_CHECK_LAUNCH();
    }
    const SeqState st{2 * g, g, w.Lp, w.len, w.stop};
    LG_RC(tc_nn_sweep(h->tc, st, w.hi, w.lo, D, w.part, w.parg, w.pstride, stream, guided ? &gate : nullptr));
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

extern "C" int nn_match(NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnOutputs* out, void* workspace,
                        size_t workspace_bytes, void* stream) {
  return nn_run("nn_match", h, cfg, in, nullptr, out, workspace, workspace_bytes, stream);
}

extern "C" int nn_match_guided(NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnGuide* guide,
                               const NnOutputs* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!guide) return nn_error("nn_match_guided", "null argument");
  return nn_run("nn_match_guided", h, cfg, in, guide, out, workspace, workspace_bytes, stream);
}
