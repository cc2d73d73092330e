// SuperPoint extractor forward (SURVEY.md 8f1; reference lightglue/superpoint.py:163-227).
//
// Every stage is a small functor with `operator()(long i)` = the work of ONE logical thread, and the whole forward
// is one template `sp_run(Exec&, ...)` that hands those functors to an executor.  The CUDA build (sp_api.cu)
// executes them with a generic grid-stride-free kernel (one thread per index); the test-only build under oracle/
// (sp_emul.cpp, plain g++) executes THE SAME functors and THE SAME orchestration in a host loop, which is how the
// kernel logic is checked against the reference-generated fixtures on a machine without a GPU.  There is no
// shared memory, no warp intrinsic and no atomics in this path: it is the fp32 (CUDA-core) forward and the
// correctness baseline for the extractor.  precision "bf16x3" replaces the convolutions with the tensor-core backbone
// (sp_tc.cu) and the heavy post-processing stages with warp / block kernels (SpCudaStages); the rest runs from here.
//
// Layouts: feature maps NCHW fp32, weights as in the reference state_dict ([Cout, Cin, k, k] row-major).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "ws_bump.h"

#if defined(__CUDACC__)
#define SP_HD __host__ __device__ __forceinline__
#else
#define SP_HD inline
#endif

#define SP_CELL 8        // three 2x2 poolings
#define SP_DESC 256
#define SP_CO_T 8        // output channels per logical thread in SpConv
#define SP_PX_T 4        // consecutive pixels (along x) per logical thread in SpConv

struct SpConv {  // k x k convolution (k = 1 or 3, stride 1, zero padding k/2) + bias (+ ReLU)   (superpoint.py:137-153)
  const float* in; const float* w; const float* bias; float* out;
  int B, Cin, Cout, H, W, k, relu;
  SP_HD long count() const { return (long)B * ((Cout + SP_CO_T - 1) / SP_CO_T) * H * ((W + SP_PX_T - 1) / SP_PX_T); }
  SP_HD void operator()(long i) const {
    const int wt = (W + SP_PX_T - 1) / SP_PX_T, cg = (Cout + SP_CO_T - 1) / SP_CO_T;
    const int xt = (int)(i % wt); long r = i / wt;
    const int y = (int)(r % H); r /= H;
    const int g = (int)(r % cg); const int b = (int)(r / cg);
    const int x0 = xt * SP_PX_T, co0 = g * SP_CO_T, pad = k / 2;
    float acc[SP_CO_T][SP_PX_T];
    for (int c = 0; c < SP_CO_T; ++c)
      for (int p = 0; p < SP_PX_T; ++p) acc[c][p] = (co0 + c < Cout) ? bias[co0 + c] : 0.f;
    const float* inb = in + (long)b * Cin * H * W;
    for (int ci = 0; ci < Cin; ++ci) {
      const float* plane = inb + (long)ci * H * W;
      for (int ky = 0; ky < k; ++ky) {
        const int yy = y + ky - pad;
        if (yy < 0 || yy >= H) continue;
        float v[SP_PX_T + 2];
        for (int t = 0; t < SP_PX_T + k - 1; ++t) {
          const int xx = x0 + t - pad;
          v[t] = (xx >= 0 && xx < W) ? plane[(long)yy * W + xx] : 0.f;
        }
        for (int c = 0; c < SP_CO_T; ++c) {
          if (co0 + c >= Cout) break;
          const float* wr = w + (((long)(co0 + c) * Cin + ci) * k + ky) * k;
          for (int kx = 0; kx < k; ++kx) {
            const float wv = wr[kx];
            for (int p = 0; p < SP_PX_T; ++p) acc[c][p] = fmaf(v[p + kx], wv, acc[c][p]);
          }
        }
      }
    }
    for (int c = 0; c < SP_CO_T && co0 + c < Cout; ++c)
      for (int p = 0; p < SP_PX_T && x0 + p < W; ++p) {
        const float a = acc[c][p];
        out[(((long)b * Cout + co0 + c) * H + y) * W + x0 + p] = (relu && a < 0.f) ? 0.f : a;
      }
  }
};

struct SpPool2 {  // 2x2 max pooling, stride 2   (superpoint.py:135)
  const float* in; float* out; int BC, H, W;  // input H x W (even), output H/2 x W/2
  SP_HD long count() const { return (long)BC * (H / 2) * (W / 2); }
  SP_HD void operator()(long i) const {
    const int wo = W / 2, ho = H / 2;
    const int x = (int)(i % wo); long r = i / wo;
    const int y = (int)(r % ho); const long bc = r / ho;
    const float* p = in + (bc * H + 2 * y) * W + 2 * x;
    out[i] = fmaxf(fmaxf(p[0], p[1]), fmaxf(p[W], p[W + 1]));
  }
};

struct SpScores {  // 65-way soft-max per cell, dustbin dropped, 64 channels -> the 8x8 pixels of the cell   (186-190)
  const float* logits; float* scores; int B, Hc, Wc;  // logits [B,65,Hc,Wc] -> scores [B, Hc*8, Wc*8]
  SP_HD long count() const { return (long)B * Hc * Wc; }
  SP_HD void operator()(long i) const {
    const int xc = (int)(i % Wc); long r = i / Wc;
    const int yc = (int)(r % Hc); const int b = (int)(r / Hc);
    const long plane = (long)Hc * Wc;
    const float* l = logits + (long)b * 65 * plane + (long)yc * Wc + xc;
    float m = l[0];
    for (int c = 1; c < 65; ++c) m = fmaxf(m, l[c * plane]);
    float e[65], sum = 0.f;
    for (int c = 0; c < 65; ++c) { e[c] = expf(l[c * plane] - m); sum += e[c]; }
    const int W = Wc * SP_CELL;
    float* o = scores + ((long)b * Hc * SP_CELL + (long)yc * SP_CELL) * W + (long)xc * SP_CELL;
    for (int c = 0; c < 64; ++c) o[(long)(c / SP_CELL) * W + (c % SP_CELL)] = e[c] / sum;
  }
};

// window maximum of radius r along x (dir = 0) or y (dir = 1), out-of-image = -inf: two passes = max_pool2d(2r+1, 1, r)
struct SpWindowMax {
  const float* in; float* out; int B, H, W, r, dir;
  SP_HD long count() const { return (long)B * H * W; }
  SP_HD void operator()(long i) const {
    const int x = (int)(i % W); long q = i / W;
    const int y = (int)(q % H);
    const float* base = in + (q / H) * (long)H * W;
    float m = -INFINITY;
    if (dir == 0) {
      const int lo = x - r < 0 ? 0 : x - r, hi = x + r >= W ? W - 1 : x + r;
      for (int t = lo; t <= hi; ++t) m = fmaxf(m, base[(long)y * W + t]);
    } else {
      const int lo = y - r < 0 ? 0 : y - r, hi = y + r >= H ? H - 1 : y + r;
      for (int t = lo; t <= hi; ++t) m = fmaxf(m, base[(long)t * W + x]);
    }
    out[i] = m;
  }
};

// elementwise steps of simple_nms (52-68); `mode` selects the line being evaluated
struct SpNmsStep {
  const float* scores; const float* a; const float* b; float* out; long n; int mode;
  SP_HD long count() const { return n; }
  SP_HD void operator()(long i) const {
    switch (mode) {
      case 0: out[i] = scores[i] == a[i] ? 1.f : 0.f; break;                        // max_mask = scores == max_pool(scores)
      case 1: out[i] = a[i] > 0.f ? 0.f : scores[i]; break;                          // supp_scores = where(supp, 0, scores); a = max_pool(max_mask)
      case 2: {                                                                      // max_mask |= (supp_scores == max_pool(supp_scores)) & ~supp
        // scores = supp_scores, a = max_pool(supp_scores), b = max_pool(max_mask) (> 0 == suppressed); out = max_mask (in place)
        const bool nm = scores[i] == a[i] && !(b[i] > 0.f);
        if (nm) out[i] = 1.f;
        break;
      }
      default: out[i] = a[i] > 0.f ? scores[i] : 0.f; break;                         // where(max_mask, scores, 0); a = max_mask
    }
  }
};

struct SpBorders {  // scores near the border := -1   (193-198)
  float* scores; int B, H, W, pad;
  SP_HD long count() const { return (long)B * H * W; }
  SP_HD void operator()(long i) const {
    const int x = (int)(i % W), y = (int)((i / W) % H);
    if (x < pad || y < pad || x >= W - pad || y >= H - pad) scores[i] = -1.f;
  }
};

// candidates = where(scores > threshold), row-major per image (201-208): count per row, scan per image, write per row
struct SpRowCount {
  const float* scores; int* row_count; int B, H, W; float thr;
  SP_HD long count() const { return (long)B * H; }
  SP_HD void operator()(long i) const {
    const float* p = scores + i * W;
    int c = 0;
    for (int x = 0; x < W; ++x) c += p[x] > thr ? 1 : 0;
    row_count[i] = c;
  }
};
struct SpRowScan {
  const int* row_count; int* row_start; int* n_cand; int B, H;
  SP_HD long count() const { return B; }
  SP_HD void operator()(long b) const {
    int acc = 0;
    for (int y = 0; y < H; ++y) { row_start[b * H + y] = acc; acc += row_count[b * H + y]; }
    n_cand[b] = acc;
  }
};
struct SpRowWrite {
  const float* scores; const int* row_start; int* cand_pos; float* cand_score; int B, H, W; float thr; long cap;
  SP_HD long count() const { return (long)B * H; }
  SP_HD void operator()(long i) const {
    const long b = i / H; const int y = (int)(i % H);
    const float* p = scores + i * W;
    long o = b * cap + row_start[i];
    for (int x = 0; x < W; ++x)
      if (p[x] > thr) { cand_pos[o] = y * W + x; cand_score[o] = p[x]; ++o; }
  }
};

// top-k by score, sorted descending (71-76); ties: lower candidate index first.  Rank by counting: no sort network,
// no synchronisation.  If an image has <= k candidates they keep their row-major order (the reference returns early),
// unless rank_all is set (ALIKED's top-k mode sorts whatever it keeps).
struct SpSelect {
  const int* n_cand; const int* cand_pos; const float* cand_score; int* sel_pos; float* sel_score; int* n_sel;
  int B, k; long cap, out_cap;  // k <= 0: no limit
  int rank_all;                 // with k > 0: rank the candidates even when there are no more than k
  SP_HD long count() const { return (long)B * cap; }
  SP_HD void operator()(long i) const {
    const long b = i / cap, j = i % cap;
    const int n = n_cand[b];
    if (j == 0) n_sel[b] = (k > 0 && n > k) ? k : (n < out_cap ? n : (int)out_cap);
    if (j >= n) return;
    const float* s = cand_score + b * cap;
    long rank = j;
    if (k > 0 && (n > k || rank_all)) {
      const float me = s[j];
      rank = 0;
      for (int t = 0; t < n; ++t) rank += (s[t] > me || (s[t] == me && t < j)) ? 1 : 0;
      if (rank >= k) return;
    }
    if (rank >= out_cap) return;
    sel_pos[b * out_cap + rank] = cand_pos[b * cap + j];
    sel_score[b * out_cap + rank] = s[j];
  }
};

// simple_nms keeps every pixel of a plateau, so without top-k an image can have more candidates than the NMS packing
// bound (sp_keypoint_cap) that sizes the outputs.  Its count becomes -1 and its rows stay zero: no silent cut.
struct SpOverflow {
  const int* n_cand; int* n_sel; int B; long out_cap;
  SP_HD long count() const { return B; }
  SP_HD void operator()(long b) const { if (n_cand[b] > out_cap) n_sel[b] = -1; }
};

struct SpNormalizeDense {  // F.normalize(descriptors, p=2, dim=1) on the coarse map (222), in place
  float* d; int B, Hc, Wc;
  SP_HD long count() const { return (long)B * Hc * Wc; }
  SP_HD void operator()(long i) const {
    const long plane = (long)Hc * Wc;
    float* p = d + (i / plane) * SP_DESC * plane + (i % plane);
    float ss = 0.f;
    for (int c = 0; c < SP_DESC; ++c) ss = fmaf(p[c * plane], p[c * plane], ss);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    for (int c = 0; c < SP_DESC; ++c) p[c * plane] *= inv;
  }
};

// keypoints (x, y), scores and bilinearly sampled + normalised descriptors (79-96, 217-226); one logical thread per keypoint
struct SpSample {
  const int* n_sel; const int* sel_pos; const float* sel_score; const float* dense;  // dense [B,256,Hc,Wc], normalised
  float* kpts; float* kscores; float* desc; int B, Hc, Wc; long out_cap;
  SP_HD long count() const { return (long)B * out_cap; }
  SP_HD void operator()(long i) const {
    const long b = i / out_cap, j = i % out_cap;
    float* dd = desc + i * SP_DESC;
    if (j >= n_sel[b]) {  // padding slots: zeros
      kpts[i * 2] = 0.f; kpts[i * 2 + 1] = 0.f; kscores[i] = 0.f;
      for (int c = 0; c < SP_DESC; ++c) dd[c] = 0.f;
      return;
    }
    const int W = Wc * SP_CELL;
    const int pos = sel_pos[i];
    const float x = (float)(pos % W), y = (float)(pos / W);
    kpts[i * 2] = x; kpts[i * 2 + 1] = y; kscores[i] = sel_score[i];
    // sample_descriptors: k = (kp - s/2 + 0.5) / (w*s - s/2 - 0.5) in [0,1] -> grid in [-1,1] -> align_corners=True pixel
    const float s = (float)SP_CELL;
    const float gx = (x - s / 2 + 0.5f) / ((float)Wc * s - s / 2 - 0.5f) * 2.f - 1.f;
    const float gy = (y - s / 2 + 0.5f) / ((float)Hc * s - s / 2 - 0.5f) * 2.f - 1.f;
    const float px = (gx + 1.f) * 0.5f * (float)(Wc - 1), py = (gy + 1.f) * 0.5f * (float)(Hc - 1);
    const float fx = floorf(px), fy = floorf(py);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float ax = px - fx, ay = py - fy;
    const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
    const bool v00 = x0 >= 0 && x0 < Wc && y0 >= 0 && y0 < Hc, v01 = x1 >= 0 && x1 < Wc && y0 >= 0 && y0 < Hc;
    const bool v10 = x0 >= 0 && x0 < Wc && y1 >= 0 && y1 < Hc, v11 = x1 >= 0 && x1 < Wc && y1 >= 0 && y1 < Hc;
    const long plane = (long)Hc * Wc;
    const float* base = dense + b * SP_DESC * plane;
    float ss = 0.f;
    for (int c = 0; c < SP_DESC; ++c) {
      const float* p = base + c * plane;
      float v = 0.f;
      if (v00) v += p[(long)y0 * Wc + x0] * w00;
      if (v01) v += p[(long)y0 * Wc + x1] * w01;
      if (v10) v += p[(long)y1 * Wc + x0] * w10;
      if (v11) v += p[(long)y1 * Wc + x1] * w11;
      dd[c] = v;
      ss = fmaf(v, v, ss);
    }
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    for (int c = 0; c < SP_DESC; ++c) dd[c] *= inv;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// weights: the reference state_dict tensors, fp32, concatenated in this order (superpoint.py:137-153)
// ---------------------------------------------------------------------------------------------------------------
struct SpLayer { int cout, cin, k; };
static const SpLayer SP_LAYERS[12] = {
    {64, 1, 3},    {64, 64, 3},   {64, 64, 3},   {64, 64, 3},    // conv1a conv1b conv2a conv2b
    {128, 64, 3},  {128, 128, 3}, {128, 128, 3}, {128, 128, 3},  // conv3a conv3b conv4a conv4b
    {256, 128, 3}, {65, 256, 1},  {256, 128, 3}, {256, 256, 1},  // convPa convPb convDa convDb
};
inline size_t sp_layer_floats(int l) { return (size_t)SP_LAYERS[l].cout * SP_LAYERS[l].cin * SP_LAYERS[l].k * SP_LAYERS[l].k + SP_LAYERS[l].cout; }
inline size_t sp_blob_floats() { size_t n = 0; for (int l = 0; l < 12; ++l) n += sp_layer_floats(l); return n; }
inline size_t sp_layer_offset(int l) { size_t n = 0; for (int i = 0; i < l; ++i) n += sp_layer_floats(i); return n; }

struct SpParams { int nms_radius, max_num_keypoints, remove_borders; float detection_threshold; };

// workspace carve (floats / ints); `base` may be null to size it
struct SpWorkspace {
  float *bufA, *bufB, *logits, *scores, *t0, *t1, *t2, *mask, *dense, *cand_score, *sel_score;
  int *row_count, *row_start, *n_cand, *cand_pos, *sel_pos, *n_sel;
  size_t bytes;
};
inline void sp_carve(char* base, int B, int H, int W, long out_cap, SpWorkspace* w) {
  WsBump b{base, 0};
  const size_t px = (size_t)B * H * W, Hc = H / SP_CELL, Wc = W / SP_CELL;
  w->bufA = b.take<float>(px * 64);
  w->bufB = b.take<float>(px * 64);
  w->logits = b.take<float>((size_t)B * 65 * Hc * Wc);
  w->scores = b.take<float>(px);
  w->t0 = b.take<float>(px);
  w->t1 = b.take<float>(px);
  w->t2 = b.take<float>(px);
  w->mask = b.take<float>(px);
  w->dense = b.take<float>((size_t)B * SP_DESC * Hc * Wc);
  w->cand_score = b.take<float>(px);
  w->sel_score = b.take<float>((size_t)B * out_cap);
  w->row_count = b.take<int>((size_t)B * H);
  w->row_start = b.take<int>((size_t)B * H);
  w->n_cand = b.take<int>(B);
  w->cand_pos = b.take<int>(px);
  w->sel_pos = b.take<int>((size_t)B * out_cap);
  w->n_sel = b.take<int>(B);
  w->bytes = b.bytes();
}

// Keypoints per image at most (sp_max_keypoints): max_num_keypoints, or else the most NMS survivors the image can hold
inline int64_t sp_keypoint_cap(int nms_radius, int max_num_keypoints, int H, int W) {
  if (max_num_keypoints > 0) return max_num_keypoints;
  const int step = nms_radius + 1;  // no two NMS survivors lie within `nms_radius` of each other (Chebyshev)
  return (int64_t)((H + step - 1) / step) * ((W + step - 1) / step);
}

// simple_nms (52-68) of `scores` [B,H,W] into `out` (which may be `tmp`): window maxima of radius r along x then y
// (`line` holds the x pass), and the elementwise steps.  `tmp`, `mask`, `supp` and `pooled` are [B,H,W] scratch.
template <class Exec>
int sp_simple_nms(Exec& exec, const float* scores, float* out, int B, int H, int W, int r, float* tmp, float* mask,
                  float* supp, float* pooled, float* line) {
  const long n = (long)B * H * W;
  auto wmax = [&](const float* in, float* o) {
    SpWindowMax a{in, line, B, H, W, r, 0};
    int e = exec.run(a);
    if (e) return e;
    SpWindowMax b{line, o, B, H, W, r, 1};
    return exec.run(b);
  };
  int rc;
  if ((rc = wmax(scores, tmp))) return rc;
  { SpNmsStep s{scores, tmp, nullptr, mask, n, 0}; if ((rc = exec.run(s))) return rc; }
  for (int it = 0; it < 2; ++it) {
    if ((rc = wmax(mask, tmp))) return rc;                                                     // tmp = max_pool(max_mask)
    { SpNmsStep s{scores, tmp, nullptr, supp, n, 1}; if ((rc = exec.run(s))) return rc; }     // supp = supp_scores
    if ((rc = wmax(supp, pooled))) return rc;                                                  // pooled = max_pool(supp)
    { SpNmsStep s{supp, pooled, tmp, mask, n, 2}; if ((rc = exec.run(s))) return rc; }
  }
  { SpNmsStep s{scores, mask, nullptr, out, n, 3}; if ((rc = exec.run(s))) return rc; }       // nms scores
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// the forward: SuperPoint.forward (163-227) on a grayscale batch [B,1,H,W], H, W >= 8 (any size: the three poolings floor,
// 173-179, so the heads see Hc = H / 8, Wc = W / 8 cells and the score map covers the top-left 8 Hc x 8 Wc pixels, 188-190;
// the rows / columns beyond it still feed the first convolutions' 3x3 neighbourhoods, as in the reference).
// `exec.run(f)` executes functor f for every index in [0, f.count()); returns non-zero on failure.
// Outputs: kpts [B,out_cap,2] (x, y), kscores [B,out_cap], desc [B,out_cap,256], counts = ws.n_sel [B].
// ---------------------------------------------------------------------------------------------------------------
// Part 1: the convolution stack -> ws.logits [B,65,Hc,Wc], ws.dense [B,256,Hc,Wc] (un-normalised), fp32 NCHW.
template <class Exec>
int sp_run_backbone(Exec& exec, const float* wts, const float* image, int B, int H, int W, const SpWorkspace& ws) {
  auto conv = [&](int l, const float* in, float* out, int h, int w_, int relu) {
    const float* base = wts + sp_layer_offset(l);
    const SpLayer& L = SP_LAYERS[l];
    SpConv c{in, base, base + (size_t)L.cout * L.cin * L.k * L.k, out, B, L.cin, L.cout, h, w_, L.k, relu};
    return exec.run(c);
  };
  auto pool = [&](const float* in, float* out, int C, int h, int w_) { SpPool2 p{in, out, B * C, h, w_}; return exec.run(p); };
  int rc = 0;
  // shared encoder (171-181)
  if ((rc = conv(0, image, ws.bufA, H, W, 1))) return rc;
  if ((rc = conv(1, ws.bufA, ws.bufB, H, W, 1))) return rc;
  if ((rc = pool(ws.bufB, ws.bufA, 64, H, W))) return rc;
  int h = H / 2, w_ = W / 2;
  if ((rc = conv(2, ws.bufA, ws.bufB, h, w_, 1))) return rc;
  if ((rc = conv(3, ws.bufB, ws.bufA, h, w_, 1))) return rc;
  if ((rc = pool(ws.bufA, ws.bufB, 64, h, w_))) return rc;
  h /= 2; w_ /= 2;
  if ((rc = conv(4, ws.bufB, ws.bufA, h, w_, 1))) return rc;
  if ((rc = conv(5, ws.bufA, ws.bufB, h, w_, 1))) return rc;
  if ((rc = pool(ws.bufB, ws.bufA, 128, h, w_))) return rc;
  h /= 2; w_ /= 2;  // = Hc, Wc
  if ((rc = conv(6, ws.bufA, ws.bufB, h, w_, 1))) return rc;
  if ((rc = conv(7, ws.bufB, ws.bufA, h, w_, 1))) return rc;  // feat = bufA [B,128,Hc,Wc]
  // detector head (184-185)
  if ((rc = conv(8, ws.bufA, ws.bufB, h, w_, 1))) return rc;
  if ((rc = conv(9, ws.bufB, ws.logits, h, w_, 0))) return rc;
  // descriptor head (220-221)
  if ((rc = conv(10, ws.bufA, ws.bufB, h, w_, 1))) return rc;
  if ((rc = conv(11, ws.bufB, ws.dense, h, w_, 0))) return rc;
  return 0;
}

// The three heavy post-processing stages as one-logical-thread functors (the semantic definition, also run on the host by
// oracle/sp_emul.cpp).  The CUDA build substitutes warp / block kernels with the same results (sp_tc.cu SpCudaStages).
struct SpFunctorStages {
  // candidates = where(scores > threshold), row-major per image (201-208)
  template <class Exec>
  int compact(Exec& exec, const SpWorkspace& ws, int B, int H, int W, float thr, long cap) const {
    int rc;
    { SpRowCount s{ws.t0, ws.row_count, B, H, W, thr}; if ((rc = exec.run(s))) return rc; }
    { SpRowScan s{ws.row_count, ws.row_start, ws.n_cand, B, H}; if ((rc = exec.run(s))) return rc; }
    { SpRowWrite s{ws.t0, ws.row_start, ws.cand_pos, ws.cand_score, B, H, W, thr, cap}; if ((rc = exec.run(s))) return rc; }
    return 0;
  }
  // top-k by score, descending, ties by candidate index (71-76, 210-218)
  template <class Exec>
  int select(Exec& exec, const SpWorkspace& ws, int B, int k, long cap, long out_cap, int rank_all = 0) const {
    SpSelect s{ws.n_cand, ws.cand_pos, ws.cand_score, ws.sel_pos, ws.sel_score, ws.n_sel, B, k, cap, out_cap, rank_all};
    return exec.run(s);
  }
  // keypoints, scores, bilinearly sampled + normalised descriptors (79-96, 217-226)
  template <class Exec>
  int sample(Exec& exec, const SpWorkspace& ws, float* kpts, float* kscores, float* desc, int B, int Hc, int Wc, long out_cap) const {
    SpSample s{ws.n_sel, ws.sel_pos, ws.sel_score, ws.dense, kpts, kscores, desc, B, Hc, Wc, out_cap};
    return exec.run(s);
  }
};

// Part 2: scores, NMS, keypoint selection, descriptor normalisation + sampling on ws.logits / ws.dense.
// H, W here are the SCORE MAP's extents (8 Hc, 8 Wc): the image's own, rounded down to multiples of 8.
template <class Exec, class Stages = SpFunctorStages>
int sp_run_post(Exec& exec, const SpParams& prm, int B, int H, int W, long out_cap, const SpWorkspace& ws, float* kpts,
                float* kscores, float* desc, const Stages& stages = Stages()) {
  int rc = 0;
  const int Hc = H / SP_CELL, Wc = W / SP_CELL;
  // detector scores (186-190)
  { SpScores s{ws.logits, ws.scores, B, Hc, Wc}; if ((rc = exec.run(s))) return rc; }
  // simple_nms (52-68) -> t0; cand_score is scratch until the compaction
  if ((rc = sp_simple_nms(exec, ws.scores, ws.t0, B, H, W, prm.nms_radius, ws.t0, ws.mask, ws.t1, ws.cand_score, ws.t2)))
    return rc;
  if (prm.remove_borders > 0) { SpBorders s{ws.t0, B, H, W, prm.remove_borders}; if ((rc = exec.run(s))) return rc; }
  // keypoints (201-218)
  const long cap = (long)H * W;
  if ((rc = stages.compact(exec, ws, B, H, W, prm.detection_threshold, cap))) return rc;
  if ((rc = stages.select(exec, ws, B, prm.max_num_keypoints, cap, out_cap))) return rc;
  if (prm.max_num_keypoints <= 0) { SpOverflow s{ws.n_cand, ws.n_sel, B, out_cap}; if ((rc = exec.run(s))) return rc; }
  // descriptors (222-226)
  { SpNormalizeDense s{ws.dense, B, Hc, Wc}; if ((rc = exec.run(s))) return rc; }
  if ((rc = stages.sample(exec, ws, kpts, kscores, desc, B, Hc, Wc, out_cap))) return rc;
  return 0;
}

template <class Exec>
int sp_run(Exec& exec, const float* wts, const SpParams& prm, const float* image, int B, int H, int W, long out_cap,
           const SpWorkspace& ws, float* kpts, float* kscores, float* desc) {
  int rc = sp_run_backbone(exec, wts, image, B, H, W, ws);
  if (rc) return rc;
  return sp_run_post(exec, prm, B, H / SP_CELL * SP_CELL, W / SP_CELL * SP_CELL, out_cap, ws, kpts, kscores, desc);
}
