// C ABI of the SuperPoint extractor (include/superpoint_b200.h): executes the functors of sp_pipeline.h on the GPU,
// one thread per logical index.  The same functors and orchestration run on the host in oracle/sp_emul.cpp (tests).
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/superpoint_b200.h"
#include "lg_internal.h"
#include "sp_pipeline.h"
#include "sp_tc.h"

struct SpHandle {
  SpConfig cfg;
  float* wts;  // device copy of the weight blob
  TcConvWeights* tc;  // tensor-core backbone (cfg.precision == 1), else null
};

namespace {
// The convolution stack of this handle's precision -> logits [B,65,Hc,Wc], dense [B,256,Hc,Wc] (fp32 NCHW); `w` is the
// carve of `workspace`, whose tensor-core part follows the functor buffers
int run_backbone(SpHandle* h, SpCudaExec& ex, const float* image, int B, int H, int W, SpWorkspace w, char* workspace,
                 float* logits, float* dense) {
  if (h->tc) return sp_tc_backbone(h->tc, h->wts, image, B, H, W, workspace + w.bytes, logits, dense, ex.stream);
  w.logits = logits;
  w.dense = dense;
  return sp_run_backbone(ex, h->wts, image, B, H, W, w);
}

// The post-processing of w.logits / w.dense (scores, NMS, keypoints, descriptors) for an H x W image, and the counts
int run_post(SpHandle* h, SpCudaExec& ex, int B, int H, int W, long cap, const SpWorkspace& w, float* keypoints, float* scores,
             float* descriptors, int32_t* counts) {
  const SpParams prm{h->cfg.nms_radius, h->cfg.max_num_keypoints, h->cfg.remove_borders, h->cfg.detection_threshold};
  const int Hs = H / SP_CELL * SP_CELL, Ws = W / SP_CELL * SP_CELL;  // the score map's extents
  // the tensor-core mode also runs the post-processing's heavy stages as warp / block kernels (same results)
  LG_RC(h->tc ? sp_run_post(ex, prm, B, Hs, Ws, cap, w, keypoints, scores, descriptors, SpCudaStages{ex.stream})
              : sp_run_post(ex, prm, B, Hs, Ws, cap, w, keypoints, scores, descriptors));
  LG_CU(cudaMemcpyAsync(counts, w.n_sel, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, ex.stream));
  return 0;
}

// Workspace bytes for a [B, 1, H, W] batch and `cap` output rows per image: the functor buffers, then the tensor-core part
size_t workspace_need(bool tc, int B, int H, int W, long cap, SpWorkspace* w) {
  sp_carve(nullptr, B, H, W, cap, w);
  return w->bytes + (tc ? sp_tc_plan(B, H, W).total : 0);
}

// The argument checks sp_forward and sp_post share; on success `w` is the carve of `workspace`
int check_call(const char* what, const SpHandle* h, int B, int H, int W, long cap, void* workspace, size_t workspace_bytes,
               SpWorkspace* w) {
  char msg[128];
  auto fail = [&](const char* why) {
    snprintf(msg, sizeof msg, "%s: %s", what, why);
    return lg_set_error(msg);
  };
  if (B <= 0 || H < SP_CELL || W < SP_CELL) return fail("H and W must be at least 8");
  if (cap < sp_keypoint_cap(h->cfg.nms_radius, h->cfg.max_num_keypoints, H, W))
    return fail("output capacity below sp_max_keypoints()");
  if (!workspace || workspace_bytes < workspace_need(h->tc, B, H, W, cap, w)) return fail("workspace too small");
  sp_carve((char*)workspace, B, H, W, cap, w);
  return 0;
}
}  // namespace

extern "C" size_t sp_weight_blob_floats(void) { return sp_blob_floats(); }

extern "C" int sp_create(const SpConfig* cfg, const float* weights_dev, size_t n_floats, void* stream_, SpHandle** out) {
  if (!cfg || !weights_dev || !out) return lg_set_error("sp_create: null argument");
  if (cfg->abi_version != SP_ABI_VERSION) return lg_set_error("sp_create: ABI version mismatch");
  if (n_floats != sp_blob_floats()) return lg_set_error("sp_create: weight blob has the wrong size");
  if (cfg->nms_radius < 0 || cfg->remove_borders < 0) return lg_set_error("sp_create: bad conf");
  if (cfg->precision != 0 && cfg->precision != 1) return lg_set_error("sp_create: bad precision");
  SpHandle* h = new SpHandle{*cfg, nullptr, nullptr};
  struct Guard {  // every failure path below releases the handle and what it owns
    SpHandle* h;
    ~Guard() { if (h) sp_destroy(h); }
  } guard{h};
  LG_CU(cudaMalloc(&h->wts, n_floats * sizeof(float)));
  LG_CU(cudaMemcpyAsync(h->wts, weights_dev, n_floats * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  if (cfg->precision == 1) LG_RC(sp_tc_create(&h->tc, h->wts, (cudaStream_t)stream_));
  guard.h = nullptr;
  *out = h;
  return 0;
}

extern "C" int sp_destroy(SpHandle* h) {
  if (!h) return 0;
  tc_conv_weights_destroy(h->tc);
  cudaFree(h->wts);
  delete h;
  return 0;
}

extern "C" int64_t sp_max_keypoints(const SpHandle* h, int32_t H, int32_t W) {
  return h ? sp_keypoint_cap(h->cfg.nms_radius, h->cfg.max_num_keypoints, H, W) : 0;
}

extern "C" size_t sp_workspace_bytes(const SpHandle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  SpWorkspace w;
  return workspace_need(h->tc, B, H, W, sp_max_keypoints(h, H, W), &w);
}

extern "C" int64_t sp_workspace_layout(const SpConfig* cfg, int32_t B, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes) {
  if (!cfg || (cfg->precision != 0 && cfg->precision != 1) || cfg->nms_radius < 0 || B <= 0 || H < SP_CELL || W < SP_CELL)
    return 0;
  const long cap = sp_keypoint_cap(cfg->nms_radius, cfg->max_num_keypoints, H, W);
  SpWorkspace w;
  const size_t total = workspace_need(cfg->precision == 1, B, H, W, cap, &w);
  char* const base = reinterpret_cast<char*>(kLayoutBase);
  sp_carve(base, B, H, W, cap, &w);
  const size_t px = (size_t)B * H * W, cells = (size_t)B * (H / SP_CELL) * (W / SP_CELL), f = sizeof(float), i = sizeof(int);
  const struct { const void* p; size_t n; } buf[SP_LAYOUT_BUFFERS] = {
      {w.logits, 65 * cells * f}, {w.scores, px * f},         {w.t0, px * f},
      {w.mask, px * f},           {w.dense, SP_DESC * cells * f}, {w.row_count, (size_t)B * H * i},
      {w.row_start, (size_t)B * H * i}, {w.n_cand, (size_t)B * i}, {w.cand_pos, px * i},
      {w.cand_score, px * f},     {w.sel_pos, (size_t)B * cap * i}, {w.sel_score, (size_t)B * cap * f},
      {w.n_sel, (size_t)B * i}};
  for (int k = 0; k < SP_LAYOUT_BUFFERS; ++k) {
    if (offsets) offsets[k] = (int64_t)((const char*)buf[k].p - base);
    if (bytes) bytes[k] = (int64_t)buf[k].n;
  }
  return (int64_t)total;
}

extern "C" int64_t sp_tc_layout(int32_t B, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes) {
  static_assert(SPT_NBUF == SP_TC_BUFFERS, "superpoint_b200.h documents the buffers of SpTcPlan");
  if (B <= 0 || H < SP_CELL || W < SP_CELL) return 0;
  const SpTcPlan p = sp_tc_plan(B, H, W);
  for (int i = 0; i < SPT_NBUF; ++i) {
    if (offsets) offsets[i] = (int64_t)p.off[i];
    if (bytes) bytes[i] = (int64_t)p.bytes[i];
  }
  return (int64_t)p.total;
}

extern "C" int sp_forward(SpHandle* h, const float* image, int32_t B, int32_t H, int32_t W, int64_t cap, float* keypoints,
                          float* scores, float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes,
                          void* stream_) {
  if (!h || !image || !keypoints || !scores || !descriptors || !counts) return lg_set_error("sp_forward: null argument");
  SpWorkspace w;
  LG_RC(check_call("sp_forward", h, B, H, W, cap, workspace, workspace_bytes, &w));
  SpCudaExec ex{(cudaStream_t)stream_};
  LG_RC(run_backbone(h, ex, image, B, H, W, w, (char*)workspace, w.logits, w.dense));
  return run_post(h, ex, B, H, W, cap, w, keypoints, scores, descriptors, counts);
}

extern "C" int sp_post(SpHandle* h, const float* logits, const float* dense, int32_t B, int32_t H, int32_t W, int64_t cap,
                       float* keypoints, float* scores, float* descriptors, int32_t* counts, void* workspace,
                       size_t workspace_bytes, void* stream_) {
  if (!h || !logits || !dense || !keypoints || !scores || !descriptors || !counts) return lg_set_error("sp_post: null argument");
  SpWorkspace w;
  LG_RC(check_call("sp_post", h, B, H, W, cap, workspace, workspace_bytes, &w));
  SpCudaExec ex{(cudaStream_t)stream_};
  const size_t cells = (size_t)B * (H / SP_CELL) * (W / SP_CELL);
  LG_CU(cudaMemcpyAsync(w.logits, logits, 65 * cells * sizeof(float), cudaMemcpyDeviceToDevice, ex.stream));
  LG_CU(cudaMemcpyAsync(w.dense, dense, SP_DESC * cells * sizeof(float), cudaMemcpyDeviceToDevice, ex.stream));
  return run_post(h, ex, B, H, W, cap, w, keypoints, scores, descriptors, counts);
}

extern "C" int sp_backbone(SpHandle* h, const float* image, int32_t B, int32_t H, int32_t W, float* logits, float* dense,
                           void* workspace, size_t workspace_bytes, void* stream_) {
  if (!h || !image || !logits || !dense) return lg_set_error("sp_backbone: null argument");
  if (B <= 0 || H < SP_CELL || W < SP_CELL) return lg_set_error("sp_backbone: H and W must be at least 8");
  if (!workspace || workspace_bytes < sp_workspace_bytes(h, B, H, W)) return lg_set_error("sp_backbone: workspace too small");
  SpWorkspace w;
  sp_carve((char*)workspace, B, H, W, sp_max_keypoints(h, H, W), &w);
  SpCudaExec ex{(cudaStream_t)stream_};
  return run_backbone(h, ex, image, B, H, W, w, (char*)workspace, logits, dense);
}
