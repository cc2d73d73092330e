// C ABI of the SuperPoint extractor (include/superpoint_b200.h): executes the functors of sp_pipeline.h on the GPU,
// one thread per logical index.  The same functors and orchestration run on the host in oracle/sp_emul.cpp (tests).
#include <cuda_runtime.h>

#include "../../include/superpoint_b200.h"
#include "lg_internal.h"
#include "sp_pipeline.h"
#include "sp_tc.h"

struct SpHandle {
  SpConfig cfg;
  float* wts;  // device copy of the weight blob
  SpTc* tc;    // tensor-core backbone (cfg.precision == 1), else null
};

namespace {
template <class F>
__global__ void __launch_bounds__(256) sp_for_each_kernel(F f, long n) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i < n) f(i);
}

struct CudaExec {
  cudaStream_t stream;
  long launches = 0;
  template <class F>
  int run(const F& f) {
    const long n = f.count();
    if (n <= 0) return 0;
    const long blocks = (n + 255) / 256;
    if (blocks > 0x7fffffffL) return lg_set_error("superpoint: grid too large");
    sp_for_each_kernel<F><<<(unsigned)blocks, 256, 0, stream>>>(f, n);
    ++launches;
    LG_CHECK_LAUNCH();
    return 0;
  }
};

int64_t max_keypoints(const SpConfig& c, int H, int W) {
  if (c.max_num_keypoints > 0) return c.max_num_keypoints;
  const int step = c.nms_radius + 1;  // no two NMS survivors lie within `nms_radius` of each other (Chebyshev)
  return (int64_t)((H + step - 1) / step) * ((W + step - 1) / step);
}

// The convolution stack of this handle's precision -> logits [B,65,Hc,Wc], dense [B,256,Hc,Wc] (fp32 NCHW); `w` is the
// carve of `workspace`, whose tensor-core part follows the functor buffers
int run_backbone(SpHandle* h, CudaExec& ex, const float* image, int B, int H, int W, SpWorkspace w, char* workspace,
                 float* logits, float* dense) {
  if (h->tc) return sp_tc_backbone(h->tc, h->wts, image, B, H, W, workspace + w.bytes, logits, dense, ex.stream);
  w.logits = logits;
  w.dense = dense;
  return sp_run_backbone(ex, h->wts, image, B, H, W, w);
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
  cudaError_t e = cudaMalloc(&h->wts, n_floats * sizeof(float));
  if (e != cudaSuccess) { delete h; return lg_set_cuda_error(e, __FILE__, __LINE__); }
  e = cudaMemcpyAsync(h->wts, weights_dev, n_floats * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream_);
  if (e != cudaSuccess) { cudaFree(h->wts); delete h; return lg_set_cuda_error(e, __FILE__, __LINE__); }
  if (cfg->precision == 1) {
    int r = sp_tc_create(&h->tc, h->wts, (cudaStream_t)stream_);
    if (r) { cudaFree(h->wts); delete h; return r; }
  }
  *out = h;
  return 0;
}

extern "C" int sp_destroy(SpHandle* h) {
  if (!h) return 0;
  sp_tc_destroy(h->tc);
  cudaFree(h->wts);
  delete h;
  return 0;
}

extern "C" int64_t sp_max_keypoints(const SpHandle* h, int32_t H, int32_t W) { return h ? max_keypoints(h->cfg, H, W) : 0; }

extern "C" size_t sp_workspace_bytes(const SpHandle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  SpWorkspace w;
  sp_carve(nullptr, B, H, W, max_keypoints(h->cfg, H, W), &w);
  return w.bytes + (h->tc ? sp_tc_plan(B, H, W).total : 0);
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
  if (B <= 0 || H < SP_CELL || W < SP_CELL) return lg_set_error("sp_forward: H and W must be at least 8");
  if (cap < max_keypoints(h->cfg, H, W)) return lg_set_error("sp_forward: output capacity below sp_max_keypoints()");
  SpWorkspace w;
  sp_carve((char*)workspace, B, H, W, cap, &w);
  const size_t need = w.bytes + (h->tc ? sp_tc_plan(B, H, W).total : 0);
  if (!workspace || workspace_bytes < need) return lg_set_error("sp_forward: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  CudaExec ex{stream};
  const SpParams prm{h->cfg.nms_radius, h->cfg.max_num_keypoints, h->cfg.remove_borders, h->cfg.detection_threshold};
  int rc = run_backbone(h, ex, image, B, H, W, w, (char*)workspace, w.logits, w.dense);
  if (rc) return rc;
  const int Hs = H / SP_CELL * SP_CELL, Ws = W / SP_CELL * SP_CELL;  // the score map's extents
  // the tensor-core mode also runs the post-processing's heavy stages as warp / block kernels (same results)
  rc = h->tc ? sp_run_post(ex, prm, B, Hs, Ws, cap, w, keypoints, scores, descriptors, SpCudaStages{stream})
             : sp_run_post(ex, prm, B, Hs, Ws, cap, w, keypoints, scores, descriptors);
  if (rc) return rc;
  cudaError_t e = cudaMemcpyAsync(counts, w.n_sel, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, stream);
  if (e != cudaSuccess) return lg_set_cuda_error(e, __FILE__, __LINE__);
  return 0;
}

extern "C" int sp_backbone(SpHandle* h, const float* image, int32_t B, int32_t H, int32_t W, float* logits, float* dense,
                           void* workspace, size_t workspace_bytes, void* stream_) {
  if (!h || !image || !logits || !dense) return lg_set_error("sp_backbone: null argument");
  if (B <= 0 || H < SP_CELL || W < SP_CELL) return lg_set_error("sp_backbone: H and W must be at least 8");
  if (!workspace || workspace_bytes < sp_workspace_bytes(h, B, H, W)) return lg_set_error("sp_backbone: workspace too small");
  SpWorkspace w;
  sp_carve((char*)workspace, B, H, W, max_keypoints(h->cfg, H, W), &w);
  CudaExec ex{(cudaStream_t)stream_};
  return run_backbone(h, ex, image, B, H, W, w, (char*)workspace, logits, dense);
}
