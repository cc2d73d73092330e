// SIFT extractor forward (include/sift_b200.h; reference lightglue/sift.py, backend "opencv"), fp32 on CUDA cores.
//
// The stages are the functors of sift_pipeline.h, run by `sift_run` with one thread per index; the test-only host
// build (oracle/sift_emul.cpp) runs the same functors.  This file is compiled with -fmad=false so that every unfused
// multiply-add rounds as OpenCV's (and the host build's) does; fused ones are explicit fmaf() in the header.
//
// Per image, in stream order, in one set of workspace buffers:
//   gray / crop / 8-bit quantisation, 2x linear upsample, initial blur
//   per octave: decimation of the previous octave, L+2 separable blurs (row pass, column pass with the DoG)
//   per octave and DoG layer: extremum test + refinement, appending candidates (atomic counter)
//   orientation histograms, one thread per candidate (36 + 4 bins in shared memory), appending raw keypoints
//   ordering and filtering by counting over all raw keypoints: lexicographic rank, dedupe + retainBest,
//   filter_dog_point (pixel duplicates, NMS), top-k and output slots
//   descriptors, one thread per output row (its 360-bin histogram in shared memory), uint8 rounding and RootSIFT
#include <cuda_runtime.h>

#include "../../include/sift_b200.h"
#include "lg_internal.h"
#include "sift_pipeline.h"

namespace {

template <class F>
__global__ void sift_stage(const F f, long n) {
  extern __shared__ float sift_smem[];
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f(i, sift_smem + (size_t)threadIdx.x * F::SCRATCH);
}

struct CudaExec {
  cudaStream_t s;
  template <class F>
  int run(const F& f) {
    const long n = f.count();
    if (n <= 0) return 0;
    const int threads = F::SCRATCH > 64 ? 32 : 128;
    const size_t smem = sizeof(float) * F::SCRATCH * threads;
    sift_stage<F><<<(unsigned)((n + threads - 1) / threads), threads, smem, s>>>(f, n);
    LG_CHECK_LAUNCH();
    return 0;
  }
  int zero(int* p, int n) {
    LG_CU(cudaMemsetAsync(p, 0, sizeof(int) * n, s));
    return 0;
  }
};

__global__ void sift_count_kernel(const int* counters, int32_t* count) { *count = counters[3] ? -1 : counters[2]; }

}  // namespace

struct SiftHandle {
  SiftConfig cfg;
};

extern "C" int sift_create(const SiftConfig* cfg, void*, SiftHandle** out) {
  if (!cfg || !out) return lg_set_error("sift_create: null argument");
  if (cfg->abi_version != SIFT_ABI_VERSION) return lg_set_error("sift_create: ABI version mismatch");
  if (cfg->num_octave_layers < 1 || cfg->num_octave_layers > SIFT_MAX_LAYERS)
    return lg_set_error("sift_create: num_octaves (OpenCV's nOctaveLayers) must be in [1, 8]");
  if (cfg->max_num_keypoints <= 0) return lg_set_error("sift_create: max_num_keypoints must be positive");
  if (cfg->nms_radius < -1) return lg_set_error("sift_create: nms_radius must be >= 0, or -1 for None");
  *out = new SiftHandle{*cfg};
  return 0;
}

extern "C" int sift_destroy(SiftHandle* h) {
  delete h;
  return 0;
}

extern "C" int64_t sift_max_keypoints(const SiftHandle* h, int32_t, int32_t) { return h ? h->cfg.max_num_keypoints : 0; }

extern "C" size_t sift_workspace_bytes(const SiftHandle* h, int32_t, int32_t H, int32_t W) {
  if (!h || H <= 0 || W <= 0) return 0;
  SiftWs w;
  sift_carve(nullptr, H, W, h->cfg.num_octave_layers, h->cfg.max_num_keypoints, &w);
  return w.bytes + 256;
}

extern "C" int sift_forward(SiftHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B,
                            int32_t H, int32_t W, int64_t cap, float* keypoints, float* scales, float* oris, float* scores,
                            float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!h || !image || !keypoints || !scales || !oris || !scores || !descriptors || !counts)
    return lg_set_error("sift_forward: null argument");
  if (B <= 0 || H <= 0 || W <= 0) return lg_set_error("sift_forward: empty batch or image");
  if (channels != 1 && channels != 3) return lg_set_error("sift_forward: channels must be 1 or 3");
  if (cap < h->cfg.max_num_keypoints) return lg_set_error("sift_forward: output capacity below sift_max_keypoints()");
  for (int b = 0; image_size && b < B; ++b)
    if (image_size[2 * b] < 1 || image_size[2 * b] > W || image_size[2 * b + 1] < 1 || image_size[2 * b + 1] > H)
      return lg_set_error("sift_forward: image_size outside the image");
  const size_t need = sift_workspace_bytes(h, B, H, W);
  if (!workspace || workspace_bytes < need) return lg_set_error("sift_forward: workspace too small");
  char* base = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  SiftWs w;
  sift_carve(base, H, W, h->cfg.num_octave_layers, h->cfg.max_num_keypoints, &w);
  CudaExec ex{(cudaStream_t)stream_};
  const SiftConfig& c = h->cfg;
  const SiftParams p = sift_params(c.num_octave_layers, c.detection_threshold, c.edge_threshold, c.nms_radius,
                                   c.max_num_keypoints, c.rootsift);
  for (int b = 0; b < B; ++b) {
    const int iw = image_size ? image_size[2 * b] : W, ih = image_size ? image_size[2 * b + 1] : H;
    LG_RC(sift_run(ex, p, image + (long)b * channels * H * W, channels, H, W, ih, iw, w, (int)cap, keypoints + b * cap * 2,
                   scales + b * cap, oris + b * cap, scores + b * cap, descriptors + b * cap * SIFT_DESC));
    sift_count_kernel<<<1, 1, 0, ex.s>>>(w.counters, counts + b);
    LG_CHECK_LAUNCH();
  }
  return 0;
}

// DoG-HardNet's detection (dhn_api.cu): sift_forward's stages for one image, without the descriptor histograms.  The
// functors stay compiled here only, with this file's -fmad=false.
size_t sift_detect_workspace_bytes(const SiftConfig& c, int H, int W) {
  SiftWs w;
  sift_carve(nullptr, H, W, c.num_octave_layers, c.max_num_keypoints, &w);
  return w.bytes + 256;
}

int sift_detect_image(const SiftConfig& c, const float* image, int channels, int H, int W, int h, int w, void* workspace,
                      int64_t cap, float* keypoints, float* scales, float* oris, float* scores, int32_t* count,
                      cudaStream_t stream) {
  char* base = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  SiftWs ws;
  sift_carve(base, H, W, c.num_octave_layers, c.max_num_keypoints, &ws);
  CudaExec ex{stream};
  const SiftParams p = sift_params(c.num_octave_layers, c.detection_threshold, c.edge_threshold, c.nms_radius,
                                   c.max_num_keypoints, 0);
  LG_RC(sift_run(ex, p, image, channels, H, W, h, w, ws, (int)cap, keypoints, scales, oris, scores, nullptr));
  sift_count_kernel<<<1, 1, 0, stream>>>(ws.counters, count);
  LG_CHECK_LAUNCH();
  return 0;
}
