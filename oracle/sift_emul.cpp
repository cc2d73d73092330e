// TEST INFRASTRUCTURE ONLY -- host execution of the SIFT CUDA path's functors.
//
// lightglue_b200/csrc/sift_pipeline.h holds every stage of the SIFT forward as a functor (= the body of one GPU thread)
// plus the per-image orchestration `sift_run`.  This file compiles that header with plain g++ (-ffp-contract=off) and
// runs each functor in a host loop over its index space, with a per-thread scratch array where the GPU uses shared
// memory.  That checks the kernel logic (pyramid arithmetic, refinement, orientation and descriptor histograms, the
// ordering and filtering passes) against fixtures made by the reference with OpenCV, on a machine without a GPU
// (tests/test_sift_emulated.py).  Built into oracle/_build/libsift_emul.so by oracle/Makefile and loaded by tests only.
#include <stdlib.h>
#include <string.h>

#include <thread>
#include <vector>

#include "../lightglue_b200/csrc/sift_pipeline.h"

namespace {
struct HostExec {
  template <class F>
  int run(const F& f) {
    const long n = f.count();
    unsigned nt = std::thread::hardware_concurrency();
    if (nt == 0) nt = 1;
    if (nt > 16) nt = 16;
    const int S = F::SCRATCH > 0 ? F::SCRATCH : 1;
    if (n < 4096 || nt == 1) {
      std::vector<float> scratch(S);
      for (long i = 0; i < n; ++i) f(i, scratch.data());
      return 0;
    }
    std::vector<std::thread> pool;
    const long chunk = (n + nt - 1) / nt;
    for (unsigned t = 0; t < nt; ++t) {
      const long lo = t * chunk, hi = lo + chunk < n ? lo + chunk : n;
      if (lo >= hi) break;
      pool.emplace_back([&f, lo, hi, S] {
        std::vector<float> scratch(S);
        for (long i = lo; i < hi; ++i) f(i, scratch.data());
      });
    }
    for (auto& th : pool) th.join();
    return 0;
  }
  int zero(int* p, int n) {
    memset(p, 0, sizeof(int) * n);
    return 0;
  }
};
}  // namespace

extern "C" {
// Outputs as sift_forward (include/sift_b200.h); image_size: int32 [B, 2] (w, h) or NULL.  counts[b] = -1 when image b
// overflowed the raw keypoint list.  Returns 0 on success.
int sift_emul_forward(int L, double contrast, double edge, int nms_radius, int max_kpts, int rootsift, const float* image,
                      int C, const int* image_size, int B, int H, int W, long cap, float* kpts, float* scales, float* oris,
                      float* scores, float* desc, int* counts) {
  if (L < 1 || L > SIFT_MAX_LAYERS || max_kpts <= 0 || cap < max_kpts) return 1;
  SiftWs w;
  sift_carve(nullptr, H, W, L, max_kpts, &w);
  char* base = (char*)malloc(w.bytes + 256);
  if (!base) return 2;
  char* aligned = (char*)(((uintptr_t)base + 255) & ~(uintptr_t)255);
  sift_carve(aligned, H, W, L, max_kpts, &w);
  const SiftParams p = sift_params(L, contrast, edge, nms_radius, max_kpts, rootsift);
  HostExec ex;
  int rc = 0;
  for (int b = 0; b < B && !rc; ++b) {
    const int iw = image_size ? image_size[2 * b] : W, ih = image_size ? image_size[2 * b + 1] : H;
    rc = sift_run(ex, p, image + (long)b * C * H * W, C, H, W, ih, iw, w, (int)cap, kpts + b * cap * 2, scales + b * cap,
                  oris + b * cap, scores + b * cap, desc + b * cap * SIFT_DESC);
    counts[b] = w.counters[3] ? -1 : w.counters[2];
  }
  free(base);
  return rc;
}
}
