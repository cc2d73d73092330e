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
// overflowed the raw keypoint list.  workspace: a caller-owned host buffer of at least sift_emul_workspace_bytes, carved
// as sift_forward carves its device workspace, so that sift_workspace_layout locates the last image's intermediates in
// it.  Returns 0 on success.
size_t sift_emul_workspace_bytes(int L, int max_kpts, int H, int W) {
  if (L < 1 || L > SIFT_MAX_LAYERS || max_kpts <= 0 || H <= 0 || W <= 0) return 0;
  SiftWs w;
  sift_carve(nullptr, H, W, L, max_kpts, &w);
  return w.bytes + 256;
}

int sift_emul_forward_ws(int L, double contrast, double edge, int nms_radius, int max_kpts, int rootsift,
                         const float* image, int C, const int* image_size, int B, int H, int W, long cap, float* kpts,
                         float* scales, float* oris, float* scores, float* desc, int* counts, void* workspace,
                         size_t workspace_bytes) {
  if (L < 1 || L > SIFT_MAX_LAYERS || max_kpts <= 0 || cap < max_kpts) return 1;
  if (!workspace || workspace_bytes < sift_emul_workspace_bytes(L, max_kpts, H, W)) return 2;
  char* aligned = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  SiftWs w;
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
  return rc;
}

// The ordering and filtering functors of sift_run on n caller-made raw keypoints (SiftKpt records, cap >= n): order,
// flags and pix [cap], out_src [max_kpts], counters [8] as sift_workspace_layout describes them.  Reaches states an
// image does not give, such as equal-score pixel duplicates with equal angles.
int sift_emul_filter(const SiftKpt* kpt, int n, int cap, int w, int nms_radius, int max_kpts, int* order, int* flags,
                     int* pix, int* out_src, int* counters) {
  if (n < 0 || n > cap || max_kpts <= 0) return 1;
  const SiftParams p = sift_params(1, 0.0, 10.0, nms_radius, max_kpts, 0);
  HostExec ex;
  ex.zero(counters, 8);
  counters[4] = counters[5] = n;
  const SiftPost s{kpt, counters + 5, cap, order, flags, pix, counters, w};
  ex.run(SiftSortLex{s});
  ex.run(SiftRetain{s, p});
  ex.run(SiftDogFilter{s, p});
  ex.run(SiftNms{s, p});
  ex.run(SiftSelect{s, p, out_src});
  return 0;
}

// sift_emul_forward_ws on a workspace of its own.
int sift_emul_forward(int L, double contrast, double edge, int nms_radius, int max_kpts, int rootsift, const float* image,
                      int C, const int* image_size, int B, int H, int W, long cap, float* kpts, float* scales, float* oris,
                      float* scores, float* desc, int* counts) {
  const size_t bytes = sift_emul_workspace_bytes(L, max_kpts, H, W);
  if (!bytes) return 1;
  void* base = malloc(bytes);
  if (!base) return 2;
  const int rc = sift_emul_forward_ws(L, contrast, edge, nms_radius, max_kpts, rootsift, image, C, image_size, B, H, W,
                                      cap, kpts, scales, oris, scores, desc, counts, base, bytes);
  free(base);
  return rc;
}
}
