// TEST INFRASTRUCTURE ONLY -- host execution of the SuperPoint CUDA path's functors.
//
// lightglue_b200/csrc/sp_pipeline.h holds every stage of the extractor forward as a functor (= the body of one GPU
// thread) plus the orchestration `sp_run`.  This file compiles that header with plain g++ and runs each functor in a
// host loop over its index space, so the exact kernel logic (index maths, summation order, NMS passes, compaction,
// rank-by-counting top-k, bilinear sampling) is checked against the reference-generated fixtures on a machine
// without a GPU (tests/test_superpoint_emulated.py).  It is built into oracle/_build/libsp_emul.so by
// oracle/Makefile and loaded by tests only; nothing in the product links or calls it.
#include <stdlib.h>
#include <string.h>

#include <thread>
#include <vector>

#include "../lightglue_b200/csrc/sp_pipeline.h"

namespace {
struct HostExec {
  template <class F>
  int run(const F& f) {
    const long n = f.count();
    unsigned nt = std::thread::hardware_concurrency();
    if (nt == 0) nt = 1;
    if (nt > 16) nt = 16;
    if (n < 4096 || nt == 1) {
      for (long i = 0; i < n; ++i) f(i);
      return 0;
    }
    std::vector<std::thread> pool;
    const long chunk = (n + nt - 1) / nt;
    for (unsigned t = 0; t < nt; ++t) {
      const long lo = t * chunk, hi = lo + chunk < n ? lo + chunk : n;
      if (lo >= hi) break;
      pool.emplace_back([&f, lo, hi] { for (long i = lo; i < hi; ++i) f(i); });
    }
    for (auto& th : pool) th.join();
    return 0;
  }
};
}  // namespace

extern "C" {
size_t sp_emul_blob_floats(void) { return sp_blob_floats(); }

long sp_emul_max_keypoints(int nms_radius, int max_num_keypoints, int H, int W) {
  return (long)sp_keypoint_cap(nms_radius, max_num_keypoints, H, W);
}

// returns 0 on success; outputs as sp_forward (include/superpoint_b200.h)
int sp_emul_forward(const float* weights, int nms_radius, int max_num_keypoints, int remove_borders, float detection_threshold,
                    const float* image, int B, int H, int W, long cap, float* kpts, float* scores, float* desc, int* counts) {
  if (H < SP_CELL || W < SP_CELL) return 1;
  SpWorkspace w;
  sp_carve(nullptr, B, H, W, cap, &w);
  char* base = (char*)malloc(w.bytes + 256);
  if (!base) return 2;
  char* aligned = (char*)(((uintptr_t)base + 255) & ~(uintptr_t)255);
  sp_carve(aligned, B, H, W, cap, &w);
  HostExec ex;
  const SpParams prm{nms_radius, max_num_keypoints, remove_borders, detection_threshold};
  const int rc = sp_run(ex, weights, prm, image, B, H, W, cap, w, kpts, scores, desc);
  if (!rc) memcpy(counts, w.n_sel, (size_t)B * sizeof(int));
  free(base);
  return rc;
}

// sp_post (include/superpoint_b200.h) on the host: the post-processing functors on caller-given logits [B,65,H/8,W/8] and
// dense [B,256,H/8,W/8], in the caller's workspace, carved as sp_workspace_layout lays out a precision-0 workspace
// (cap = sp_max_keypoints), so each stage's output can be read where the GPU leaves it.  Returns 0 on success.
int sp_emul_post(int nms_radius, int max_num_keypoints, int remove_borders, float detection_threshold, const float* logits,
                 const float* dense, int B, int H, int W, long cap, float* kpts, float* scores, float* desc, int* counts,
                 void* workspace, size_t workspace_bytes) {
  if (B <= 0 || H < SP_CELL || W < SP_CELL || cap < sp_keypoint_cap(nms_radius, max_num_keypoints, H, W)) return 1;
  SpWorkspace w;
  sp_carve(nullptr, B, H, W, cap, &w);
  if (!workspace || workspace_bytes < w.bytes) return 2;
  sp_carve((char*)workspace, B, H, W, cap, &w);
  const size_t cells = (size_t)B * (H / SP_CELL) * (W / SP_CELL);
  memcpy(w.logits, logits, 65 * cells * sizeof(float));
  memcpy(w.dense, dense, SP_DESC * cells * sizeof(float));
  HostExec ex;
  const SpParams prm{nms_radius, max_num_keypoints, remove_borders, detection_threshold};
  const int rc = sp_run_post(ex, prm, B, H / SP_CELL * SP_CELL, W / SP_CELL * SP_CELL, cap, w, kpts, scores, desc);
  if (!rc) memcpy(counts, w.n_sel, (size_t)B * sizeof(int));
  return rc;
}
}
