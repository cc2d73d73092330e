// SuperPoint backbone on the tensor cores (sp_tc.cu): state owned by an SpHandle whose conf asks for it.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "lg_tc.h"
#include "sp_pipeline.h"

struct SpTc {
  TcEngine tc;        // bf16x3 GEMMs over the bf16 hi / lo images of wpk
  float* wpk;         // packed fp32 weights (device)
  size_t w_off[12];   // float offsets into wpk: weights repacked to [256, k*k*Cin] ...
  size_t b_off[12];   // ... and biases padded to [256]
};

// The backbone's workspace: one buffer plan shared by its sizing (sp_workspace_bytes), its carving (sp_tc_backbone) and
// its host-side export (sp_tc_layout).  Buffers in workspace order; offsets are from the start of the backbone's part.
enum SpTcBuffer { SPT_XH, SPT_XL, SPT_YH, SPT_YL, SPT_FH, SPT_FL, SPT_LOGITS, SPT_DENSE, SPT_STATE, SPT_NBUF };
struct SpTcPlan {
  size_t off[SPT_NBUF], bytes[SPT_NBUF];
  size_t total;
};
SpTcPlan sp_tc_plan(int B, int H, int W);

int sp_tc_create(SpTc** out, const float* wts_dev, cudaStream_t stream);
void sp_tc_destroy(SpTc* t);
int sp_tc_backbone(SpTc* t, const float* wts_dev, const float* image, int B, int H, int W, void* workspace, float* logits_nchw,
                   float* dense_nchw, cudaStream_t stream);

// Stages policy of sp_run_post (sp_pipeline.h): warp / block kernels for candidate compaction, top-k and descriptor
// sampling; top-k beyond SP_SEL_KMAX (4096) falls back to the functor.
struct SpCudaStages {
  cudaStream_t stream;
  int compact_impl(const SpWorkspace& ws, int B, int H, int W, float thr, long cap) const;
  int select_impl(const SpWorkspace& ws, int B, int k, long cap, long out_cap, int rank_all) const;
  int sample_impl(const SpWorkspace& ws, float* kpts, float* kscores, float* desc, int B, int Hc, int Wc, long out_cap) const;
  template <class Exec>
  int compact(Exec&, const SpWorkspace& ws, int B, int H, int W, float thr, long cap) const { return compact_impl(ws, B, H, W, thr, cap); }
  // rank_all: see SpSelect (ALIKED's top-k mode)
  template <class Exec>
  int select(Exec& exec, const SpWorkspace& ws, int B, int k, long cap, long out_cap, int rank_all = 0) const {
    if (k > 4096) return SpFunctorStages().select(exec, ws, B, k, cap, out_cap, rank_all);
    return select_impl(ws, B, k, cap, out_cap, rank_all);
  }
  template <class Exec>
  int sample(Exec&, const SpWorkspace& ws, float* kpts, float* kscores, float* desc, int B, int Hc, int Wc, long out_cap) const {
    return sample_impl(ws, kpts, kscores, desc, B, Hc, Wc, out_cap);
  }
};
