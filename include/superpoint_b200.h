/* superpoint_b200 -- C ABI of the SuperPoint extractor forward (SURVEY.md 8f1: the caller-side row next to the
 * matcher), first CUDA path: fp32 on CUDA cores, no tensor cores yet.  Same library (liblightglue_b200.so), same
 * conventions as lightglue_b200.h: plain pointers and sizes, device memory owned by the caller, asynchronous on the
 * given stream, int status (0 = ok, message via lg_last_error()).
 *
 * Reference interface replaced: lightglue/superpoint.py  SuperPoint.__init__ (126-160) and SuperPoint.forward
 * (163-227) -- encoder, detector head + soft-max, simple_nms (52-68), border removal, threshold, top-k (71-76),
 * descriptor head, sample_descriptors (79-96).  Image loading / resizing / RGB->gray (utils.py, kornia) are the
 * caller's business, as they are outside `forward`.
 */
#ifndef SUPERPOINT_B200_H
#define SUPERPOINT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define SP_ABI_VERSION 2

/* Mirrors SuperPoint.default_conf (superpoint.py:112-118). */
typedef struct SpConfig {
  int32_t abi_version;         /* SP_ABI_VERSION */
  int32_t nms_radius;          /* conf.nms_radius (4) */
  int32_t max_num_keypoints;   /* conf.max_num_keypoints; <= 0 = None (no limit) */
  int32_t remove_borders;      /* conf.remove_borders (4) */
  float detection_threshold;   /* conf.detection_threshold (0.0005) */
  int32_t precision;           /* arithmetic of the twelve convolutions (superpoint.py:137-153): 0 = fp32 on the CUDA
                                  cores (the checker), 1 = wgmma tensor cores, split-bf16 operands (hi + lo, 3 MMAs per
                                  product), fp32 accumulate */
} SpConfig;

typedef struct SpHandle SpHandle;

/* Number of floats in the weight blob: the reference state_dict tensors, fp32, concatenated as
 *   conv1a.weight [64,1,3,3] conv1a.bias [64] conv1b.* conv2a.* conv2b.* conv3a.* conv3b.* conv4a.* conv4b.*
 *   convPa.* convPb.* [65,256,1,1] convDa.* convDb.* [256,256,1,1]            (superpoint.py:137-153) */
LG_API size_t sp_weight_blob_floats(void);

/* Replaces SuperPoint.__init__ + load_state_dict: keeps a device copy of the weight blob. */
LG_API int sp_create(const SpConfig* cfg, const float* weights_dev, size_t n_floats, void* stream, SpHandle** out);
LG_API int sp_destroy(SpHandle* h);

/* Upper bound on keypoints per image for (H, W) under this handle's conf: max_num_keypoints if set, else the
 * packing bound of the NMS window; the per-image capacity `cap` of sp_forward's outputs must be >= this. */
LG_API int64_t sp_max_keypoints(const SpHandle* h, int32_t H, int32_t W);
LG_API size_t sp_workspace_bytes(const SpHandle* h, int32_t B, int32_t H, int32_t W);

/* Replaces SuperPoint.forward (163-227) for a grayscale batch image [B, 1, H, W] fp32 (any H, W >= 8: the poolings floor as in the reference).
 * keypoints [B, cap, 2] (x, y) fp32, scores [B, cap], descriptors [B, cap, 256] (unit norm), counts [B]:
 * the first counts[b] rows of image b are valid -- in the reference's order (row-major, or by descending score
 * when top-k applies) -- the rest is zero. */
LG_API int sp_forward(SpHandle* h, const float* image, int32_t B, int32_t H, int32_t W, int64_t cap, float* keypoints,
               float* scores, float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);

/* The convolution stack alone, exactly as sp_forward runs it for this handle (either precision): the raw detector logits
 * [B, 65, H/8, W/8] (superpoint.py:185) and the un-normalised descriptor map [B, 256, H/8, W/8] (221), fp32 NCHW.
 * Same image and workspace (sp_workspace_bytes) as sp_forward. */
LG_API int sp_backbone(SpHandle* h, const float* image, int32_t B, int32_t H, int32_t W, float* logits, float* dense,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Host-only introspection (no handle, no device): the workspace plan of the tensor-core backbone (precision 1) for a
 * [B, 1, H, W] batch.  Writes, when non-null, the byte offset (from the start of the backbone's part of the workspace) and
 * the size of each of its SP_TC_BUFFERS buffers, in this order: activations X hi, X lo, Y hi, Y lo (the ping-pong maps),
 * features hi, lo (conv4b), logits, dense descriptors (fp32, padded NHWC), tile state.  Returns the part's total size in
 * bytes, 0 for B < 1 or H, W < 8. */
#define SP_TC_BUFFERS 9
LG_API int64_t sp_tc_layout(int32_t B, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes);

#ifdef __cplusplus
}
#endif
#endif
