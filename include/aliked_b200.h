/* aliked_b200 -- C ABI of the ALIKED extractor forward, fp32 on CUDA cores.  Same library (liblightglue_b200.so) and
 * same conventions as lightglue_b200.h / superpoint_b200.h: plain pointers and sizes, device memory owned by the
 * caller, asynchronous on the given stream, int status (0 = ok, message via lg_last_error()).
 *
 * Reference interface replaced: lightglue/aliked.py  ALIKED.__init__ + load_state_dict, extract_dense_map (padding to a
 * multiple of 32, encoder with deformable block3 / block4, aggregation, score head, L2-normalised feature map), DKD.forward
 * (simple_nms, borders, threshold / n_limit / top-k / mean-fallback selection, 5x5 soft-argmax, score sampling) and
 * SDDH.forward (descriptors).  Image loading, resizing and gray -> RGB are the caller's business.
 */
#ifndef ALIKED_B200_H
#define ALIKED_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define AL_ABI_VERSION 1

/* Mirrors ALIKED.default_conf plus the row of ALIKED.cfgs for conf.model_name. */
typedef struct AlConfig {
  int32_t abi_version;         /* AL_ABI_VERSION */
  int32_t c1, c2, c3, c4, dim; /* encoder widths and descriptor size (dim == c4, dim % 4 == 0, dim <= 128) */
  int32_t K;                   /* SDDH patch size (3) */
  int32_t M;                   /* SDDH sample positions (16 or 32, <= 32) */
  int32_t nms_radius;          /* conf.nms_radius (2) */
  int32_t max_num_keypoints;   /* conf.max_num_keypoints; <= 0 = none */
  float detection_threshold;   /* conf.detection_threshold (0.2); <= 0 with max_num_keypoints > 0 = top-k mode */
} AlConfig;

typedef struct AlHandle AlHandle;

/* Number of floats in the weight blob of this configuration: every tensor of the reference state_dict except the
 * BatchNorm `num_batches_tracked` counters, fp32, in state_dict order:
 *   block1: conv1.weight bn1.{weight,bias,running_mean,running_var} conv2.weight bn2.{...}
 *   block2: the same, then downsample.weight downsample.bias
 *   block3, block4: conv1.offset_conv.{weight,bias} conv1.regular_conv.weight bn1.{...}
 *                   conv2.offset_conv.{weight,bias} conv2.regular_conv.weight bn2.{...} downsample.{weight,bias}
 *   conv1.weight conv2.weight conv3.weight conv4.weight
 *   score_head.0.weight score_head.2.weight score_head.4.weight score_head.6.weight
 *   desc_head.agg_weights desc_head.offset_conv.0.{weight,bias} desc_head.offset_conv.2.{weight,bias} desc_head.sf_conv.weight
 * Returns 0 for an invalid configuration. */
LG_API size_t al_weight_blob_floats(const AlConfig* cfg);

/* Replaces ALIKED.__init__ + load_state_dict: keeps a device copy of the blob and folds eval-mode BatchNorm into the
 * weights and biases of the eight batch-normalised convolutions (in double, on the device). */
LG_API int al_create(const AlConfig* cfg, const float* weights_dev, size_t n_floats, void* stream, AlHandle** out);
LG_API int al_destroy(AlHandle* h);

/* Upper bound on keypoints per image for (H, W): max_num_keypoints if set, else n_limit_max (20000); at most H * W.
 * The per-image capacity `cap` of al_forward's outputs must be >= this. */
LG_API int64_t al_max_keypoints(const AlHandle* h, int32_t H, int32_t W);
LG_API size_t al_workspace_bytes(const AlHandle* h, int32_t B, int32_t H, int32_t W);

/* Replaces ALIKED.forward for an RGB batch image [B, 3, H, W] fp32, any H, W >= 8.  image_size [B, 2] fp32 (w, h per
 * image, as DKD.forward takes it) or NULL.  keypoints [B, cap, 2] (x, y) in pixels, scores [B, cap], descriptors
 * [B, cap, dim] (unit norm), counts [B] int32: the first counts[b] rows of image b are valid, in the reference's order
 * (row-major, or by descending NMS score when top-k or n_limit applies); the rest is zero. */
LG_API int al_forward(AlHandle* h, const float* image, const float* image_size, int32_t B, int32_t H, int32_t W, int64_t cap,
                      float* keypoints, float* scores, float* descriptors, int32_t* counts, void* workspace,
                      size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
