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

/* Host-only introspection (no device work, no handle needed): the workspace plan of al_forward for a handle created
 * with this configuration, a [B, 3, H, W] batch and cap = al_max_keypoints(H, W).  Writes, when non-null, the byte
 * offset from the workspace's start and the size of each of its AL_LAYOUT_BUFFERS buffers, in this order, with what
 * each holds when al_forward returns.  All fp32 NCHW unless
 * stated; Hp x Wp is the image replicate-padded to multiples of 32 (top = (Hp - H) / 2 rows above, left = (Wp - W) / 2
 * columns to the left), level l of the encoder is (Hp / s) x (Wp / s) with s = 1, 2, 8, 32, P0 = B Hp Wp, q = dim / 4.
 * Only what is listed here may be relied on; the buffers are disjoint.
 *   0      img    first P0 floats: the score head's sigmoid output on the padded frame [B, 1, Hp, Wp], before the crop
 *                 (the padded image it held first is partly overwritten);
 *   1      ta     first 4 P0 floats: score_head.2 + SELU [B, 4, Hp, Wp]; next 4 P0: score_head.4 + SELU (block1's
 *                 first convolution, which this buffer held first, is lost);
 *   2      x1     block1's output [B, c1, Hp, Wp];
 *   3      s1     score_head.0 + SELU [B, 8, Hp, Wp];
 *   4      invn   1 / max(|x1234|, 1e-12) per padded pixel [B, Hp, Wp];
 *   5 .. 9   p1 t2 d2 x2 a2: 2x2 pool of x1 [B, c1, .] and at 1/2: block2's SELU(bn1(conv1 p1)) [B, c2, .], its
 *                 downsample (1x1 + bias) of p1 [B, c2, .], block2's output x2 [B, c2, .], SELU(conv2 x2) [B, q, .];
 *   10 .. 15 p2 o3 t3 d3 x3 a3: 4x4 pool of x2 [B, c2, .] and at 1/8: block3's *second* offset convolution (+ bias,
 *                 clamped to +-max(h, w) / 4) of t3 [B, 18, .], t3 = SELU(bn1(deform conv1 p2)) [B, c3, .], the
 *                 downsample of p2, x3, SELU(conv3 x3) [B, q, .];
 *   16 .. 21 p3 o4 t4 d4 x4 a4: the same for block4 at 1/32 (c3 -> c4 channels);
 *   22     score  the cropped score map [B, H, W];
 *   23     nms    simple_nms of score with the borders zeroed; in threshold mode every value not above the image's
 *                 threshold (detection_threshold, or its mean score in the fallback) is then -1 [B, H, W];
 *   24     kpn    normalised keypoints (x, y) in [-1, 1] [B, cap, 2], zero past counts[b];
 *   25     mean   threshold mode only: each image's mean score [B];
 *   26     cnt    threshold mode only: int32 count of NMS values above detection_threshold per image [B];
 *   27     sel_pos    int32 flat pixel index y W + x of each output row [B, cap] (rows < counts[b]);
 *   28     sel_score  the NMS score of each output row, 0 for top-k filler rows [B, cap] (rows < counts[b]);
 *   29     n_sel      int32 counts [B].
 * Returns the workspace size (al_workspace_bytes), 0 for an invalid configuration or a non-positive size. */
#define AL_LAYOUT_BUFFERS 30
LG_API int64_t al_workspace_layout(const AlConfig* cfg, int32_t B, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes);

#ifdef __cplusplus
}
#endif
#endif
