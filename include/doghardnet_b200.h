/* doghardnet_b200 -- C ABI of the DoG-HardNet extractor forward (lightglue/dog_hardnet.py: OpenCV's SIFT keypoints as
 * lightglue.SIFT gives them, then kornia's LAFDescriptor(HardNet) on 32x32 patches sampled from an image pyramid).
 * Same library (liblightglue_b200.so) and conventions as sift_b200.h / disk_b200.h: plain pointers and sizes, device
 * memory owned by the caller, asynchronous on the given stream, int status (0 = ok, message via lg_last_error()).
 *
 * Detection is the SIFT extractor's (sift_b200.h) without its descriptor histograms: keypoints, scales, oris and scores
 * are bit-identical to sift_forward's with the same conf.  The patch sampling, the patch normalisation and HardNet's
 * first convolution run in fp32 on CUDA cores; HardNet's other six convolutions run on tensor cores with split-bf16
 * operands (hi + lo, three MMAs per product, fp32 accumulate).  BatchNorm is folded into the convolutions at dhn_create.
 */
#ifndef DOGHARDNET_B200_H
#define DOGHARDNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define DHN_ABI_VERSION 1

/* Mirrors SiftConfig (sift_b200.h) without `rootsift`: the reference overrides SIFT.forward and never applies it. */
typedef struct DhnConfig {
  int32_t abi_version;        /* DHN_ABI_VERSION */
  int32_t num_octave_layers;  /* conf.num_octaves, OpenCV's nOctaveLayers (4); 1..8 */
  int32_t nms_radius;         /* conf.nms_radius (0); -1 = None (no filter_dog_point) */
  int32_t max_num_keypoints;  /* conf.max_num_keypoints (4096) > 0 */
  double detection_threshold; /* conf.detection_threshold, OpenCV's contrastThreshold (0.0066667) */
  double edge_threshold;      /* conf.edge_threshold (10) */
} DhnConfig;

typedef struct DhnHandle DhnHandle;

/* Number of floats in the weight blob: kornia's HardNet, fp32, for i in 0..6 the convolution features.{0,3,6,9,12,15,19}
 * .weight [cout, cin, k, k] followed by its BatchNorm's running_mean [cout] and running_var [cout]
 * (features.{1,4,7,10,13,16,20}; num_batches_tracked is not part of the blob), with (cin, cout, k) = (1, 32, 3)
 * (32, 32, 3) (32, 64, 3) (64, 64, 3) (64, 128, 3) (128, 128, 3) (128, 128, 8). */
LG_API size_t dhn_weight_blob_floats(void);

LG_API int dhn_create(const DhnConfig* cfg, const float* weights_dev, size_t n_floats, void* stream, DhnHandle** out);
LG_API int dhn_destroy(DhnHandle* h);

/* Keypoints per image at most: max_num_keypoints.  The per-image capacity `cap` of the outputs must be >= this. */
LG_API int64_t dhn_max_keypoints(const DhnHandle* h, int32_t H, int32_t W);
/* Images are processed one after the other, and patches in chunks of fixed size, so this does not grow with B. */
LG_API size_t dhn_workspace_bytes(const DhnHandle* h, int32_t B, int32_t H, int32_t W);

/* Replaces DoGHardNet.forward for image [B, channels, H, W] fp32 (channels 1 or 3; values in [0, 1]).  Arguments and
 * outputs as sift_forward's, with HardNet descriptors (unit norm) in place of SIFT's: image_size HOST int32 [B, 2]
 * (w, h) or NULL; keypoints [B, cap, 2], scales [B, cap] (cv::KeyPoint::size), oris [B, cap] (radians), scores [B, cap],
 * descriptors [B, cap, 128], counts [B] (-1: image b overflowed the internal keypoint list).  Rows past counts[b] are
 * zero. */
LG_API int dhn_forward(DhnHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B, int32_t H,
                       int32_t W, int64_t cap, float* keypoints, float* scales, float* oris, float* scores,
                       float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);

/* kornia's LAFDescriptor(HardNet) for the LAFs the reference builds from given keypoints: laf_from_center_scale_ori(
 * keypoints, 6 scales, rad2deg(oris)) on the gray image cropped to image_size (HOST int32 [B, 2] (w, h), or NULL).
 * keypoints [B, cap, 2], scales [B, cap], oris [B, cap] (radians), counts [B] (DEVICE int32: the first counts[b] rows of
 * image b are described); descriptors [B, cap, 128], zero past counts[b].  cap <= dhn_max_keypoints(); same workspace
 * as dhn_forward. */
LG_API int dhn_describe(DhnHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B, int32_t H,
                        int32_t W, int64_t cap, const float* keypoints, const float* scales, const float* oris,
                        const int32_t* counts, float* descriptors, void* workspace, size_t workspace_bytes, void* stream);

/* Host-only introspection (no device work): the workspace plan of dhn_forward / dhn_describe for this handle and an
 * H x W image.  Patches run in chunks of 256; each level of a chunk is a padded NHWC map of 256 patches (34 x 34,
 * 18 x 18 or 10 x 10 rows per patch, a 1-pixel zero border), stored as the rows of tc_rows(256 * rows per patch).
 * Writes, when non-null, the byte offset from the workspace's start and the size of each of its DHN_LAYOUT_BUFFERS
 * buffers, in this order (bf16 hi / lo pairs; after a call they hold the last chunk of the last image):
 *   0, 1    conv 0's output (34 x 34, 64 channels, 32 live), then the four polyphase images of conv 1's output: phase
 *           2 py + px from row (2 py + px) R, R = the rows of the 18 x 18 level, holds padded pixel
 *           (2 (i - 1) + py, 2 (j - 1) + px) at frame position (i, j) of an 18 x 18 frame per patch, i, j >= 1;
 *   2, 3    conv 1's output (34 x 34, 64 channels), then the polyphase images of conv 3's output (10 x 10 frames);
 *   4, 5    conv 2's output; 6, 7 conv 3's output (18 x 18, 64 channels);
 *   8, 9    conv 4's output; 10, 11 conv 5's output (10 x 10, 128 channels);
 *   12, 13  conv 6's input rows [rows, 8192] (column (ky 8 + kx) 128 + ci), row k for keypoint k of the image;
 *   14      conv 6's output, fp32 [rows, 128] (folded BatchNorm included, before F.normalize);
 *   15      the row-plan state: int32 words (len[2], stop_layer, unused) per chunk and level, then conv 6's.
 * Returns the workspace size (dhn_workspace_bytes), 0 for a null handle or a non-positive size. */
#define DHN_LAYOUT_BUFFERS 16
LG_API int64_t dhn_workspace_layout(const DhnHandle* h, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes);

#ifdef __cplusplus
}
#endif
#endif
