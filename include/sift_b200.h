/* sift_b200 -- C ABI of the SIFT extractor forward (OpenCV's SIFT as the reference runs it, then the reference's
 * post-processing), fp32 on CUDA cores.  Same library (liblightglue_b200.so) and conventions as lightglue_b200.h /
 * superpoint_b200.h / aliked_b200.h: plain pointers and sizes, device memory owned by the caller, asynchronous on the
 * given stream, int status (0 = ok, message via lg_last_error()).
 *
 * Reference interface replaced: lightglue/sift.py  SIFT with backend "opencv": rgb_to_grayscale, the image_size crop,
 * (image * 255).astype(uint8), cv2.SIFT_create(contrastThreshold, nfeatures, edgeThreshold, nOctaveLayers).detectAndCompute
 * (2x upsampled first octave, sigma 1.6), filter_dog_point, the top-k by score and sift_to_rootsift.  There are no
 * weights.
 */
#ifndef SIFT_B200_H
#define SIFT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define SIFT_ABI_VERSION 1

/* Mirrors SIFT.default_conf (backend "opencv"). */
typedef struct SiftConfig {
  int32_t abi_version;        /* SIFT_ABI_VERSION */
  int32_t num_octave_layers;  /* conf.num_octaves, which the reference passes as nOctaveLayers (4); 1..8 */
  int32_t nms_radius;         /* conf.nms_radius (0); -1 = None (no filter_dog_point) */
  int32_t max_num_keypoints;  /* conf.max_num_keypoints (4096) > 0: nfeatures and the top-k */
  int32_t rootsift;           /* conf.rootsift (1) */
  int32_t reserved;
  double detection_threshold; /* conf.detection_threshold, OpenCV's contrastThreshold (0.0066667) */
  double edge_threshold;      /* conf.edge_threshold (10) */
} SiftConfig;

typedef struct SiftHandle SiftHandle;

LG_API int sift_create(const SiftConfig* cfg, void* stream, SiftHandle** out);
LG_API int sift_destroy(SiftHandle* h);

/* Keypoints per image at most: max_num_keypoints.  The per-image capacity `cap` of sift_forward's outputs must be >= this. */
LG_API int64_t sift_max_keypoints(const SiftHandle* h, int32_t H, int32_t W);
/* Images are processed one after the other in one set of buffers, so this does not grow with B. */
LG_API size_t sift_workspace_bytes(const SiftHandle* h, int32_t B, int32_t H, int32_t W);

/* Replaces SIFT.forward for image [B, channels, H, W] fp32 (channels 1 or 3; values in [0, 1]), H, W >= 1.
 * image_size: HOST int32 [B, 2] (w, h per image, each image cropped to [:h, :w] first) or NULL.  keypoints [B, cap, 2]
 * (x, y), scales [B, cap] (cv::KeyPoint::size), oris [B, cap] (radians), scores [B, cap] (response), descriptors
 * [B, cap, 128], counts [B] int32: the first counts[b] rows of image b are valid, the rest is zero.  Row order: OpenCV's
 * (x, y, size desc, angle, response desc) order, or descending score (ties in that order) when the nfeatures cut or the
 * top-k applied.  counts[b] = -1: image b had more raw keypoints than the internal list holds (its rows are not valid). */
LG_API int sift_forward(SiftHandle* h, const float* image, int32_t channels, const int32_t* image_size, int32_t B, int32_t H,
                        int32_t W, int64_t cap, float* keypoints, float* scales, float* oris, float* scores,
                        float* descriptors, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
