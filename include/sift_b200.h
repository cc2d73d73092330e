/* sift_b200 -- C ABI of the SIFT extractor forward (OpenCV's SIFT as the reference runs it, then the reference's
 * post-processing), fp32 on CUDA cores.  Same library (liblightglue_b200.so) and conventions as lightglue_b200.h /
 * superpoint_b200.h / aliked_b200.h: plain pointers and sizes, device memory owned by the caller, asynchronous on the
 * given stream, int status (0 = ok, message via lg_last_error()).
 *
 * Reference interface replaced: lightglue/sift.py  SIFT with backend "opencv": rgb_to_grayscale, the image_size crop,
 * (image * 255).astype(uint8), cv2.SIFT_create(contrastThreshold, nfeatures, edgeThreshold, nOctaveLayers).detectAndCompute
 * (2x upsampled first octave, sigma 1.6), filter_dog_point, the top-k by score and sift_to_rootsift.  There are no
 * weights.
 *
 * sift_workspace_layout exposes where sift_forward leaves its intermediates (the pyramid, the candidate and raw keypoint
 * lists, the filtering state), so that each stage can be checked against float64 from the kernels' own inputs.  The
 * list records have fixed byte layouts (SiftCand: x, y, size, response fp32, then r, c, layer, octave_packed int32, 32
 * bytes; SiftKpt: x, y, size, angle, response fp32, then octave_packed, o, layer int32, 32 bytes; angle in degrees).
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

/* Host-only introspection (no device work, no handle needed): the workspace plan of sift_forward for a handle created
 * with this configuration, an [B, C, H, W] batch, and the pyramid of an image cropped to (h, w) (1 <= h <= H,
 * 1 <= w <= W).  Offsets are in bytes from the workspace's first 256-byte-aligned address, where sift_forward carves.
 * Images are processed one after the other in one set of buffers, so when sift_forward returns they hold the state of
 * the LAST image of the batch only (and the pyramid is laid out by that image's crop).  Writes, when non-null, the
 * offset and size of each of SIFT_LAYOUT_BUFFERS buffers, in this order:
 *   0  counters  int32 [8]: [0] raw keypoints in the list, min(n_kpt, raw_cap); [1] 1 if the nfeatures cut
 *                (retainBest) applied; [2] output rows (counts when not overflowed); [3] 1 if the candidate or raw list
 *                overflowed (counts = -1); [4] candidates found (n_cand, may exceed raw_cap); [5] raw keypoints found
 *                (n_kpt, may exceed raw_cap); [6], [7] unused;
 *   1  q         fp32 [h * w] the 8-bit gray crop (uint8 values), stride w;
 *   2  tmp       unspecified (the row pass of the blurs);
 *   3  pyr       every Gaussian and DoG layer (located by gauss / dog below);
 *   4  cand      SiftCand [raw_cap] refined extrema (adjustLocalExtrema's output, coordinates of the upsampled image),
 *                valid up to min(counters[4], raw_cap), in atomic (nondeterministic) order;
 *   5  kpt       SiftKpt [raw_cap] raw keypoints, one per orientation peak (final coordinates), valid up to
 *                min(counters[5], raw_cap), in atomic order;
 *   6  order     int32 [raw_cap] lexicographic position -> raw index (KeyPoint_LessThan, ties by raw index);
 *   7  flags     int32 [raw_cap] by lexicographic position: bit 0 unique (removeDuplicatedSorted), 1 kept by
 *                retainBest, 2 kept by filter_dog_point's pixel duplicates, 3 kept by its NMS;
 *   8  pix       int32 [raw_cap] by lexicographic position: filter_dog_point's pixel i * w + j;
 *   9  out_src   int32 [max_num_keypoints] output row -> lexicographic position (rows < counters[2]).
 * Positions past counters[0] hold stale values.  The pyramid plan: *n_octaves octaves; dims[2 o], dims[2 o + 1] the
 * (rows, columns) of octave o (octave 0 is the 2x upsampled crop, each next one every other pixel of the previous);
 * gauss[o * (L + 3) + i] (i < L + 3) and dog[o * (L + 2) + i] (i < L + 2) the byte offsets of Gaussian layer i and of
 * DoG layer i = gauss i+1 - gauss i (fp32, row-major with stride dims[2 o + 1]), L = num_octave_layers.  Arrays of
 * SIFT_LAYOUT_MAX_OCTAVES (dims: twice that, gauss: times L + 3, dog: times L + 2) entries suffice.  gauss[0][1] holds
 * blurred layer 1; the upsampled image it held first is lost.
 * Returns sift_workspace_bytes, 0 for an invalid configuration or sizes. */
#define SIFT_LAYOUT_BUFFERS 10
#define SIFT_LAYOUT_MAX_OCTAVES 16
LG_API int64_t sift_workspace_layout(const SiftConfig* cfg, int32_t H, int32_t W, int32_t h, int32_t w, int64_t* offsets,
                                     int64_t* bytes, int32_t* n_octaves, int32_t* dims, int64_t* gauss, int64_t* dog);

#ifdef __cplusplus
}
#endif
#endif
