/* disk_b200 -- C ABI of the DISK extractor forward (kornia.feature.DISK as lightglue/disk.py runs it).  Same library
 * (liblightglue_b200.so), same conventions as lightglue_b200.h: plain pointers and sizes, device memory owned by the
 * caller, asynchronous on the given stream, int status (0 = ok, message via lg_last_error()).
 *
 * The U-Net's convolutions run on tensor cores with split-bf16 operands (hi + lo, three MMAs per product, fp32
 * accumulate); the first convolution, the heatmap channel and the instance-norm statistics run in fp32 on CUDA cores.
 * The 128 descriptor channels of the last convolution are computed at the selected keypoints only.
 */
#ifndef DISK_B200_H
#define DISK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define DISK_ABI_VERSION 1

/* Mirrors lightglue.DISK.default_conf (desc_dim is always 128). */
typedef struct DiskConfig {
  int32_t abi_version;          /* DISK_ABI_VERSION */
  int32_t max_num_keypoints;    /* conf.max_num_keypoints; -1 = None (no top-k) */
  int32_t nms_window_size;      /* conf.nms_window_size (5), odd */
  int32_t pad_if_not_divisible; /* conf.pad_if_not_divisible (1): zero-pad right / bottom to multiples of 16 */
  float detection_threshold;    /* conf.detection_threshold (0.0) */
} DiskConfig;

typedef struct DiskHandle DiskHandle;

/* Number of floats in the weight blob: kornia's DISK state_dict tensors, fp32, in state_dict order:
 *   for i in 0..4: unet.path_down.{i}.1.1.weight [cin] (PReLU), .1.3.weight [cout, cin, 5, 5], .1.3.bias [cout]
 *   for i in 0..3: unet.path_up.{i}.conv.1.weight [cin], .conv.3.weight [cout, cin, 5, 5], .conv.3.bias [cout]
 * with (cin, cout) = (3, 16) (16, 32) (32, 64) (64, 64) (64, 64) | (128, 64) (128, 64) (96, 64) (80, 129). */
LG_API size_t disk_weight_blob_floats(void);

LG_API int disk_create(const DiskConfig* cfg, const float* weights_dev, size_t n_floats, void* stream, DiskHandle** out);
LG_API int disk_destroy(DiskHandle* h);

/* Upper bound on keypoints per image for (H, W): max_num_keypoints if set (at least 1), else the packing bound of the NMS
 * window, ceil(H / (w/2 + 1)) ceil(W / (w/2 + 1)); the per-image capacity `cap` of disk_forward must be >= this. */
LG_API int64_t disk_max_keypoints(const DiskHandle* h, int32_t H, int32_t W);
LG_API size_t disk_workspace_bytes(const DiskHandle* h, int32_t B, int32_t H, int32_t W);

/* DISK forward for an image batch [B, C, H, W] fp32, C = 1 (repeated to RGB) or 3.  keypoints [B, cap, 2] (x, y) fp32,
 * scores [B, cap] (raw heatmap values), descriptors [B, cap, 128] (unit norm), counts [B]: the first counts[b] rows of
 * image b are valid, in row-major pixel order; the rest is zero. */
LG_API int disk_forward(DiskHandle* h, const float* image, int32_t C, int32_t B, int32_t H, int32_t W, int64_t cap,
                        float* keypoints, float* scores, float* descriptors, int32_t* counts, void* workspace,
                        size_t workspace_bytes, void* stream);

/* Test entry: the network alone, as disk_forward runs it.  heatmap [B, H, W] (cropped to the image), and the raw
 * (un-normalised) 128 descriptor channels [B, P, 128] at the P pixels pos [B, P] (flat index y W + x, 0 <= y < H,
 * 0 <= x < W) of each image.  Same workspace as disk_forward; P must be <= disk_max_keypoints(H, W). */
LG_API int disk_heads(DiskHandle* h, const float* image, int32_t C, int32_t B, int32_t H, int32_t W, const int32_t* pos,
                      int32_t P, float* heatmap, float* descriptors, void* workspace, size_t workspace_bytes, void* stream);

/* Test entry: the detection alone, as disk_forward runs it on the network's heatmap: NMS (a pixel is kept iff it is the
 * first maximum, in row-major order, of its nms_window_size window), detection_threshold (strict) and kornia's top-k of
 * max_num_keypoints, on a caller-given heatmap [B, H, W] fp32.  positions [B, cap] int32 (pixel y W + x) and scores
 * [B, cap] fp32: the first counts[b] rows of image b are the keypoints disk_forward would return, in row-major pixel
 * order; the rest is zero.  Same H, W, cap and workspace as disk_forward. */
LG_API int disk_detect(DiskHandle* h, const float* heatmap, int32_t B, int32_t H, int32_t W, int64_t cap, int32_t* positions,
                       float* scores, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);

/* Host-only introspection (no device work): the workspace plan of disk_forward / disk_heads for this handle and a
 * [B, C, H, W] batch.  Writes, when non-null, the byte offset from the workspace's start and the size of each of its
 * DISK_LAYOUT_BUFFERS buffers, in this order:
 *   0 .. 7  raw outputs of down0 .. down4, up0 .. up2: fp32 padded NHWC (2-pixel zero border, row b (h+4)(w+4) +
 *           (y+2)(w+4) + (x+2) at the layer's level h x w of the 16-padded image), cout channels (16, 32, 64,
 *           64, 64, 64, 64, 64), bias included; their padding rows hold garbage;
 *   8       x3, up3's input (normalised, PReLU'd), fp32 padded NHWC, 80 channels, padding zero;
 *   9, 10   the descriptor GEMM's im2col rows, bf16 hi / lo [rows, 2048] (column tap 80 + ci, zero past 2000), row
 *           b P + j for disk_heads' P (b max_keypoints + j for disk_forward);
 *   11      the descriptor GEMM's output, fp32 [rows, 128] (bias included);
 *   12      the row-plan state: 6 x 4 int32 words (len[2], stop_layer, unused) of levels 0 .. 4 and of the descriptor
 *           GEMM.
 * After a call the buffers hold that call's values.  Returns the workspace size (disk_workspace_bytes), 0 for a null
 * handle or a non-positive size. */
#define DISK_LAYOUT_BUFFERS 13
LG_API int64_t disk_workspace_layout(const DiskHandle* h, int32_t B, int32_t H, int32_t W, int64_t* offsets, int64_t* bytes);

#ifdef __cplusplus
}
#endif
#endif
