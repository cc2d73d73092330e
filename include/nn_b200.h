/* nn_b200 -- C ABI of the nearest-neighbour matcher: mutual nearest neighbours with Lowe's ratio test and a distance
 * threshold on unit-norm descriptors, for every pair of a batch in one call, on the tensor cores in split-bf16.  Same
 * library (liblightglue_b200.so) and conventions as lightglue_b200.h: plain pointers and sizes, device memory owned by
 * the caller, asynchronous on the given stream, int status (0 = ok, message via lg_last_error()).  No host
 * synchronisation and a launch sequence that depends on (B, M, N, D) only, so a call can be captured in a CUDA graph.
 * The B x M x N similarity matrix is never written to memory.
 *
 * Semantics (oracle/nn_oracle.py restates them in float64).  Pair b has image 0 rows i < m_b and image 1 rows j < n_b,
 * m_b = lens0[b] and n_b = lens1[b] (clamped to [0, M] / [0, N]) when given, M and N otherwise.
 *   s_ij = d0_i . d1_j, the dot product of the descriptors.  They are expected to be unit-norm, as every extractor of
 *        this library returns them; the matcher does not re-normalise them.
 *   Image 0 -> image 1, per row i:
 *     j1 = the j with the largest s_ij (on a tie the lowest j), s1 = s_i,j1;
 *     s2 = the largest s_ij over j != j1 (it may equal s1; -inf when n_b = 1);
 *     D1 = 2 (1 - s1), D2 = 2 (1 - s2) (+inf when s2 = -inf): the squared L2 distances of unit vectors;
 *     row i keeps j1 when n_b >= 1 and (ratio_thresh <= 0 or D1 <= r2 * D2) and (distance_thresh <= 0 or D1 <= t2),
 *     with r2 = (float)(ratio_thresh^2) and t2 = (float)(distance_thresh^2) formed in double, and D1, D2, the product
 *     and the comparisons in fp32.
 *   Image 1 -> image 0 likewise, per row j.
 *   mutual_check != 0: a kept i -> j survives only if j -> i is kept as well, and the same from the other side.
 *   Outputs: matches0[b, i] = the surviving j or -1, matching_scores0[b, i] = (s1 + 1) / 2 for a matched row (in [0, 1]
 *   for unit descriptors, like LightGlue's scores) and 0 otherwise; matches1 / matching_scores1 from image 1's side.
 *   Rows past a pair's count get -1 and 0.  A pair with m_b = 0 or n_b = 0 matches nothing.  matches[b] lists the
 *   pairs (i, matches0[b, i]) of the matched rows in ascending i, match_scores[b] their scores, n_matches[b] how many.
 *   Without the mutual check these come from image 0's side only, and several rows of image 0 may name the same j.
 *
 * Arithmetic: s_ij comes from three bf16 tensor-core products with fp32 accumulation, d = hi + lo with hi = bf16(d) and
 * lo = bf16(d - hi): hi0 hi1 + hi0 lo1 + lo0 hi1 (lo0 lo1 is dropped).  For unit descriptors and D <= 512 it differs
 * from the exact dot product by about 5e-5 at most; it is exact when every descriptor entry is a bf16 value and the sums
 * are exact in fp32.
 *
 * Work: the pairs run in groups of G pairs (G * Lp <= NN_GROUP_ROWS rows per image, at least one pair; Lp = max(M, N)
 * rounded up to a multiple of 128), three launches per group: the split into bf16 hi / lo images, one tensor-core
 * sweep that computes every S tile of both directions and keeps, per row and per 128 columns, the best two similarities
 * and the arg-max, and one CTA per pair that merges them, applies the tests and writes the outputs.
 */
#ifndef NN_B200_H
#define NN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define NN_ABI_VERSION 1
#define NN_MIN_DIM 64       /* dim: a multiple of 64 in [NN_MIN_DIM, NN_MAX_DIM] */
#define NN_MAX_DIM 512
#define NN_GROUP_ROWS 32768 /* rows of one image's side the pairs of one group hold together */

/* Mirrors NearestNeighborMatcher.default_conf; thresholds <= 0 switch their test off. */
typedef struct NnConfig {
  int32_t abi_version;   /* NN_ABI_VERSION */
  int32_t dim;           /* descriptor size D */
  int32_t mutual_check;  /* non-zero: keep mutual nearest neighbours only */
  float ratio_thresh;    /* Lowe's ratio r on distances, in (0, 1]; <= 0: off */
  float distance_thresh; /* t on the L2 distance; <= 0: off */
} NnConfig;

typedef struct NnInputs {
  int32_t B, M, N;
  const float* desc0;   /* [B, M, D] fp32, 16-byte aligned */
  const float* desc1;   /* [B, N, D] */
  const int32_t* lens0; /* optional DEVICE [B]: pair b uses the first lens0[b] rows of desc0; NULL = M */
  const int32_t* lens1; /* optional DEVICE [B]; NULL = N */
} NnInputs;

typedef struct NnOutputs {
  int64_t* matches0;       /* [B, M] -1 = unmatched */
  int64_t* matches1;       /* [B, N] */
  float* matching_scores0; /* [B, M] */
  float* matching_scores1; /* [B, N] */
  int32_t* n_matches;      /* [B] */
  int64_t* matches;        /* [B, M, 2] (i, j), ascending i; the first n_matches[b] rows are valid.  M rows: without
                              the mutual check every row of image 0 may match */
  float* match_scores;     /* [B, M] */
} NnOutputs;

typedef struct NnHandle NnHandle;

/* The handle holds the tensor-map cache of the tensor-core sweep; it has no weights. */
LG_API int nn_create(void* stream, NnHandle** out);
LG_API int nn_destroy(NnHandle* h);

/* Scratch bytes of nn_match for a (B, M, N, D) problem (0 for invalid sizes): the bf16 images and the per-slot
 * partials of one group of pairs, O(G Lp (D + Lp / 128 * 3) * 8) bytes.  No zero fill is needed. */
LG_API size_t nn_workspace_bytes(int32_t B, int32_t M, int32_t N, int32_t D);

LG_API int nn_match(NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnOutputs* out, void* workspace,
                    size_t workspace_bytes, void* stream);

/* Host-only introspection (no handle, no device): where nn_match (guided = 0) or nn_match_guided (guided != 0,
 * below) leaves each stage's output in its workspace for a (B, M, N, D) problem.  The pairs run in groups of G (the
 * last group holds g = B - (groups - 1) G <= G of them); a group of g pairs has 2g sequences of Lp rows each, sequence
 * s < g holding image 0 of the group's pair s and sequence g + s image 1 of it, so row r of sequence s is row s Lp + r
 * of the buffers below, which are sized for R = 2 G Lp rows.  Every buffer is reused by each group: after a call it
 * holds the LAST group's values (pairs (groups - 1) G .. B - 1).  Writes, when non-null, plan = {G, Lp, pstride,
 * groups} and the byte offset from the workspace start and the size of each of the NN_LAYOUT_BUFFERS buffers, in
 * order:
 *   0 hi      bf16 [R, D]: bf16_rn(d) of each live row, zero past the row's pair length;
 *   1 lo      bf16 [R, D]: bf16_rn(d - hi), zero past the pair length;
 *   2 part    fp32 [R, pstride, 2]: per row and 128-column slot t of the partner sequence (its columns
 *             128 t .. 128 t + 127), (s1, s2) of the live (guided: live and gated) columns: the slot's best
 *             similarity and the best over its other columns (s1 on a tie; -inf with one such column; s1 = s2 = -inf
 *             with none);
 *   3 parg    int32 [R, pstride]: the slot's j1, the lowest column among its maxima (INT32_MAX with no such column);
 *             part and parg are written for the live rows, in the slot pairs of every 256-column tile with a live
 *             column; the tail reads slots t < ceil(n / 128), n the partner's length;
 *   4 jbest   int32 [R]: the row's j1 when it passes the ratio and distance tests, else -1 (live rows only);
 *   5 sbest   fp32 [R]: the row's s1 (live rows only);
 *   6 len     int32 [2G]: the clamped length of each sequence (the first 2g);
 *   7 stop    int32 [G]: zero (the first g);
 *   8 rec     fp32 [6, R]: guided only (offset -1 and size 0 otherwise): field f of row r at f 2g Lp + r, the gate
 *             records of nn_match_guided (H: fields 0 and 1, F: all six), zero for rows past M or N;
 *   9 gate_on int32 [G]: guided only: non-zero for a pair matched under its model (the first g).
 * Returns the workspace size (nn_workspace_bytes or nn_guided_workspace_bytes), 0 for B < 1 or an invalid size. */
#define NN_LAYOUT_BUFFERS 10
LG_API int64_t nn_workspace_layout(int32_t B, int32_t M, int32_t N, int32_t D, int32_t guided, int64_t* offsets,
                                   int64_t* bytes, int32_t* plan);

/* Guided matching: each pair is matched again under its estimated homography H (image 0 -> image 1) or fundamental
 * matrix F (x1^T F x0 = 0), with the conventions of geo_estimate (include/geometry_b200.h), and a candidate (i, j)
 * counts only when it is consistent with that model (oracle/nn_guided_oracle.py restates the rules in float64).
 *   gate(i, j) holds iff err(i, j) < t2, t2 = (float)(max_error * max_error) formed in double, where err is exactly
 *   step 5 of include/geometry_b200.h on x0 = kpts0[b, i], x1 = kpts1[b, j]: the model rounded to float, fp32 without
 *   fused multiply-adds; H the forward transfer error, F the larger (fmaxf) of the two squared point-to-line distances.
 *   So (i, j) passes at max_error = t exactly when geo_estimate at threshold t counts it as an inlier of that model.  A
 *   NaN error (a non-finite keypoint, a zero F) fails the gate.  The gate depends on the pair (i, j) only, not on the
 *   direction of the sweep.
 *   Pair b with valid[b] != 0 (or valid NULL) follows nn_match's rules with "every column" read as "every gated
 *   column": j1 is the lowest gated j among the maxima, s2 the best over the other gated columns (-inf when there are
 *   none), and a row with no gated column matches nothing; image 1's side likewise, then the mutual check.  Scores,
 *   matches, match_scores and n_matches are defined as in nn_match.
 *   Pair b with valid[b] == 0 is matched ungated: its outputs equal nn_match's bit for bit, so passing an estimator's
 *   success flags as valid never loses a pair whose estimation failed.
 * Work: nn_match's three launches per group plus one that writes a gate record per row (H: the projected point of an
 * image-0 row, the point of an image-1 row; F: the point, its epipolar line in the other image and 1 / (a^2 + b^2));
 * the tensor-core sweep evaluates the gate in its top-2 epilogue.  The launch sequence depends on (B, M, N, D, kind).
 */
#define NN_GUIDE_H 0 /* the model is a homography, as GEO_HOMOGRAPHY */
#define NN_GUIDE_F 1 /* the model is a fundamental matrix, as GEO_FUNDAMENTAL */

typedef struct NnGuide {
  int32_t kind;         /* NN_GUIDE_H or NN_GUIDE_F */
  const double* model;  /* DEVICE [B, 9] row-major, 8-byte aligned */
  const uint8_t* valid; /* optional DEVICE [B]: 0 = match the pair ungated; NULL = every pair is guided */
  const float* kpts0;   /* DEVICE [B, M, 2] pixels, 8-byte aligned */
  const float* kpts1;   /* DEVICE [B, N, 2] */
  double max_error;     /* pixels, positive and finite */
} NnGuide;

/* Scratch bytes of nn_match_guided for a (B, M, N, D) problem (0 for invalid sizes): nn_workspace_bytes' buffers and
 * the gate records of one group, 24 bytes per row. */
LG_API size_t nn_guided_workspace_bytes(int32_t B, int32_t M, int32_t N, int32_t D);

LG_API int nn_match_guided(NnHandle* h, const NnConfig* cfg, const NnInputs* in, const NnGuide* guide,
                           const NnOutputs* out, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NN_B200_H */
