/* geometry_b200 -- C ABI of batched RANSAC on the matcher's output: a homography or a fundamental matrix per pair, for
 * every pair of a batch in one call.  Same library (liblightglue_b200.so), same conventions as lightglue_b200.h: plain
 * pointers and sizes, device memory owned by the caller, asynchronous on the given stream, int status (0 = ok, message
 * via lg_last_error()).  No handle: there are no weights.  No host synchronisation, fixed output shapes, and a launch
 * sequence that depends on (B, M, max_iters) only, so a call can be captured in a CUDA graph.
 *
 * The algorithm, exactly (oracle/geometry_oracle.py restates it in numpy and matches it bit for bit):
 *
 * 1. Compaction.  Match i of pair b is valid when 0 <= matches0[b, i] < N.  The valid matches are compacted per pair in
 *    ascending i; n is their number.  Point k of the pair is (x0, y0) = kpts0[b, i_k], (x1, y1) = kpts1[b, matches0[b, i_k]].
 *
 * 2. Hartley normalisation, per pair and image, in double.  Sums over the n points use one fixed order: 256 partial sums,
 *    partial t adds the terms t, t + 256, t + 512, ... in that order starting from 0.0, then a halving tree
 *    p[t] = p[t] + p[t + h] for h = 128, 64, ..., 1.  c = sum(x) / n (for x and y), d = sum(sqrt(dx*dx + dy*dy)) / n with
 *    dx = x - cx, and s = sqrt(2) / d.  A normalised coordinate is (x - cx) * s.  d == 0 fails the pair.
 *
 * 3. Sampling.  Hypothesis h of a pair draws s distinct indices (s = 4 for H, 8 for F) from draws t = 0, 1, ...:
 *      mix(x)  = x ^= x >> 16; x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^= x >> 16   (32-bit)
 *      r(t)    = mix(mix(mix(seed ^ 0x9e3779b9) ^ h) + t)
 *      index   = (uint64) r(t) * n >> 32
 *    A draw equal to an earlier index of the sample is skipped.  A sample still short of s indices after GEO_MAX_DRAWS
 *    draws is degenerate.  The pair's position in the batch does not enter the hash, so a pair gives the same result in
 *    any batch and on any GPU of a sharded batch.
 *
 * 4. Minimal solvers, in double, on normalised coordinates (x, y) in image 0 and (u, v) in image 1.
 *    H: rows [x, y, 1, 0, 0, 0, -u*x, -u*y, -u] and [0, 0, 0, x, y, 1, -v*x, -v*y, -v] per point, points in sample order.
 *       Before solving, the sample is rejected when, for any triple (i, j, k) of {(0,1,2), (1,2,3), (0,2,3), (0,1,3)} in
 *       either image, |D| <= GEO_FLT_EPS * (((|xj-xi| + |yj-yi|) + |xk-xi|) + |yk-yi|) with
 *       D = (xj-xi)*(yk-yi) - (xk-xi)*(yj-yi) (collinear), or when the products D0*D1 of the four triples are neither all
 *       >= 0 nor all < 0 (OpenCV's orientation test: the signs of the triangle areas differ between the images).
 *    F: row [u*x, u*y, u, v*x, v*y, v, x, y, 1] per point (x1^T F x0 = 0).
 *    The 8x9 system is reduced by Gaussian elimination with partial pivoting (the first row of largest |a| in column k;
 *    rows r > k: f = a[r][k] / a[k][k], a[r][c] = a[r][c] - f*a[k][c] for c > k).  A pivot with |a[k][k]| <= GEO_PIVOT_EPS
 *    marks a rank-deficient sample.  The null vector has x8 = 1 and, for k = 7 .. 0,
 *    x[k] = -(a[k][8] + a[k][k+1]*x[k+1] + ... + a[k][7]*x[7]) / a[k][k], summed left to right.
 *    F is then made rank 2 (below).
 *    Denormalisation: H = T1^-1 Hn T0, F = T1^T Fn T0 with T = [[s, 0, -(s*cx)], [0, s, -(s*cy)], [0, 0, 1]] and
 *    T^-1 = [[1/s, 0, cx], [0, 1/s, cy], [0, 0, 1]]; a 3x3 product is (A_i0*B_0j + A_i1*B_1j) + A_i2*B_2j.
 *    Scale: with f = sqrt of the row-major running sum of squares, H is divided by H[2][2] when |H[2][2]| >= 1e-12 * f,
 *    else by f; F is divided by f and negated if its first entry of largest magnitude is negative.
 *    Rank 2: one-sided Jacobi on the columns of Fn (pairs (0,1), (0,2), (1,2), GEO_SVD_SWEEPS sweeps; a pair with
 *    |g| <= 1e-15 * sqrt(a*b) is skipped, a, b, g the column dot products; z = (b - a) / (2g),
 *    t = sign(z) / (|z| + sqrt(1 + z*z)), c = 1 / sqrt(1 + t*t), s = c*t, columns p' = c*p - s*q, q' = s*p + c*q on Fn and
 *    V), the column of least squared norm set to zero, Fn = A V^T.
 *
 * 5. Scoring, in fp32 (the model rounded to float, no fused multiply-adds; x0 = (x0, y0, 1), x1 = (x1, y1, 1)):
 *    H: w = 1 / ((h6*x0 + h7*y0) + h8); dx = x1 - ((h0*x0 + h1*y0) + h2) * w; dy likewise with h3..h5;
 *       err = dx*dx + dy*dy.
 *    F: (a, b, c) = F x0 row by row, d2 = (x1*a + y1*b) + c, s2 = 1 / (a*a + b*b);
 *       (a, b, c) = F^T x1, d1 = (x0*a + y0*b) + c, s1 = 1 / (a*a + b*b); err = fmaxf(d1*d1*s1, d2*d2*s2).
 *    A point is an inlier when err < (float)(threshold * threshold).  The score is the inlier count; ties go to the lowest
 *    hypothesis index.  A degenerate hypothesis has no score.
 *
 * 6. Adaptive stopping.  Hypotheses run in chunks of GEO_CHUNK.  After chunk c a pair stops once
 *    min(GEO_CHUNK*(c+1), max_iters) >= RANSACUpdateNumIters(confidence, 1 - best/n, s, max_iters), OpenCV's formula in
 *    double with pow(1 - ep, s) as s - 1 left-to-right products; with confidence >= 1 no pair stops early.
 *    num_hypotheses is the number of hypotheses drawn.
 *
 * 7. Refit.  With at least s inliers, the best hypothesis's inliers give a least-squares refit by the same rows: the upper
 *    triangle of A^T A (45 entries, per point the sum over its rows of a_i*a_j, summed over the points in the order of
 *    step 2 with non-inliers adding 0), the eigenvector of its smallest eigenvalue by cyclic Jacobi (GEO_EIG_SWEEPS sweeps
 *    over p < q in row order, skip a_pq == 0, z = (a_qq - a_pp) / (2 a_pq), t = sign(z) / (|z| + sqrt(z*z + 1)),
 *    c = 1 / sqrt(t*t + 1), s = t*c, columns then rows then V; the first least diagonal entry), rank 2 for F, then the
 *    same denormalisation and scale.  The refit replaces the hypothesis unless it has fewer inliers.  No Levenberg-
 *    Marquardt refinement follows.
 *
 * A pair fails (success 0, model all zero, no inliers, best_hypothesis -1) when n < s, when its normalisation fails, or
 * when every hypothesis is degenerate.
 */
#ifndef GEOMETRY_B200_H
#define GEOMETRY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef LG_API
#define LG_API __attribute__((visibility("default")))
#endif

#define GEO_ABI_VERSION 1
#define GEO_HOMOGRAPHY 0
#define GEO_FUNDAMENTAL 1

#define GEO_CHUNK 256
#define GEO_MAX_DRAWS 64
#define GEO_MAX_ITERS (1 << 24)
#define GEO_FLT_EPS 1.1920928955078125e-07 /* FLT_EPSILON */
#define GEO_PIVOT_EPS 1e-10
#define GEO_SVD_SWEEPS 8
#define GEO_EIG_SWEEPS 12

typedef struct GeoConfig {
  int32_t abi_version; /* GEO_ABI_VERSION */
  int32_t model;       /* GEO_HOMOGRAPHY or GEO_FUNDAMENTAL */
  int32_t max_iters;   /* hypotheses per pair, in [1, GEO_MAX_ITERS] */
  uint32_t seed;
  double threshold;    /* pixels, > 0: transfer error (H) or epipolar distance (F) */
  double confidence;   /* in [0, 1] */
} GeoConfig;

typedef struct GeoInputs {
  int32_t B, M, N;
  const float* kpts0;      /* [B, M, 2] */
  const float* kpts1;      /* [B, N, 2] */
  const int64_t* matches0; /* [B, M]; indices outside [0, N) are unmatched */
} GeoInputs;

typedef struct GeoOutputs {
  double* model;           /* [B, 3, 3] */
  uint8_t* inliers;        /* [B, M] */
  int32_t* num_inliers;    /* [B] */
  uint8_t* success;        /* [B] */
  int32_t* best_hypothesis; /* [B], -1 without one */
  int32_t* num_hypotheses;  /* [B] */
} GeoOutputs;

LG_API size_t geo_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_estimate(const GeoConfig* cfg, const GeoInputs* in, GeoOutputs* out, void* workspace,
                        size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
