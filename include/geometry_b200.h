/* geometry_b200 -- C ABI of batched RANSAC on the matcher's output: a homography, a fundamental matrix, a relative
 * pose (E, R, t) or an absolute pose (R, t from 2D-3D matches) per pair, for every pair of a batch in one call.  Same
 * library (liblightglue_b200.so), same conventions as lightglue_b200.h: plain pointers and sizes, device memory owned
 * by the caller, asynchronous on the given stream, int status (0 = ok, message via lg_last_error()).  No handle: there
 * are no weights.  No host synchronisation, fixed output shapes, and a launch
 * sequence that depends on (B, M, max_iters) only, so a call can be captured in a CUDA graph.
 *
 * The algorithm, exactly (oracle/geometry_oracle.py restates it in numpy and matches it bit for bit):
 *
 * 1. Compaction.  Match i of pair b is valid when 0 <= matches0[b, i] < N and both kpts0[b, i] and
 *    kpts1[b, matches0[b, i]] have finite coordinates (float): a match with a NaN or infinite keypoint is never an inlier
 *    and does not count in n.  The valid matches are compacted per pair in ascending i; n is their number.  Point k of the pair is (x0, y0) = kpts0[b, i_k], (x1, y1) = kpts1[b, matches0[b, i_k]].
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
 *
 * Relative pose (geo_relative_pose; oracle/pose_oracle.py restates it bit for bit): an essential matrix E with
 * x1^T E x0 = 0 on calibrated coordinates, and the (R, t) of x1 = R x0 + t that recoverPose would choose.
 *
 * P1. Compaction as step 1 (a non-finite keypoint invalidates its match).  K = [[fx, s, cx], [0, fy, cy], [0, 0, 1]] per pair and image (K[1][0] is not read);
 *     y = ((double)v - cy) / fy, x = (((double)u - cx) - s*y) / fx, rounded to float.  The solver, the refit and the
 *     triangulation read these floats widened to double.  No Hartley step.  A K with a non-finite entry, fx <= 0, fy <= 0
 *     or a bottom row other than (0, 0, 1) fails its pair.  The threshold is t = threshold / f with
 *     f = (((fx0 + fy0) + fx1) + fy1) / 4, compared as (float)(t*t).
 * P2. Sampling as step 3 with s = 5.
 * P3. Five-point solver, in double.  Rows [u*x, u*y, u, v*x, v*y, v, x, y, 1] (as F) in sample order; the 5x9 system is
 *     reduced as in step 4 (5 pivots, GEO_PIVOT_EPS).  For free column f = 5..8 a null vector has x_f = 1, the other
 *     free entries 0 and x[k] = -(a[k][f] + a[k][k+1]*x[k+1] + ... + a[k][4]*x[4]) / a[k][k] for k = 4..0, summed left
 *     to right: X, Y, Z, W.  Modified Gram-Schmidt in that order (d = running dot product, b_i = b_i - d*b_j for
 *     j < i, then b_i / sqrt(running sum of squares)).  E = x X + y Y + z Z + W: each entry a polynomial over the
 *     graded monomials 1 | x y z | xx xy xz yy yz zz | xxx xxy xxz xyy xyz xzz yyy yyz yzz zzz.  A product of two
 *     polynomials adds a_i*b_j into its monomial for i, then j, ascending, starting from 0.  Constraint 0 is
 *     (E0*d0 - E1*d1) + E2*d2 with d0 = E4*E8 - E5*E7, d1 = E3*E8 - E5*E6, d2 = E3*E7 - E4*E6 (row-major E0..E8).
 *     S_ij = (E_i0*E_j0 + E_i1*E_j1) + E_i2*E_j2, tr = (S_00 + S_11) + S_22, and constraint 1 + 3i + j is
 *     2*((S_i0*E_0j + S_i1*E_1j) + S_i2*E_2j) - tr*E_ij.  The 10x20 matrix has the monomial columns
 *     xxx yyy xxy xyy xxz xx yyz yy xyz xy | xzz xz x yzz yz y zzz zz z 1.  It is degenerate with a non-finite entry;
 *     else Gauss-Jordan for k = 0..9: the first row r >= k of largest |g[r][k]| is the pivot (degenerate unless
 *     > GEO_PIVOT_EPS * max|g|), swapped in, g[k][c] = g[k][c] / g[k][k] and then g[r][c] = g[r][c] - g[r][k]*g[k][c]
 *     for every r != k in ascending order, c > k.  With R_r = g[r][10..19], rows (4, 5), (6, 7), (8, 9) give
 *     e - z*f = x*px(z) + y*py(z) + p1(z) with px = [e2, e1 - f2, e0 - f1, -f0], py = [e5, e4 - f5, e3 - f4, -f3],
 *     p1 = [e9, e8 - f9, e7 - f8, e6 - f7, -f6] (ascending powers): the rows (k, l, m) of a 3x3 B(z).
 *     det B = (kx*c0 - ky*c1) + k1*c2, c0 = ly*m1 - l1*my, c1 = lx*m1 - l1*mx, c2 = lx*my - ly*mx (univariate
 *     products in ascending (i, j) from 0): p(z) of degree 10.  Degenerate with a non-finite coefficient or
 *     |p10| <= GEO_LEAD_EPS * max|p_i|.  q = p / p10; r_b = 1 + max_{i<10} |q_i|.  Sturm sequence: s0 = q,
 *     s1_i = (i + 1) * q_(i+1); s_k = -r / max|r| with r = s_(k-2) mod s_(k-1) (r_i = a_i - (a_da/b_db)*b_(i-1), then
 *     r_i = r_i - (r_(da-1)/b_db)*b_i); the sequence ends before a remainder with a non-finite entry or a zero leading
 *     coefficient.  V(z): sign changes over the members (Horner, zeros skipped); V(-inf), V(+inf) from the leading
 *     signs; n = max(V(-inf) - V(+inf), 0) roots.  Root k = 1..n: lo = -r_b, hi = r_b and GEO_STURM_STEPS bisections
 *     (mid = 0.5*(lo + hi); hi = mid when V(-inf) - V(mid) >= k, else lo = mid), then from z = 0.5*(lo + hi)
 *     GEO_NEWTON_STEPS Newton steps on q (Horner for q and q' together), a non-finite step leaving z.  No real root is
 *     a degenerate sample.  Per root: B(z) by Horner; of the cross products r0 x r1, r0 x r2, r1 x r2 the first of
 *     largest |third entry| w gives x = c0 / w, y = c1 / w; E = ((x*X + y*Y) + z*Z) + W is kept when its running sum of
 *     squares f is finite and positive, scaled to unit Frobenius norm and negated if its first entry of largest
 *     magnitude is negative.  Solution r is the r-th kept one, in ascending z; a sample has at most
 *     GEO_MAX_SOLUTIONS.
 * P4. Scoring in fp32 without fused multiply-adds, every solution of every sample, OpenCV's squared Sampson error:
 *     (a0, a1, a2) = E x0 row by row as in step 5, d = (u*a0 + v*a1) + a2, b0 = (e0*u + e3*v) + e6,
 *     b1 = (e1*u + e4*v) + e7, err = (d*d) / (((a0*a0 + a1*a1) + b0*b0) + b1*b1); an inlier has err < (float)(t*t).
 *     Ties go to the lowest (sample h, solution r): the key packs ~(h*16 + r).  max_iters counts samples.
 * P5. Stopping as step 6 with s = 5.
 * P6. Refit.  With at least GEO_REFIT_MIN inliers, the upper triangle of A^T A over the best solution's inliers as
 *     step 7 (rows of P3), its least eigenvector by the 9x9 cyclic Jacobi, then U diag(1, 1, 0) V^T: one-sided Jacobi
 *     of step 4 on the 3x3, column m of least squared norm dropped, the other two (i < j) give u1 = a_i / sqrt(n_i),
 *     u2 = a_j / sqrt(n_j), v1, v2 (columns of V), E_ab = u1_a*v1_b + u2_a*v2_b, scaled as in P3.  The refit replaces
 *     the solution unless it has fewer inliers.
 * P7. Pose.  u1, u2, v1, v2 of the final E as in P6, u3 = u1 x u2, v3 = v1 x v2 (so U and V are proper rotations),
 *     R1_ab = (u2_a*v1_b - u1_a*v2_b) + u3_a*v3_b (U W V^T, W = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]),
 *     R2_ab = (u1_a*v2_b - u2_a*v1_b) + u3_a*v3_b, candidates (R1, u3), (R2, u3), (R1, -u3), (R2, -u3).  Each inlier
 *     is triangulated per candidate with P0 = [I | 0], P1 = [R | t]: rows [-1, 0, x, 0], [0, -1, y, 0],
 *     u*P1_2 - P1_0, v*P1_2 - P1_1, N_ij = ((r0_i*r0_j + r1_i*r1_j) + r2_i*r2_j) + r3_i*r3_j, Q its least eigenvector
 *     by the same cyclic Jacobi (4x4).  It passes when Q2*Q3 > 0, Z = Q2/Q3 < distance_threshold and
 *     z1 = ((R_20*X + R_21*Y) + R_22*Z) + t2 lies in (0, distance_threshold), X = Q0/Q3, Y = Q1/Q3.  The candidate
 *     with most passing points wins (ties: the lowest); its passing points are pose_inliers.
 * P8. A pair fails (success 0, E, R and t zero, no inliers, best_hypothesis = best_solution = -1) when n < 5, a K is
 *     invalid, or every sample is degenerate.
 *
 * LO-RANSAC relative pose (geo_relative_pose_lo; oracle/lo_pose_oracle.py restates it bit for bit): the outputs of
 * geo_relative_pose, from an MSAC-scored five-point RANSAC with Levenberg-Marquardt local optimisation (Chum, Matas and
 * Kittler, DAGM 2003; the schedule of PoseLib's LO-RANSAC, with the deviations below).  Expressions evaluate left to
 * right as written; every multiply and add rounds on its own.
 *
 * L1. Compaction, calibration, K checks and the threshold thr2 = (float)(t*t) exactly as P1.  M <= GEO_LO_MAX_MATCHES.
 * L2. Sampling and the five-point solutions exactly as P2 and P3: with the same seed both estimators draw the same
 *     samples and solve the same solutions.
 * L3. MSAC score, per solution of every sample, from P4's fp32 err (the solution rounded to float):
 *     w = GEO_LO_QSCALE / thr2 in fp32; for err < thr2, q = 0 when err == 0, else
 *     (uint32)fminf(err * w, GEO_LO_QSCALE) (fp32 product, truncated), so a subnormal thr2 with w = +inf stays
 *     defined; q = GEO_LO_QSCALE otherwise.  score = sum of q over the points in uint64 (exact in any order), count = the number of err < thr2.  Lower is
 *     better; ties go to the lowest (sample h, solution r).
 * L4. Local optimisation, after every chunk of GEO_CHUNK samples, once per pair.  Chunk c's best solution (lowest
 *     (score, h, r)) is taken when the pair has no model yet or its score is strictly below the model's score; else
 *     nothing happens.  Taken, it becomes the pair's model (score, count, h, r) with the (R, t) of P7's candidate choice
 *     on its inliers (its fp32 E widened to double as P7's E).  Then GEO_LO_STEPS LM steps (below) from that (R, t)
 *     give (R', t'), which are scored as L3 through E' = [t']x R' scaled as P3 and rounded to float; with a strictly
 *     lower score they replace the model (keeping h and r) and num_local_optimizations counts one.
 * L5. Stopping as P5 from the model's count (a local optimisation's count included).
 * L6. Final refinement: GEO_LO_FINAL_STEPS LM steps from the model's (R, t), kept unless their L3 score is higher.
 * L7. LM, in double on the calibrated points read as floats widened.  At a pose (R, t):
 *     E = [t]x R unscaled (column j is t x R[:, j], cross products a x b = (a1*b2 - a2*b1, a2*b0 - a0*b2,
 *     a0*b1 - a1*b0)); per point a0 = (E0*x + E1*y) + E2, a1, a2 likewise, d = (u*a0 + v*a1) + a2,
 *     b0 = (E0*u + E3*v) + E6, b1 = (E1*u + E4*v) + E7, den = ((a0*a0 + a1*a1) + b0*b0) + b1*b1, err = (d*d) / den,
 *     r = d / sqrt(den).  A point is an inlier at this pose when err < (double)thr2.  The tangent basis of t: m the
 *     first index of least |t_m|, c = t x e_m, b1 = c / sqrt((c0*c0 + c1*c1) + c2*c2), b2 = t x b1.  The parameters
 *     delta0..4 move the pose to R' = Q R with Q the quaternion rotation of A7, and t' = v / sqrt((v0*v0 + v1*v1) + v2*v2)
 *     with v_i = (t_i + delta3*b1_i) + delta4*b2_i.  dE_k = [t]x ([e_k]x R) for k < 3 and [b_(k-2)]x R for k = 3, 4
 *     (column-wise cross products as above); da, dd, db of dE_k as a, d, b of E,
 *     dden = ((a0*da0 + a1*da1) + b0*db0) + b1*db1, J_k = (dd - d*dden / den) / sqrt(den).  The 21 terms J_i*J_j
 *     (i <= j in row order) and J_i*r over the inliers, and the truncated cost (err for an inlier, else (double)thr2)
 *     over every point, are each summed in the order of step 2.  A step solves the 5x5 system of A7 (damping, Cholesky,
 *     right-hand side -J^T r), lambda starts at GEO_LO_LAMBDA0, and the step is taken only if the truncated cost at the
 *     new pose, with its own inliers, is strictly lower: A7's schedule.
 * L8. Outputs: E = [t]x R of the final (R, t) scaled as P3; R and t as they are; inliers the points with err < thr2
 *     under that E rounded to float (num_inliers their number, cost its L3 score); pose_inliers the inliers that pass
 *     P7's triangulation test for that single (R, t).  best_hypothesis and best_solution name the solution that seeded
 *     the final model; num_hypotheses the samples drawn.  A pair fails as P8, with num_local_optimizations and cost 0.
 *     Deviations from PoseLib: local optimisation runs at most once per chunk rather than at every new best, so the
 *     launch sequence is fixed and the result is deterministic; the score is quantised to integers; there is no
 *     non-minimal refit inside the LO and no PROSAC ordering.
 *
 * LO-RANSAC homography (geo_homography_lo; oracle/lo_homography_oracle.py restates it bit for bit): the outputs of
 * geo_estimate for GEO_HOMOGRAPHY, from an MSAC-scored four-point RANSAC with Levenberg-Marquardt local optimisation,
 * on the schedule of L1-L8.  Expressions evaluate left to right as written; every multiply and add rounds on its own.
 *
 * LH1. Compaction and Hartley normalisation exactly as steps 1-2; thr2 = (float)(threshold * threshold).
 *      M <= GEO_LO_MAX_MATCHES.
 * LH2. Sampling and the four-point DLT exactly as steps 3-4, with OpenCV's collinearity and orientation rejection and
 *      the same scale: with the same seed both estimators draw the same samples and solve the same hypotheses.
 * LH3. MSAC score, per hypothesis, from step 5's fp32 forward transfer error err (the model rounded to float):
 *      q as L3 (0 at err == 0, else (uint32)fminf(err * w, GEO_LO_QSCALE) for err < thr2, else GEO_LO_QSCALE),
 *      so a non-finite err (a point mapped to infinity, w = 1/0) scores as an outlier.  score = sum of q over the
 *      points in uint64, count = the number of err < thr2.  Lower is better; ties go to the lowest h.
 * LH4. Local optimisation, after every chunk of GEO_CHUNK samples, once per pair.  Chunk c's best hypothesis (lowest
 *      (score, h)) is taken when the pair has no model yet or its score is strictly below the model's score; else
 *      nothing happens.  Taken, its double H of step 4 becomes the pair's model (score, count, h).  Then GEO_LO_STEPS
 *      LM steps (LH7) from it give Hn', whose pixel model H' = T1^-1 Hn' T0 scaled as step 4 is scored as LH3; with a
 *      strictly lower score H' replaces the model (keeping h) and num_local_optimizations counts one.
 * LH5. Stopping as step 6 with s = 4 from the model's count (a local optimisation's count included).
 * LH6. Final refinement: GEO_LO_FINAL_STEPS LM steps from the model, kept unless their LH3 score is higher.
 * LH7. LM, in double, on the normalised model at unit Frobenius norm: from a pixel H (row-major, as everywhere here),
 *      Hn = (T1 H) T0^-1 (3x3 products as step 4; T1 = [[s1, 0, -(s1*cx1)], [0, s1, -(s1*cy1)], [0, 0, 1]],
 *      T0^-1 = [[1/s0, 0, cx0], [0, 1/s0, cy0], [0, 0, 1]]) divided by the square root of its running sum of squares.
 *      Tangent basis at Hn: m the first index of least |Hn_m|, v = e_m - Hn (v_i = (i == m ? 1.0 : 0.0) - Hn_i),
 *      vv = running sum of v_i*v_i, c = 2.0 / vv; the reflection I - c v v^T maps e_m to Hn, and its columns j != m
 *      in ascending j are b_0..b_7: b_k,i = (i == j ? 1.0 : 0.0) - c*v_i*v_j.  The parameters delta0..7 move Hn to
 *      Hn' = x / sqrt(running sum of x_i*x_i) with x_i = Hn_i + delta0*b_0,i + ... + delta7*b_7,i (left to right).
 *      Residuals in pixels, on the compacted floats widened: with h = (T1^-1 Hn) T0 unscaled (T1^-1 as step 4),
 *      w = 1.0 / ((h6*x0 + h7*y0) + h8), px = ((h0*x0 + h1*y0) + h2) * w, py = ((h3*x0 + h4*y0) + h5) * w,
 *      dx = x1 - px, dy = y1 - py, err = dx*dx + dy*dy; an inlier at this model has err < (double)thr2.  With
 *      g = (T1^-1 b_k) T0 and da = (g0*x0 + g1*y0) + g2, db, dc likewise (g3..g5, g6..g8): jx_k = -((da - px*dc) * w),
 *      jy_k = -((db - py*dc) * w).  The 36 terms jx_i*jx_j + jy_i*jy_j (i <= j in row order) and the 8 terms
 *      jx_i*dx + jy_i*dy over the inliers, and the truncated cost (err for an inlier, else (double)thr2) over every
 *      point, are each summed in the order of step 2.  A step solves the 8x8 system of A7 (damping, Cholesky,
 *      right-hand side -J^T r), lambda starts at GEO_LO_LAMBDA0, and the step is taken only if the truncated cost at
 *      Hn', with its own inliers, is strictly lower: A7's schedule.
 * LH8. Outputs: model the final H (a hypothesis's H of step 4, or T1^-1 Hn T0 scaled as step 4); inliers the points
 *      with err < thr2 under it rounded to float, num_inliers their number and cost its LH3 score; best_hypothesis the
 *      hypothesis that seeded it; num_hypotheses the samples drawn.  A pair fails as step 7's failures (n < 4, a failed
 *      normalisation, every sample degenerate), with num_local_optimizations and cost 0.  Deviations from PoseLib:
 *      local optimisation runs at most once per chunk rather than at every new best, so the launch sequence is fixed
 *      and the result is deterministic; the score is quantised to integers; there is no non-minimal (DLT) refit inside
 *      the LO and no PROSAC ordering.
 *
 * LO-RANSAC fundamental matrix (geo_fundamental_lo; oracle/lo_fundamental_oracle.py restates it bit for bit): the
 * outputs of geo_estimate for GEO_FUNDAMENTAL, from an MSAC-scored eight-point RANSAC with Levenberg-Marquardt local
 * optimisation of a rank-2 F, on the schedule of L1-L8.  Expressions evaluate left to right as written; every multiply
 * and add rounds on its own.
 *
 * LF1. Compaction and Hartley normalisation exactly as steps 1-2; thr2 = (float)(threshold * threshold).
 *      M <= GEO_LO_MAX_MATCHES.
 * LF2. Sampling (s = 8) and the eight-point solver, rank 2, denormalisation and scale exactly as steps 3-4: with the
 *      same seed both estimators draw the same samples and solve the same hypotheses.
 * LF3. MSAC score, per hypothesis, from step 5's fp32 error err (the larger of the two squared point-to-epipolar-line
 *      distances, the model rounded to float): q as L3 (0 at err == 0, else (uint32)fminf(err * w, GEO_LO_QSCALE) for
 *      err < thr2, else GEO_LO_QSCALE), so a non-finite err scores as an outlier.  score = sum of q over the points in
 *      uint64, count = the number of err < thr2.  Lower is better; ties go to the lowest h.
 * LF4. Local optimisation, after every chunk of GEO_CHUNK samples, once per pair.  Chunk c's best hypothesis (lowest
 *      (score, h)) is taken when the pair has no model yet or its score is strictly below the model's score; else
 *      nothing happens.  Taken, its double F of step 4 becomes the pair's model (score, count, h).  Then GEO_LO_STEPS
 *      LM steps (LF7) from it give (U', V', sig'), whose pixel model F' = T1^T Fn' T0 scaled as step 4 is scored as
 *      LF3; with a strictly lower score F' replaces the model (keeping h) and num_local_optimizations counts one.
 * LF5. Stopping as step 6 with s = 8 from the model's count (a local optimisation's count included).
 * LF6. Final refinement: GEO_LO_FINAL_STEPS LM steps from the model, kept unless their LF3 score is higher.
 * LF7. LM, in double, on the normalised model in the orthonormal representation of Bartoli and Sturm (PoseLib's
 *      FactorizedFundamentalMatrix: 7 degrees of freedom, rank 2 by construction).  From a pixel F (row-major),
 *      Fn = (T1^-T F) T0^-1 (3x3 products as step 4; T1^-T = [[1/s1, 0, 0], [0, 1/s1, 0], [cx1, cy1, 1]],
 *      T0^-1 = [[1/s0, 0, cx0], [0, 1/s0, cy0], [0, 0, 1]]).  Factorisation: step 4's one-sided Jacobi on Fn, the column
 *      m of least squared norm n_m (the first) dropped; of the two kept columns (i < j) the one of larger squared norm
 *      (i on a tie) is p, the other q: u1 = a_p / sqrt(n_p), u2 = a_q / sqrt(n_q), v1, v2 the columns p, q of V,
 *      u3 = u1 x u2, v3 = v1 x v2 (a x b = (a1*b2 - a2*b1, a2*b0 - a0*b2, a0*b1 - a1*b0)), sig = sqrt(n_q) / sqrt(n_p).
 *      U = [u1 u2 u3] and V = [v1 v2 v3] are rotations, and Fn(U, V, sig)_ab = u1_a*v1_b + sig*u2_a*v2_b.  The
 *      parameters delta0..6 move the model to U' = Q(delta0..2) U, V' = Q(delta3..5) V (3x3 products as step 4, Q the
 *      quaternion rotation of A7) and sig' = sig + delta6; sig is not clamped.  Directions at Fn = Fn(U, V, sig):
 *      D_k = [e_k]x Fn (column j is e_k x Fn[:, j]) for k = 0..2, D_(3+k) = -Fn [e_k]x (row i is e_k x Fn[i, :]) and
 *      D_6_ab = u2_a*v2_b.  Residuals in pixels, on the compacted floats widened: with f = (T1^T Fn) T0 unscaled
 *      (T1^T as step 4), a0 = (f0*x0 + f1*y0) + f2, a1 = (f3*x0 + f4*y0) + f5, a2 = (f6*x0 + f7*y0) + f8,
 *      d = (x1*a0 + y1*a1) + a2, b0 = (f0*x1 + f3*y1) + f6, b1 = (f1*x1 + f4*y1) + f7,
 *      den = ((a0*a0 + a1*a1) + b0*b0) + b1*b1, err = (d*d) / den and r = d / sqrt(den): L7's Sampson error with F in
 *      place of E.  An inlier at this model has err < (double)thr2.  With g = (T1^T D_k) T0 and da, dd, db of g as a, d,
 *      b of f, dden = ((a0*da0 + a1*da1) + b0*db0) + b1*db1 and J_k = (dd - d*dden / den) / sqrt(den).  The 28 terms
 *      J_i*J_j (i <= j in row order) and the 7 terms J_i*r over the inliers, and the truncated cost (err for an inlier,
 *      else (double)thr2) over every point, are each summed in the order of step 2.  A step solves the 7x7 system of
 *      A7 (damping, Cholesky, right-hand side -J^T r), lambda starts at GEO_LO_LAMBDA0, and the step is taken only if
 *      the truncated cost at (U', V', sig'), with its own inliers, is strictly lower: A7's schedule.
 * LF8. Outputs: model the final F (a hypothesis's F of step 4, or T1^T Fn T0 scaled as step 4: rank 2, unit Frobenius
 *      norm, its first entry of largest magnitude positive); inliers the points with err < thr2 under it rounded to
 *      float (step 5's error), num_inliers their number and cost its LF3 score; best_hypothesis the hypothesis that
 *      seeded it; num_hypotheses the samples drawn.  A pair fails as step 7's failures (n < 8, a failed
 *      normalisation, every sample degenerate), with num_local_optimizations and cost 0.  Deviations from PoseLib:
 *      local optimisation runs at most once per chunk rather than at every new best, so the launch sequence is fixed
 *      and the result is deterministic; the score is quantised to integers; samples have 8 points rather than 7, so
 *      they are find_fundamental's; there is no non-minimal refit inside the LO, and no DEGENSAC or PROSAC.
 *
 * MAGSAC++ homography and fundamental matrix (geo_homography_magsac, geo_fundamental_magsac;
 * oracle/magsac_oracle.py restates them bit for bit): LH1-LH8 and LF1-LF8 with the truncated squared error replaced
 * by MAGSAC++'s loss marginalised over the noise scale sigma in [0, sigma_max] (Barath, Noskova, Ivashechkin and Matas,
 * CVPR 2020), nu = 4 degrees of freedom, and its local optimisation by iteratively reweighted least squares with the
 * weights of the same marginalisation.  threshold (thr2 = (float)(threshold * threshold)) keeps its meaning: it sets
 * the inliers, num_inliers and the count that drives stopping.  max_threshold = T = GEO_MAGSAC_K * sigma_max sets the
 * loss: mt2 = (float)(max_threshold * max_threshold), z = err / mt2.  With c = GEO_MAGSAC_K^2 / 2 and gamma_l, Gamma_u
 * the unnormalised lower and upper incomplete gamma functions, for z < 1
 *   rho(z) = [gamma_l(5/2, c z) + c z (Gamma_u(3/2, c z) - Gamma_u(3/2, c))] / gamma_l(5/2, c),
 *   w(z) = (Gamma_u(3/2, c z) - Gamma_u(3/2, c)) / (Gamma_u(3/2, 0) - Gamma_u(3/2, c)),
 * and rho = 1, w = 0 for z >= 1 or a non-finite err: rho rises from 0 to 1, w falls from 1 to 0, and w is
 * proportional to d rho / dz.  Neither is evaluated: both are the tables R and W of GEO_MAGSAC_KNOTS + 1 knots at
 * z = i / GEO_MAGSAC_KNOTS, the double literals of lightglue_b200/csrc/magsac_table.h (linear interpolation is within
 * 1.8e-6 of rho and 5.8e-5 of w), read by linear interpolation as below.
 *
 * MH1, MF1. As LH1 and LF1; mt2 as above.  M <= GEO_LO_MAX_MATCHES.
 * MH2, MF2. As LH2 and LF2: with the same seed, sample h and its hypothesis are LO's sample h.
 * MH3, MF3. Score, per hypothesis, from step 5's fp32 err (the model rounded to float): u = err * ks in fp32 with
 *      ks = (float)GEO_MAGSAC_KNOTS / mt2 (fp32 quotient); for u < GEO_MAGSAC_KNOTS, i = (int)u, f = u - (float)i,
 *      r = R'_i + f * (R'_(i+1) - R'_i) with R' = R rounded to float, and q = (uint32)fminf(r * GEO_LO_QSCALE,
 *      GEO_LO_QSCALE); otherwise (a NaN included) q = GEO_LO_QSCALE.  score = sum of q over the points in uint64,
 *      count = the number of err < thr2, packed as L3's count << 40 | score.  Since q <= GEO_LO_QSCALE, the bound
 *      GEO_LO_MAX_MATCHES holds.  Lower is better; ties go to the lowest h.
 * MH4, MF4. As LH4 and LF4 with MH3's score and MH7's LM.
 * MH5, MF5. As LH5 and LF5: stopping from the model's count at thr2.
 * MH6, MF6. As LH6 and LF6 with MH3's score and MH7's LM.
 * MH7, MF7. LM as LH7 and LF7 (parametrisation, residuals, Jacobians, damping, steps), on the MAGSAC++ cost: per point
 *      u = err * ((double)GEO_MAGSAC_KNOTS / (double)mt2); a point with u < GEO_MAGSAC_KNOTS has i = (int)u,
 *      f = u - (double)i, cost R_i + f * (R_(i+1) - R_i) and weight wt = W_i + f * (W_(i+1) - W_i) (double), and adds
 *      wt * (jx_i*jx_j + jy_i*jy_j) and wt * (jx_i*dx + jy_i*dy) (H) or wt * (J_i*J_j) and wt * (J_i*r) (F); any other
 *      point costs 1.0 and adds no terms.  So every point within T contributes, not only those within thr2.  The sums
 *      run in step 2's order and the step is taken only if the summed cost is strictly lower.
 * MH8, MF8. Outputs as LH8 and LF8 (inliers and num_inliers at thr2), cost the final model's MH3 / MF3 score.
 *
 * Absolute pose (geo_absolute_pose; oracle/pnp_oracle.py restates it bit for bit): the (R, t) of x_cam = R X + t that
 * maps the world points of image 1's keypoints into the query camera 0, OpenCV's rvec/tvec convention.  Expressions
 * below evaluate left to right as written (a + b + c is (a + b) + c); no step whose result must match bit for bit calls
 * cbrt, acos, atan2, sin, cos or pow: + - * / and sqrt round alike everywhere.
 *
 * A1. Compaction as step 1, where match i is valid when the pixel kpts0[b, i] has two and the float point
 *     X = points3d1[b, matches0[b, i]] has three finite coordinates.  Point k is the pixel (u, v) = kpts0[b, i_k] and the world point X_k, both float.
 * A2. Calibrated coordinates of the pixels through K0 as P1 (K0 checked as P1).  The solver reads them and the world
 *     points widened to double.
 * A3. Sampling as step 3 with s = 3.
 * A4. Lambda Twist P3P (Persson & Nordberg, ECCV 2018), in double.  Bearings y_k = (x, y, 1) / sqrt(x*x + y*y + 1.0);
 *     b12 = -2.0 * y0.y1, b13 = -2.0 * y0.y2, b23 = -2.0 * y1.y2 (a.b = a0*b0 + a1*b1 + a2*b2); d12 = X0 - X1,
 *     d13 = X0 - X2, d23 = X1 - X2, a12 = d12.d12, a13 = d13.d13, a23 = d23.d23, n = d12 x d13.  The sample is degenerate
 *     (collinear or coincident points) unless n.n > GEO_PNP_COLLINEAR_EPS * (a12 * a13).  With c31 = -0.5 * b13,
 *     c23 = -0.5 * b23, c12 = -0.5 * b12, blob = c12 * c23 * c31 - 1.0, sij = 1.0 - cij * cij:
 *       p3 = a13 * (a23 * s31 - a13 * s23)
 *       p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31
 *       p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23)
 *       p0 = a12 * (a12 * s23 - a23 * s12)
 *     h(g) = ((g + cb) * g + cc) * g + cd with cb = p2 / p3, cc = p1 / p3, cd = p0 / p3 (degenerate unless all finite).
 *     Root: rb = 1.0 + max(|cb|, |cc|, |cd|), bracket [-rb, rb]; when disc = cb * cb - 3.0 * cc >= 0, v = sqrt(disc),
 *     t1 = (-cb - v) / 3.0: [-rb, t1] if h(t1) > 0 (the leftmost root), else [(-cb + v) / 3.0, rb] (the rightmost).
 *     GEO_PNP_BISECT_STEPS bisections (mid = 0.5 * (lo + hi); hi = mid when h(mid) > 0, else lo = mid), then from
 *     g = 0.5 * (lo + hi) GEO_PNP_NEWTON_STEPS steps g - h(g) / ((3.0 * g + 2.0 * cb) * g + cc), a non-finite step
 *     leaving g.  Then A00 = a23 * (1.0 - g), A01 = a23 * b12 * 0.5, A02 = a23 * b13 * g * -0.5,
 *     A11 = a23 - a12 + a13 * g, A12 = b23 * (a13 * g - a12) * 0.5, A22 = g * (a13 - a23) - a12.
 *     root2(b, c): y = sqrt(fmax(b * b - 4.0 * c, 0.0)), q = -0.5 * (b + (b >= 0 ? y : -y)), roots (q, c / q).
 *     (e1, e2) = root2(-A00 - A11 - A22, -(A01 * A01) - A02 * A02 - A12 * A12 + A00 * (A11 + A22) + A11 * A22),
 *     swapped when |e1| < |e2|.  For e = e1, e2: tmp = 1.0 / (e * (A00 + A11) + mx - e * e + A01 * A01) with
 *     mx = -(A00 * A11), a1 = -(e * A02 + pr0) * tmp, a2 = -(e * A12 + pr1) * tmp with pr0 = A01 * A12 - A02 * A11,
 *     pr1 = A01 * A02 - A00 * A12, rn = 1.0 / sqrt(a1 * a1 + a2 * a2 + 1.0): the vectors v1 (of e1), v2 (of e2) =
 *     (a1 * rn, a2 * rn, rn).  sv = sqrt(fmax(0.0, -e2 / e1)).  For s = sv, then -sv: w2 = 1.0 / (s * v2_0 - v1_0),
 *     w0 = (v1_1 - s * v2_1) * w2, w1 = (v1_2 - s * v2_2) * w2,
 *       ia = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
 *       qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * ia
 *       qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * ia;
 *     when qb * qb - 4.0 * qc >= 0, for tau of root2(qb, qc) in order: with tau > 0, d = a23 / (tau * (b23 + tau) + 1.0)
 *     > 0, l2 = sqrt(d), l3 = tau * l2, l1 = w0 * l2 + w1 * l3 >= 0, the lambdas take GEO_PNP_GN_STEPS Gauss-Newton
 *     steps: r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12, r2 (l1, l3, b13, a13), r3 (l2, l3, b23, a23);
 *     v0 = 2.0 * l1 + b12 * l2, v1 = 2.0 * l2 + b12 * l1, v3 = 2.0 * l1 + b13 * l3, v5 = 2.0 * l3 + b13 * l1,
 *     v7 = 2.0 * l2 + b23 * l3, v8 = 2.0 * l3 + b23 * l2, det = -(v0 * v5 * v7) - v1 * v3 * v8,
 *     j0 = -(v5 * v7) * r1 - v1 * v8 * r2 + v1 * v5 * r3, j1 = -(v3 * v8) * r1 + v0 * v8 * r2 - v0 * v5 * r3,
 *     j2 = v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3, l_i = l_i - j_(i-1) / det unless a new l is non-finite.
 *     Pose: ry_k = y_k * l_k, e1 = ry0 - ry1, e2 = ry0 - ry2, e3 = e1 x e2; R_ij = e1_i * Xi_0j + e2_i * Xi_1j +
 *     e3_i * Xi_2j with Xi the inverse of [d12 d13 n] (columns) by cofactors (C_ij of row i, column j,
 *     det = x00 * C00 + x01 * C01 + x02 * C02, Xi_ij = C_ji / det); t_i = ry0_i - (R_i0 * X0_0 + R_i1 * X0_1 +
 *     R_i2 * X0_2).  A solution is kept when its R and t are finite; solution r is the r-th kept one, at most
 *     GEO_PNP_MAX_SOLUTIONS.  A sample without one is degenerate.
 * A5. Scoring in fp32 without fused multiply-adds, every solution of every sample: P = K0 [R | t], P_ij = K_i0 * M_0j +
 *     K_i1 * M_1j + K_i2 * M_2j in double with M = [R | t], rounded to float (p0..p11 row-major);
 *     w = p8 * X + p9 * Y + p10 * Z + p11, iw = 1 / w, du = u - (p0 * X + p1 * Y + p2 * Z + p3) * iw, dv likewise with
 *     p4..p7.  An inlier has w > 0 (in front of the camera) and du * du + dv * dv < (float)(threshold * threshold).
 *     Ties go to the lowest (sample h, solution r): the key packs ~(h*16 + r).  max_iters counts samples.
 * A6. Stopping as step 6 with s = 3.
 * A7. Refit.  With at least GEO_PNP_REFIT_MIN inliers, GEO_PNP_LM_STEPS Levenberg-Marquardt steps in double on the
 *     squared pixel error of the best solution's inliers, from that solution's (R, t); no convergence test.  At a pose,
 *     per inlier: Xc_i = R_i0 * X + R_i1 * Y + R_i2 * Z + t_i, iz = 1.0 / Xc2, a = Xc0 * iz, b = Xc1 * iz,
 *     pu = fx * a + s * b, ru = pu + cx - u, rv = fy * b + cy - v (fx = K0[0], s = K0[1], cx = K0[2], fy = K0[4],
 *     cy = K0[5]); gu = (fx * iz, s * iz, -(pu * iz)), gv = (0.0, fy * iz, -(fy * b * iz)); for g = gu, gv the Jacobian
 *     row (g2 * Xc1 - g1 * Xc2, g0 * Xc2 - g2 * Xc0, g1 * Xc0 - g0 * Xc1, g0, g1, g2) = ju, jv.  The 28 terms
 *     ju_i * ju_j + jv_i * jv_j (i <= j in row order), ju_i * ru + jv_i * rv and ru * ru + rv * rv are each summed over
 *     the points in the order of step 2, other points adding 0: H, g and the cost.  A step: H with its diagonal times
 *     (1.0 + lambda), Cholesky (for j: d = A_jj - L_j0^2 - ... left to right, failing unless d > 0, L_jj = sqrt(d),
 *     L_ij = (A_ij - L_i0 * L_j0 - ...) / L_jj for i > j), forward then back substitution for delta with right-hand
 *     side -g, failing on a non-finite delta.  q = (1.0, delta0 * 0.5, delta1 * 0.5, delta2 * 0.5) / sqrt(w*w + x*x +
 *     y*y + z*z), Q its rotation ([1.0 - 2.0 * (y*y + z*z), 2.0 * (x*y - w*z), 2.0 * (x*z + w*y)], [2.0 * (x*y + w*z),
 *     1.0 - 2.0 * (x*x + z*z), 2.0 * (y*z - w*x)], [2.0 * (x*z - w*y), 2.0 * (y*z + w*x), 1.0 - 2.0 * (x*x + y*y)]),
 *     R' = Q R (3x3 product as in step 4), t'_i = Q_i0 * t0 + Q_i1 * t1 + Q_i2 * t2 + delta_(3+i).  The step is taken
 *     only if the cost at (R', t') is strictly lower, then lambda = lambda / 10.0; a failed or rejected step sets
 *     lambda = lambda * 10.0.  lambda starts at GEO_PNP_LM_LAMBDA0.  The refit is re-scored as A5 and replaces the
 *     solution unless it has fewer inliers; inliers and num_inliers are the final pose's.
 * A8. A pair fails (success 0, R and t zero, no inliers, best_hypothesis = best_solution = -1, num_hypotheses the
 *     samples drawn) when n < 3, K0 is invalid, or every sample is degenerate.
 *
 * LO-RANSAC absolute pose (geo_absolute_pose_lo; oracle/lo_pnp_oracle.py restates it bit for bit): the outputs of
 * geo_absolute_pose, from an MSAC-scored P3P RANSAC with Levenberg-Marquardt local optimisation of (R, t), on the
 * schedule of L1-L8.  Expressions evaluate left to right as written; every multiply and add rounds on its own.
 *
 * LA1. Compaction, calibration, the K0 check and thr2 = (float)(threshold * threshold) exactly as A1-A2.
 *      M <= GEO_LO_MAX_MATCHES.
 * LA2. Sampling and the Lambda Twist solutions exactly as A3-A4: with the same seed both estimators draw the same
 *      samples and solve the same solutions.
 * LA3. MSAC score, per solution of every sample, from A5's fp32 test (P = K0 [R | t] rounded to float): err =
 *      du * du + dv * dv when w > 0, else the point is an outlier; q as L3 (0 at err == 0, else
 *      (uint32)fminf(err * w', GEO_LO_QSCALE) with w' = GEO_LO_QSCALE / thr2 for err < thr2, else GEO_LO_QSCALE), so a
 *      point behind the camera or with a non-finite err scores GEO_LO_QSCALE.  score = sum of q over the points in
 *      uint64, count = the number of inliers (A5's test).  Lower is better; ties go to the lowest (sample h,
 *      solution r).
 * LA4. Local optimisation, after every chunk of GEO_CHUNK samples, once per pair.  Chunk c's best solution (lowest
 *      (score, h, r)) is taken when the pair has no model yet or its score is strictly below the model's score; else
 *      nothing happens.  Taken, sample h is drawn and solved again as LA2, and the (R, t) of its solution r in double
 *      becomes the pair's model (score, count, h, r).  Then GEO_LO_STEPS LM steps (LA7) from it give (R', t'), which
 *      are scored as LA3 through P = K0 [R' | t'] rounded to float; with a strictly lower score they replace the model
 *      (keeping h and r) and num_local_optimizations counts one.
 * LA5. Stopping as A6 (s = 3) from the model's count (a local optimisation's count included).
 * LA6. Final refinement: GEO_LO_FINAL_STEPS LM steps from the model's (R, t), kept unless their LA3 score is higher.
 * LA7. LM, in double on the compacted pixels and world points read as floats widened: A7's parametrisation
 *      (R' = Q R, t'_i = Q_i0 * t0 + Q_i1 * t1 + Q_i2 * t2 + delta_(3+i)), residuals (ru, rv), err = ru * ru + rv * rv
 *      and Jacobian rows ju, jv at each pose.  A point is an inlier at this pose when Xc2 > 0 and err < (double)thr2.
 *      The 21 terms ju_i * ju_j + jv_i * jv_j (i <= j in row order) and the 6 terms ju_i * ru + jv_i * rv over the
 *      inliers, and the truncated cost (err for an inlier, else (double)thr2) over every point, are each summed in the
 *      order of step 2.  A step solves the 6x6 system of A7 (damping, Cholesky, right-hand side -J^T r), lambda starts
 *      at GEO_LO_LAMBDA0, and the step is taken only if the truncated cost at (R', t'), with its own inliers, is
 *      strictly lower: A7's schedule.
 * LA8. Outputs: R and t the final pose; inliers the rows that pass A5's test under its P = K0 [R | t] rounded to float,
 *      num_inliers their number and cost its LA3 score; best_hypothesis and best_solution the solution that seeded
 *      the final model; num_hypotheses the samples drawn.  A pair fails as A8, with num_local_optimizations and cost
 *      0.  Deviations from PoseLib and COLMAP: local optimisation runs at most once per chunk rather than at every new
 *      best, so the launch sequence is fixed and the result is deterministic; the score is quantised to integers;
 *      there is no non-minimal (EPnP) refit inside the LO and no PROSAC ordering.
 *
 * Affine and partial affine (geo_estimate_affine; oracle/affine_oracle.py restates it bit for bit): cv2.estimateAffine2D
 * (GEO_AFFINE, x1 = A x0 with A = [[a00, a01, a02], [a10, a11, a12]], 6 degrees of freedom) and
 * cv2.estimateAffinePartial2D (GEO_AFFINE_PARTIAL, A = [[a, -b, tx], [b, a, ty]]: rotation, uniform scale and
 * translation, 4 degrees of freedom) with method=RANSAC and refineIters.  Expressions evaluate left to right as written;
 * every multiply and add rounds on its own.
 *
 * AF1. Compaction and Hartley normalisation exactly as steps 1-2, with the same fixed-order sums.  The sample size is
 *      s = 3 (GEO_AFFINE) or s = 2 (GEO_AFFINE_PARTIAL).
 * AF2. Sampling as step 3 with that s.
 * AF3. Minimal solvers, in double, on the normalised coordinates (x, y) of image 0 and (u, v) of image 1, points in
 *      sample order.
 *      Affine: Cramer's rule on the differences to point 0: dxj = x1 - x0, dyj = y1 - y0, dxk = x2 - x0,
 *      dyk = y2 - y0, D = dxj*dyk - dxk*dyj, and likewise duj, dvj, duk, dvk of image 1.  The sample is rejected when
 *      the triple is collinear in either image by step 4's rule (|D| <= GEO_FLT_EPS * (((|dxj| + |dyj|) + |dxk|) +
 *      |dyk|), and the same with (duj, dvj, duk, dvk) and duj*dvk - duk*dvj: OpenCV's haveCollinearPoints).  Then
 *      a = (duj*dyk - duk*dyj) / D, b = (dxj*duk - dxk*duj) / D, c = u0 - (a*x0 + b*y0),
 *      d = (dvj*dyk - dvk*dyj) / D, e = (dxj*dvk - dxk*dvj) / D, f = v0 - (d*x0 + e*y0): An = [[a, b, c], [d, e, f],
 *      [0, 0, 1]].  The pixel model is T1^-1 An T0 by step 4's T0, T1^-1 and 3x3 products, whose bottom row is
 *      exactly (0, 0, 1); it is not rescaled.
 *      Partial: dx = x1 - x0, dy = y1 - y0, du = u1 - u0, dv = v1 - v0, dd = dx*dx + dy*dy.  The sample is degenerate
 *      when dd > 0 fails (coincident points in image 0) or du == 0 and dv == 0 (coincident points in image 1: a zero
 *      scale).  Else a = (dx*du + dy*dv) / dd, b = (dx*dv - dy*du) / dd, tx = u0 - (a*x0 - b*y0),
 *      ty = v0 - (b*x0 + a*y0).  T0 and T1 are isotropic, so the pixel model keeps the similarity form: with
 *      r = 1.0 / s1, kx = s0*cx0 and ky = s0*cy0, a' = (a*s0)*r, b' = (b*s0)*r,
 *      tx' = (tx - (a*kx - b*ky))*r + cx1, ty' = (ty - (b*kx + a*ky))*r + cy1, and A = [[a', -b', tx'], [b', a', ty']]
 *      with A[0][1] the exact negation of A[1][0] and A[1][1] a copy of A[0][0].
 *      Either kind: a sample whose normalised parameters or pixel model have a non-finite entry is degenerate.
 * AF4. Scoring as step 5's H error in fp32 on the model rounded to float with h6 = h7 = 0 and h8 = 1: then
 *      w = 1 / ((0*x0 + 0*y0) + 1) is exactly 1, so err = dx*dx + dy*dy with dx = x1 - ((a00*x0 + a01*y0) + a02),
 *      dy = y1 - ((a10*x0 + a11*y0) + a12), bit for bit.  An inlier has err < (float)(threshold * threshold).  The
 *      score is the inlier count; ties go to the lowest hypothesis.
 * AF5. Stopping as step 6 with s = 3 or 2.
 * AF6. Refinement.  With at least s inliers and refine_iters > 0, refine_iters Levenberg-Marquardt steps in double on
 *      the untruncated squared transfer error of the best hypothesis's inliers (its AF4 inliers, a fixed set), from
 *      its normalised parameters.  Per inlier, on the normalised coordinates of AF3: affine rx = ((a*x + b*y) + c) - u,
 *      ry = ((d*x + e*y) + f) - v, Jacobian rows jx = (x, y, 1, 0, 0, 0), jy = (0, 0, 0, x, y, 1); partial
 *      rx = ((a*x - b*y) + tx) - u, ry = ((b*x + a*y) + ty) - v, jx = (x, -y, 1, 0), jy = (y, x, 0, 1).  The terms
 *      jx_i*jx_j + jy_i*jy_j (i <= j in row order), jx_i*rx + jy_i*ry and rx*rx + ry*ry are each summed over the
 *      points in the order of step 2, other points adding 0: J^T J, J^T r and the cost.  A step solves A7's system
 *      (damping, Cholesky, right-hand side -J^T r; 6x6 or 4x4), moves the parameters to p + delta, and is taken only
 *      if the cost there is strictly lower; lambda starts at GEO_LO_LAMBDA0 and falls or rises tenfold: A7's
 *      schedule.  An isotropic T1 scales every residual by s1, so the minimiser is the pixel one; the residual is
 *      linear in the parameters, so the steps converge to the linear least-squares fit on those inliers.  The refined
 *      parameters give the pixel model as AF3, which is re-scored as AF4 and replaces the hypothesis unless it has
 *      fewer inliers.
 * AF7. Outputs: model [B, 3, 3] the final A with the bottom row (0, 0, 1); inliers the points with err < thr2 under it
 *      rounded to float, num_inliers their number; best_hypothesis the hypothesis the final model grew from;
 *      num_hypotheses the samples drawn.  A pair fails (success 0, model all zero, no inliers, best_hypothesis -1)
 *      when n < s, when its normalisation fails, or when every sample is degenerate.  Differences from OpenCV: inliers
 *      are those of the final (refined) model, where OpenCV returns the minimal model's mask; stopping is checked per
 *      chunk of GEO_CHUNK; the sampler is step 3's counter hash; there is no special case when n equals s; OpenCV's
 *      refinement is its own Levenberg-Marquardt solver on the same inliers, converging to the same least-squares fit.
 *
 * Lens distortion (geo_undistort_points, geo_distort_points; oracle/camera_oracle.py restates it bit for bit):
 * OpenCV's rational model with thin prism terms.  The coefficients are (k1, k2, p1, p2[, k3[, k4, k5, k6[, s1, s2, s3,
 * s4]]]): 4, 5, 8 or 12 of them, missing trailing ones zero.  COLMAP's SIMPLE_RADIAL (k), RADIAL (k1, k2), OPENCV
 * (k1, k2, p1, p2) and FULL_OPENCV (k1, k2, p1, p2, k3, k4, k5, k6) are special cases.  Expressions evaluate left to
 * right as written; every multiply and add rounds on its own.
 *
 * D1. Distort a normalised point (x, y): r2 = x*x + y*y, r4 = r2*r2, r6 = r4*r2, a1 = 2*x*y, a2 = r2 + 2*x*x,
 *     a3 = r2 + 2*y*y, cdist = 1 + k1*r2 + k2*r4 + k3*r6, icdist2 = 1 / (1 + k4*r2 + k5*r4 + k6*r6),
 *     xd = x*cdist*icdist2 + p1*a1 + p2*a2 + s1*r2 + s2*r4, yd = y*cdist*icdist2 + p1*a3 + p2*a1 + s3*r2 + s4*r4
 *     (cv2.projectPoints' formula).  geo_distort_points maps a pixel (u, v) to y = (v - cy) / fy,
 *     x = ((u - cx) - s*y) / fx (A2's rule), D1, and the pixel (fx*xd + s*yd + cx, fy*yd + cy).
 * D2. Undistort a pixel (u, v), OpenCV's fixed-point iteration as cv2.undistortPointsIter runs it:
 *     y0 = (v - cy) / fy, x0 = ((u - cx) - s*y0) / fx, (x, y) = (x0, y0), e = DBL_MAX.  Up to max_iters times: stop
 *     when e < eps; r2 = x*x + y*y, icdist = (1 + ((k6*r2 + k5)*r2 + k4)*r2) / (1 + ((k3*r2 + k2)*r2 + k1)*r2);
 *     when icdist < 0, (x, y) = (x0, y0) and stop; dx = 2*p1*x*y + p2*(r2 + 2*x*x) + s1*r2 + s2*r2*r2,
 *     dy = p1*(r2 + 2*y*y) + 2*p2*x*y + s3*r2 + s4*r2*r2, x = (x0 - dx)*icdist, y = (y0 - dy)*icdist; with eps > 0,
 *     (xd, yd) of D1 at (x, y), du = fx*xd + s*yd + cx - u, dv = fy*yd + cy - v and e = sqrt(du*du + dv*dv).  (eps = 0
 *     never stops early: e >= 0.)  The output pixel is (fx*x + s*y + cx, fy*y + cy), cv2.undistortPoints with P = K.
 *     OpenCV ignores the skew K[0][1] on input; with s = 0 the two agree.
 * D3. Validity.  K is valid as P1 states it; the coefficients when all are finite.  An invalid K or coefficients, or a
 *     non-finite input pixel, give a NaN output row, which every estimator here treats as an invalid match.  Inputs
 *     are float or double, read as double; outputs are computed in double and written in the input's type.
 *
 * Distortion-aware absolute pose (geo_absolute_pose_dist, geo_absolute_pose_lo_dist; oracle/pnp_dist_oracle.py
 * restates them bit for bit): cv2.solvePnPRansac with distCoeffs.  The minimal
 * solutions see undistorted bearings; the inlier test and Levenberg-Marquardt see distorted pixels.  Each step is A1-A8
 * (LA1-LA8 for the LO estimator) with these changes:
 *
 * AD1. Compaction as A1.  The calibrated coordinates that P3P reads are D2's (x, y) of the pixel with 5 iterations and
 *      eps = 0 (cv2.solvePnP inside cv2.solvePnPRansac), rounded to float.  Coefficients that fail D3 fail the pair as
 *      an invalid K0 does (A8).
 * AD2. The inlier test, in fp32 without fused multiply-adds, in distorted pixels: M = [R | t] rounded to float
 *      (m0..m11 row-major), Xc0 = m0*X + m1*Y + m2*Z + m3, Xc1 likewise with m4..m7, w = m8*X + m9*Y + m10*Z + m11;
 *      x = Xc0 / w, y = Xc1 / w; D1 in fp32 with K0 and the coefficients rounded to float; du = u - (fx*xd + s*yd + cx),
 *      dv = v - (fy*yd + cy).  An inlier has w > 0 and du*du + dv*dv < (float)(threshold * threshold).  The LO
 *      estimator's MSAC term reads this error as LA3 reads A5's (+inf behind the camera).
 * AD3. Levenberg-Marquardt (the refit of A7 and the LM of LA7), in double: Xc_i = R_i0*X + R_i1*Y + R_i2*Z + t_i,
 *      iz = 1.0 / Xc2, a = Xc0*iz, b = Xc1*iz, (xd, yd) of D1 at (a, b), ru = fx*xd + s*yd + cx - u,
 *      rv = fy*yd + cy - v.  D1's Jacobian at (a, b): r2 = a*a + b*b, r4 = r2*r2, id = 1.0 / (1.0 + k4*r2 + k5*r4 +
 *      k6*r2*r4), c = (1.0 + k1*r2 + k2*r4 + k3*r2*r4)*id, dc = (k1 + 2.0*k2*r2 + 3.0*k3*r4 - c*(k4 + 2.0*k5*r2 +
 *      3.0*k6*r4))*id, gx = s1 + 2.0*s2*r2, gy = s3 + 2.0*s4*r2, J00 = c + 2.0*a*(a*dc + gx) + 2.0*p1*b + 6.0*p2*a,
 *      J01 = 2.0*b*(a*dc + p2 + gx) + 2.0*p1*a, J10 = 2.0*a*(b*dc + p1 + gy) + 2.0*p2*b, J11 = c + 2.0*b*(b*dc + gy)
 *      + 6.0*p1*b + 2.0*p2*a.  With ua = fx*J00 + s*J10, ub = fx*J01 + s*J11, va = fy*J10, vb = fy*J11:
 *      gu = (ua*iz, ub*iz, -((ua*a + ub*b)*iz)), gv = (va*iz, vb*iz, -((va*a + vb*b)*iz)), and A7's Jacobian rows
 *      from gu and gv.  The refit's fixed inliers are those of AD2; LA7's inlier at a pose has Xc2 > 0 and
 *      ru*ru + rv*rv < (double)thr2.  The parametrisation, schedule and sums are A7's and LA7's.
 * AD4. Outputs, failures and diagnostics as A8 and LA8, with AD2's test in place of A5's.
 *
 * Fisheye camera (geo_fisheye_undistort_points, geo_fisheye_distort_points; oracle/fisheye_oracle.py restates it bit
 * for bit): cv2.fisheye's equidistant (Kannala-Brandt) model, COLMAP's OPENCV_FISHEYE.  The coefficients are D = (k1, k2,
 * k3, k4), exactly 4; the skew s = K[0][1] is OpenCV's alpha = s / fx.  Expressions evaluate left to right as written;
 * every multiply and add rounds on its own.  No step calls a library transcendental: atan and tan are FE1's.
 *
 * FE1. atan and tan, a range reduction and an odd polynomial p = t + t*(z*Q), z = t*t, Q = q0 + q1*z + ... by Horner
 *      from the last coefficient (acc = q_last, then acc = acc*z + q_i).  The constants and coefficients are the
 *      hexadecimal literals of lightglue_b200/csrc/fisheye_poly.h (generated by oracle/make_fisheye_poly.py).
 *      atan in double, a = |r|: when a > FE_TAN_3PI_8, FE_PI_2_HI + (FE_PI_2_LO + p(-1.0 / a)); else when
 *      a > FE_TAN_PI_8, FE_PI_4_HI + (FE_PI_4_LO + p((a - 1.0) / (a + 1.0))); else p(a); Q = FE_ATAN_D; negated for
 *      r < 0.  atan in float: when a > 1, FE_PI_2_HI_F + (FE_PI_2_LO_F + p(-1 / a)), else p(a); Q = FE_ATAN_F; negated
 *      for r < 0.  tan in double: n = rint(x * FE_2_PI) (ties to even), y = ((x - n*FE_PIO2_1) - n*FE_PIO2_2) -
 *      n*FE_PIO2_3, p(y) with Q = FE_TAN_D, and -1.0 / p when n is odd (floor(n * 0.5) != n * 0.5).  On [0, 1e6]
 *      the double atan is within 2 ulp of the correctly rounded value and the float one within 1 ulp; the double tan
 *      within 2 ulp on [0, pi/2).
 * FE2. Distort a normalised point (x, y), cv2.fisheye.distortPoints' model: r = sqrt(x*x + y*y), th = atan(r),
 *      t2 = th*th, t4 = t2*t2, t6 = t4*t2, t8 = t4*t4, thd = th*(1 + k1*t2 + k2*t4 + k3*t6 + k4*t8), cdist = thd / r
 *      when r > 1e-8, else 1; (xd, yd) = (cdist*x, cdist*y).  geo_fisheye_distort_points maps a pixel to (x, y) by
 *      D1's rule (skew included), FE2, and the pixel (fx*xd + s*yd + cx, fy*yd + cy).
 * FE3. Undistort a pixel (u, v), as cv2.fisheye.undistortPoints(pts, K, D, P=K, criteria) runs it: (x0, y0) by D2's
 *      rule (OpenCV ignores the skew on input; with s = 0 the two agree); thd = sqrt(x0*x0 + y0*y0), clamped to
 *      [-FE_PI_2_HI, FE_PI_2_HI]; th = thd.  With eps > 0 and |thd| <= eps the point converges with scale 0.  Otherwise
 *      up to max_iters times: t2 = th*th, t4 = t2*t2, t6 = t4*t2, t8 = t6*t2, a2 = k1*t2, a4 = k2*t4, a6 = k3*t6,
 *      a8 = k4*t8, fix = (th*(1 + a2 + a4 + a6 + a8) - thd) / (1 + 3*a2 + 5*a4 + 7*a6 + 9*a8), th = th - fix, and with
 *      eps > 0 the point converges and stops once |fix| < eps; then scale = tan(th) / thd.  The output is
 *      (scale*x0, scale*y0) through K as D2's.  A point fails when th and thd have opposite signs, or when eps > 0
 *      and it did not converge; its output row is NaN where OpenCV writes (-1e6, -1e6).  With eps = 0 the principal
 *      point is 0 / 0, NaN as in OpenCV.  eps is in radians of theta, not pixels.  The clamp is OpenCV's: a point
 *      whose thd exceeds pi/2 (beyond the model's 180 degree field) comes back at a plausible but wrong angle.
 * FE4. Validity.  K is valid as P1; the coefficients are exactly 4, all finite.  An invalid K or coefficients, a
 *      non-finite input pixel or a failing FE3 give a NaN output row.  Inputs and outputs as D3.
 *
 * Fisheye absolute pose (geo_absolute_pose_fisheye, geo_absolute_pose_lo_fisheye; oracle/fisheye_oracle.py restates
 * them bit for bit): cv2.solvePnPRansac with the fisheye camera, with the test and the refinement in fisheye pixels.
 * The minimal solutions see undistorted bearings; everything that scores or refines sees the fisheye image.  Each step
 * is A1-A8 (LA1-LA8 for the LO estimator) with these changes:
 *
 * AE1. Compaction as A1, with FE3's (x, y) at GEO_FISHEYE_ITERS and GEO_FISHEYE_EPS (cv2.fisheye.solvePnPRansac's
 *      default criteria), rounded to float, as the P3P input.  A match whose FE3 fails is invalid at compaction, as a
 *      NaN keypoint is: it is not counted in n, never sampled and never an inlier.  Coefficients that fail FE4 fail the
 *      pair as an invalid K0 does (A8).
 * AE2. The inlier test as AD2 with FE2 in fp32 in place of D1: the float atan of FE1, K0 and D rounded to float.  An
 *      inlier has w > 0 and du*du + dv*dv < (float)(threshold * threshold); the LO estimator's MSAC term reads this
 *      error, +inf behind the camera.
 * AE3. Levenberg-Marquardt as AD3 with FE2 in double in place of D1, and FE2's Jacobian at (a, b): r2 = a*a + b*b,
 *      r = sqrt(r2), th, t2..t8 and thd as FE2; when r > 1e-8, c = thd / r, dd = 1.0 + 3.0*k1*t2 + 5.0*k2*t4 +
 *      7.0*k3*t6 + 9.0*k4*t8 (d thd / d th), g = ((dd / (1.0 + r2) - c) / r) / r ((dc/dr) / r, with d th / d r =
 *      1 / (1 + r2)); else c = 1.0, g = 0.0.  ga = g*a, gb = g*b, J00 = c + ga*a, J01 = ga*b, J10 = gb*a,
 *      J11 = c + gb*b, chained onto A7's rows as AD3 chains D1's.
 * AE4. Outputs, failures and diagnostics as A8 and LA8, with AE2's test in place of A5's.
 *
 * 3D rigid and similarity transforms (geo_estimate_rigid; oracle/rigid_oracle.py restates it bit for bit): x1 = scale
 * R x0 + t between matched 3D points, with R a proper rotation and scale = 1 (GEO_RIGID_3D, SE(3)) or scale > 0
 * (GEO_SIMILARITY_3D, Sim(3)).  kpts0 and kpts1 of GeoInputs hold [B, M, 3] and [B, N, 3] points.  Expressions
 * evaluate left to right as written; every multiply and add rounds on its own.
 *
 * RG1. Compaction as step 1: match i is valid when 0 <= matches0[b, i] < N and all six coordinates of p =
 *      kpts0[b, i] and q = kpts1[b, matches0[b, i]] (float) are finite.  There is no normalisation: the solver centres
 *      its points.  The solver reads the floats widened to double.
 * RG2. Sampling as step 3 with s = 3.
 * RG3. Minimal solver, in double: Horn's closed-form quaternion method.  The sample is degenerate when either triangle
 *      p0 p1 p2 or q0 q1 q2 is collinear or coincident: with d1 = x1 - x0, d2 = x2 - x0, c = d1 x d2 (a x b =
 *      (a1*b2 - a2*b1, a2*b0 - a0*b2, a0*b1 - a1*b0)) and a.b = (a0*b0 + a1*b1) + a2*b2, unless
 *      c.c > GEO_RIGID_COLLINEAR_EPS * (d1.d1 * d2.d2).  Centroids in sample order, pb = ((p0 + p1) + p2) / 3.0 and qb
 *      likewise per coordinate; a_k = p_k - pb, b_k = q_k - qb; S_ij = sum_k a_k,i * b_k,j and saa = sum_k a_k.a_k,
 *      each summed over k = 0, 1, 2 from 0.0.  Then the closed form, shared with RG6, from (pb, qb, S, saa):
 *        N = [[(Sxx + Syy) + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
 *             [Syz - Szy, (Sxx - Syy) - Szz, Sxy + Syx, Szx + Sxz],
 *             [Szx - Sxz, Sxy + Syx, (Syy - Sxx) - Szz, Syz + Szy],
 *             [Sxy - Syx, Szx + Sxz, Syz + Szy, (Szz - Sxx) - Syy]]   (Sxy = S_01 and so on);
 *      v = the least eigenvector of -N (each entry negated) by step 7's cyclic Jacobi on a 4x4, the eigenvector of N's
 *      largest eigenvalue; nq = sqrt(((v0*v0 + v1*v1) + v2*v2) + v3*v3), (w, x, y, z) = v / nq; R = A7's rotation of
 *      that quaternion ([1.0 - 2.0 * (y*y + z*z), 2.0 * (x*y - w*z), 2.0 * (x*z + w*y)], ...).  Similarity:
 *      scale = num / saa with num = sum of R_ij * S_ji over i, then j, ascending from 0.0, which is
 *      sum_k b_k.(R a_k) (Umeyama's least-squares scale); rigid: scale = 1.0.  t_i = qb_i - scale *
 *      ((R_i0*pb0 + R_i1*pb1) + R_i2*pb2).  A scale that is not finite and positive, or a non-finite entry of R or t,
 *      makes the sample degenerate.  A unit quaternion's R is a proper rotation, so no reflection can arise.
 * RG4. Scoring in fp32 without fused multiply-adds: the model rounded to float as the 3x4 row-major [M | t] with
 *      M_ij = scale * R_ij (g0..g11); e_i = (((g_4i*x + g_4i+1*y) + g_4i+2*z) + g_4i+3) - q_i for p = (x, y, z),
 *      err = (e0*e0 + e1*e1) + e2*e2.  An inlier has err < (float)(threshold * threshold): the threshold is a distance
 *      in the units of kpts1.  The score is the inlier count; ties go to the lowest hypothesis.
 * RG5. Stopping as step 6 with s = 3.
 * RG6. Refit.  With at least 3 inliers, RG3's closed form on the inliers of the best hypothesis (its RG4 inliers, k
 *      of them), in two passes of step 2's fixed-order sums, other points adding 0: first pb_i = sum(p_i) / k and
 *      qb_i = sum(q_i) / k; then S_ij = sum(a_i * b_j) and saa = sum(a.a) with a = p - pb, b = q - qb.  The refit is
 *      scored as RG4 and replaces the hypothesis unless it has fewer inliers; a degenerate refit (RG3's rule) has none.
 *      The closed form is the least-squares fit on those inliers, so no iterative refinement follows.
 * RG7. Outputs: R [B, 3, 3], t [B, 3] and scale [B] of the final model (scale exactly 1.0 for GEO_RIGID_3D); inliers
 *      the points with err < thr2 under it rounded to float, num_inliers their number; best_hypothesis the hypothesis
 *      the final model grew from; num_hypotheses the samples drawn.  A pair fails (success 0, R, t and scale zero, no
 *      inliers, best_hypothesis -1) when n < 3 or when every sample is degenerate.  Differences from the usual tools:
 *      inliers are those of the final (refitted) model; stopping is checked per chunk of GEO_CHUNK; the sampler is
 *      step 3's counter hash.  On a fixed inlier set the fit equals Umeyama's (and, for Sim(3),
 *      cv2.estimateAffine3D(src, dst, force_rotation=True)).
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
#define GEO_ESSENTIAL 2       /* the relative pose's model, for geo_relative_pose */
#define GEO_MAX_SOLUTIONS 10
#define GEO_LEAD_EPS 1e-12
#define GEO_STURM_STEPS 40
#define GEO_NEWTON_STEPS 8
#define GEO_REFIT_MIN 8

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

typedef struct GeoPoseConfig {
  int32_t abi_version;        /* GEO_ABI_VERSION */
  int32_t max_iters;          /* samples per pair, in [1, GEO_MAX_ITERS] */
  uint32_t seed;
  int32_t reserved;
  double threshold;           /* pixels, > 0: Sampson distance, divided by the pair's mean focal length */
  double confidence;          /* in [0, 1] */
  double distance_threshold;  /* > 0: triangulated depth bound of the cheirality test */
} GeoPoseConfig;

typedef struct GeoPoseInputs {
  int32_t B, M, N;
  const float* kpts0;      /* [B, M, 2] */
  const float* kpts1;      /* [B, N, 2] */
  const int64_t* matches0; /* [B, M]; indices outside [0, N) are unmatched */
  const double* K0;        /* [B, 9] row-major intrinsics of image 0 */
  const double* K1;        /* [B, 9] of image 1 */
} GeoPoseInputs;

typedef struct GeoPoseOutputs {
  double* E;                 /* [B, 3, 3] */
  double* R;                 /* [B, 3, 3] */
  double* t;                 /* [B, 3], unit */
  uint8_t* inliers;          /* [B, M] */
  int32_t* num_inliers;      /* [B] */
  uint8_t* pose_inliers;     /* [B, M] inliers that pass the chosen pose's cheirality test */
  int32_t* num_pose_inliers; /* [B] */
  uint8_t* success;          /* [B] */
  int32_t* best_hypothesis;  /* [B], -1 without one */
  int32_t* best_solution;    /* [B], -1 without one */
  int32_t* num_hypotheses;   /* [B] */
} GeoPoseOutputs;

LG_API size_t geo_pose_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_relative_pose(const GeoPoseConfig* cfg, const GeoPoseInputs* in, GeoPoseOutputs* out, void* workspace,
                             size_t workspace_bytes, void* stream);

#define GEO_LO_QSCALE 65536
#define GEO_LO_STEPS 8
#define GEO_LO_FINAL_STEPS 16
#define GEO_LO_LAMBDA0 1e-3
#define GEO_LO_MAX_MATCHES ((1 << 20) - 1) /* M bound: QSCALE * M < 2^36 fits the 36 score bits of the (score, h) key */

typedef struct GeoLoPoseConfig {
  int32_t abi_version;        /* GEO_ABI_VERSION */
  int32_t max_iters;          /* samples per pair, in [1, GEO_MAX_ITERS] */
  uint32_t seed;
  int32_t reserved;
  double threshold;           /* pixels, > 0: Sampson distance, divided by the pair's mean focal length */
  double confidence;          /* in [0, 1] */
  double distance_threshold;  /* > 0: triangulated depth bound of the cheirality test */
} GeoLoPoseConfig;

typedef struct GeoLoPoseOutputs {
  GeoPoseOutputs pose;               /* as geo_relative_pose's */
  int32_t* num_local_optimizations;  /* [B] local optimisations whose model was adopted */
  int64_t* cost;                     /* [B] L3 score of the final model */
} GeoLoPoseOutputs;

LG_API size_t geo_lo_pose_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_relative_pose_lo(const GeoLoPoseConfig* cfg, const GeoPoseInputs* in, GeoLoPoseOutputs* out,
                                void* workspace, size_t workspace_bytes, void* stream);

typedef struct GeoLoOutputs {
  GeoOutputs geo;                    /* as geo_estimate's; model is H or F */
  int32_t* num_local_optimizations;  /* [B] local optimisations whose model was adopted */
  int64_t* cost;                     /* [B] LH3 or LF3 score of the final model */
} GeoLoOutputs;

/* LO-RANSAC homography (steps LH1-LH8): cfg->model must be GEO_HOMOGRAPHY, in->M <= GEO_LO_MAX_MATCHES. */
LG_API size_t geo_lo_homography_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_homography_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                             size_t workspace_bytes, void* stream);

/* LO-RANSAC fundamental matrix (steps LF1-LF8): cfg->model must be GEO_FUNDAMENTAL, in->M <= GEO_LO_MAX_MATCHES. */
LG_API size_t geo_lo_fundamental_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_fundamental_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                              size_t workspace_bytes, void* stream);

#define GEO_MAGSAC_KNOTS 1024             /* intervals of the loss and weight tables (lightglue_b200/csrc/magsac_table.h) */
#define GEO_MAGSAC_K 3.6437211935036444   /* k = sqrt(chi2_0.99(4)): max_threshold = k * sigma_max */

typedef struct GeoMagsacConfig {
  GeoConfig geo;         /* as geo_homography_lo's and geo_fundamental_lo's; threshold sets the inliers and the count */
  double max_threshold;  /* T, pixels, finite and > 0: the scale of the MAGSAC++ loss and weights */
} GeoMagsacConfig;

/* MAGSAC++ homography (steps MH1-MH8): cfg->geo.model must be GEO_HOMOGRAPHY, in->M <= GEO_LO_MAX_MATCHES.  The
 * workspace is geo_lo_homography_workspace_bytes'. */
LG_API int geo_homography_magsac(const GeoMagsacConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* MAGSAC++ fundamental matrix (steps MF1-MF8): cfg->geo.model must be GEO_FUNDAMENTAL, in->M <= GEO_LO_MAX_MATCHES.
 * The workspace is geo_lo_fundamental_workspace_bytes'. */
LG_API int geo_fundamental_magsac(const GeoMagsacConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                  size_t workspace_bytes, void* stream);

#define GEO_PNP_MAX_SOLUTIONS 4
#define GEO_PNP_COLLINEAR_EPS 1e-10
#define GEO_PNP_BISECT_STEPS 60
#define GEO_PNP_NEWTON_STEPS 4
#define GEO_PNP_GN_STEPS 3
#define GEO_PNP_LM_STEPS 10
#define GEO_PNP_LM_LAMBDA0 1e-3
#define GEO_PNP_REFIT_MIN 6

typedef struct GeoPnpConfig {
  int32_t abi_version; /* GEO_ABI_VERSION */
  int32_t max_iters;   /* samples per pair, in [1, GEO_MAX_ITERS] */
  uint32_t seed;
  int32_t reserved;
  double threshold;    /* pixels, > 0: reprojection error in image 0 */
  double confidence;   /* in [0, 1] */
} GeoPnpConfig;

typedef struct GeoPnpInputs {
  int32_t B, M, N;
  const float* kpts0;      /* [B, M, 2] query pixels */
  const float* points3d1;  /* [B, N, 3] world point of each keypoint of image 1; a non-finite coordinate: none */
  const int64_t* matches0; /* [B, M]; indices outside [0, N) are unmatched */
  const double* K0;        /* [B, 9] row-major intrinsics of image 0 */
} GeoPnpInputs;

typedef struct GeoPnpOutputs {
  double* R;                /* [B, 3, 3] world to camera: x_cam = R X + t */
  double* t;                /* [B, 3] */
  uint8_t* inliers;         /* [B, M] */
  int32_t* num_inliers;     /* [B] */
  uint8_t* success;         /* [B] */
  int32_t* best_hypothesis; /* [B], -1 without one */
  int32_t* best_solution;   /* [B], -1 without one */
  int32_t* num_hypotheses;  /* [B] */
} GeoPnpOutputs;

LG_API size_t geo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_absolute_pose(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoPnpOutputs* out, void* workspace,
                             size_t workspace_bytes, void* stream);

typedef struct GeoLoPnpOutputs {
  GeoPnpOutputs pnp;                 /* as geo_absolute_pose's */
  int32_t* num_local_optimizations;  /* [B] local optimisations whose model was adopted */
  int64_t* cost;                     /* [B] LA3 score of the final model */
} GeoLoPnpOutputs;

/* LO-RANSAC absolute pose (steps LA1-LA8): in->M <= GEO_LO_MAX_MATCHES. */
LG_API size_t geo_lo_pnp_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_absolute_pose_lo(const GeoPnpConfig* cfg, const GeoPnpInputs* in, GeoLoPnpOutputs* out,
                                void* workspace, size_t workspace_bytes, void* stream);

#define GEO_CAMERA_FLOAT32 0
#define GEO_CAMERA_FLOAT64 1
#define GEO_UNDISTORT_MAX_ITERS 1000

typedef struct GeoCameraConfig {
  int32_t abi_version; /* GEO_ABI_VERSION */
  int32_t num_dist;    /* coefficients per pair: 4, 5, 8 or 12 */
  int32_t max_iters;   /* D2's iterations, in [0, GEO_UNDISTORT_MAX_ITERS]; geo_distort_points ignores it */
  int32_t dtype;       /* GEO_CAMERA_FLOAT32 or GEO_CAMERA_FLOAT64: the type of in->pts and out->pts */
  double eps;          /* D2's reprojection stop in pixels, finite and >= 0; 0: none */
} GeoCameraConfig;

typedef struct GeoCameraInputs {
  int32_t B, N;
  const void* pts;     /* [B, N, 2] pixels */
  const double* K;     /* [B, 9] row-major intrinsics */
  const double* dist;  /* [B, num_dist] */
} GeoCameraInputs;

typedef struct GeoCameraOutputs {
  void* pts;           /* [B, N, 2] pixels, the input's type */
} GeoCameraOutputs;

/* Lens distortion (steps D1-D3): one launch, B <= 65535, no workspace. */
LG_API int geo_undistort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                void* stream);
LG_API int geo_distort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                              void* stream);

typedef struct GeoPnpDistInputs {
  GeoPnpInputs pnp;        /* as geo_absolute_pose's */
  int32_t num_dist;        /* 4, 5, 8 or 12; 4 for the fisheye entry points */
  const double* dist0;     /* [B, num_dist] distortion coefficients of image 0 */
} GeoPnpDistInputs;

/* Distortion-aware absolute pose (steps AD1-AD4); the workspaces are geo_pnp_workspace_bytes' and
 * geo_lo_pnp_workspace_bytes'. */
LG_API int geo_absolute_pose_dist(const GeoPnpConfig* cfg, const GeoPnpDistInputs* in, GeoPnpOutputs* out,
                                  void* workspace, size_t workspace_bytes, void* stream);
LG_API int geo_absolute_pose_lo_dist(const GeoPnpConfig* cfg, const GeoPnpDistInputs* in, GeoLoPnpOutputs* out,
                                     void* workspace, size_t workspace_bytes, void* stream);

#define GEO_FISHEYE_ITERS 10 /* FE3's iterations in cv2.fisheye's default criteria */
#define GEO_FISHEYE_EPS 1e-8 /* FE3's stop in those criteria, radians of theta */

/* Fisheye camera (steps FE1-FE4), on the structs of the lens distortion: cfg->num_dist must be 4, cfg->max_iters is
 * FE3's in [0, GEO_UNDISTORT_MAX_ITERS] and cfg->eps FE3's stop in radians of theta (not pixels), finite and >= 0
 * (0: none, OpenCV's COUNT-only criterion); geo_fisheye_distort_points ignores both.  One launch, B <= 65535, no
 * workspace. */
LG_API int geo_fisheye_undistort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                        void* stream);
LG_API int geo_fisheye_distort_points(const GeoCameraConfig* cfg, const GeoCameraInputs* in, GeoCameraOutputs* out,
                                      void* stream);

/* Fisheye absolute pose (steps AE1-AE4): in->num_dist must be 4; the workspaces are geo_pnp_workspace_bytes' and
 * geo_lo_pnp_workspace_bytes'. */
LG_API int geo_absolute_pose_fisheye(const GeoPnpConfig* cfg, const GeoPnpDistInputs* in, GeoPnpOutputs* out,
                                     void* workspace, size_t workspace_bytes, void* stream);
LG_API int geo_absolute_pose_lo_fisheye(const GeoPnpConfig* cfg, const GeoPnpDistInputs* in, GeoLoPnpOutputs* out,
                                        void* workspace, size_t workspace_bytes, void* stream);

#define GEO_RIGID_3D 5
#define GEO_SIMILARITY_3D 6
#define GEO_RIGID_COLLINEAR_EPS 1e-10

typedef struct GeoRigidOutputs {
  double* R;                /* [B, 3, 3] proper rotation: x1 = scale R x0 + t */
  double* t;                /* [B, 3] */
  double* scale;            /* [B]; exactly 1.0 for GEO_RIGID_3D */
  uint8_t* inliers;         /* [B, M] */
  int32_t* num_inliers;     /* [B] */
  uint8_t* success;         /* [B] */
  int32_t* best_hypothesis; /* [B], -1 without one */
  int32_t* num_hypotheses;  /* [B] */
} GeoRigidOutputs;

/* 3D rigid and similarity transforms (steps RG1-RG7): cfg->model is GEO_RIGID_3D or GEO_SIMILARITY_3D and
 * cfg->threshold a distance in the units of the points; in->kpts0 and in->kpts1 hold [B, M, 3] and [B, N, 3] points. */
LG_API size_t geo_rigid_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_estimate_rigid(const GeoConfig* cfg, const GeoInputs* in, GeoRigidOutputs* out, void* workspace,
                              size_t workspace_bytes, void* stream);

#define GEO_AFFINE 3
#define GEO_AFFINE_PARTIAL 4
#define GEO_AFFINE_MAX_REFINE 100

typedef struct GeoAffineConfig {
  int32_t abi_version;  /* GEO_ABI_VERSION */
  int32_t model;        /* GEO_AFFINE or GEO_AFFINE_PARTIAL */
  int32_t max_iters;    /* hypotheses per pair, in [1, GEO_MAX_ITERS] */
  uint32_t seed;
  int32_t refine_iters; /* Levenberg-Marquardt steps, in [0, GEO_AFFINE_MAX_REFINE]; 0: none */
  int32_t reserved;
  double threshold;     /* pixels, > 0: transfer error */
  double confidence;    /* in [0, 1] */
} GeoAffineConfig;

/* Affine and partial affine (steps AF1-AF7): out->model is [B, 3, 3] with the bottom row (0, 0, 1). */
LG_API size_t geo_affine_workspace_bytes(int32_t B, int32_t M, int32_t max_iters);
LG_API int geo_estimate_affine(const GeoAffineConfig* cfg, const GeoInputs* in, GeoOutputs* out, void* workspace,
                               size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
