// Batched LO-RANSAC homography and fundamental matrix on the matcher's output: MSAC-scored four-point (H) or
// eight-point (F) sampling with Levenberg-Marquardt local optimisation and a final refinement (include/geometry_b200.h,
// steps LH1-LH8 and LF1-LF8).  H is refined at unit norm in the tangent space of the sphere, F at rank 2 in its
// orthonormal representation (U, V, sigma).  Both run on lo_common.cuh's schedule: geo_api.cu's compaction and
// Hartley normalisation kernel prepares the pair; geo_hyp_kernel makes step 4's minimal solve, one model per sample
// (r = 0); a local optimisation starts from the hypothesis solved again in double and runs LM on the truncated
// transfer (H) or Sampson (F) cost.  The MAGSAC++ estimators (MH1-MH8, MF1-MF8) are the same models and schedule
// over lo_common.cuh's Magsac loss: the sigma-marginalised score, and LM weighted by its IRLS weights.  Compiled with
// -fmad=false: oracle/lo_homography_oracle.py, oracle/lo_fundamental_oracle.py and oracle/magsac_oracle.py take the
// same steps.
#include <stdint.h>

#include "geo_hf.cuh"
#include "lg_internal.h"
#include "lo_common.cuh"

namespace {

// The chunk's LH3 / LF3 scores, count << 40 | MSAC score
template <int KIND>
struct LoHfScore {
  using Args = LoArgs<GeoArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = 1, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const GeoWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  float thr2, w;
  __device__ LoHfScore(const Args& a, const GeoPair&, int b)
      : src{a.p.w.pts + (long)b * a.p.M}, sums(a.l.acc), thr2(a.p.thr2), w((float)GEO_LO_QSCALE / a.p.thr2) {}
  __device__ unsigned long long term(const float* h, const float4* p) const {
    return lo_term(geo_err(KIND, h, p[0]), thr2, w);
  }
};

// The MAGSAC++ estimators' arguments: GeoArgs and T^2
struct MagsacArgs : GeoArgs {
  float mt2;
};

__global__ void __launch_bounds__(1024) magsac_prepare_kernel(MagsacArgs a) { geo_prepare(a); }

// The chunk's MH3 / MF3 scores, count << 40 | MAGSAC++ score
template <int KIND>
struct MagsacHfScore {
  using Args = LoArgs<MagsacArgs>;
  using Acc = unsigned long long;
  static constexpr int SOLS = 1, NF = 9, K = 1, TILE = ::TILE;
  static __device__ const GeoWs& ws(const Args& a) { return a.p.w; }
  const float4* src[K];
  unsigned long long* sums;
  Magsac::Term q;
  __device__ MagsacHfScore(const Args& a, const GeoPair&, int b)
      : src{a.p.w.pts + (long)b * a.p.M}, sums(a.l.acc), q(Magsac{a.p.thr2, a.p.mt2}.term()) {}
  __device__ unsigned long long term(const float* h, const float4* p) const { return q(geo_err(KIND, h, p[0])); }
};

// The loss of each argument type: MSAC at thr2 for LO-RANSAC, MAGSAC++ at mt2 (counting at thr2) for MAGSAC++
__device__ __forceinline__ Msac hf_loss(const GeoArgs& p) { return {p.thr2}; }
__device__ __forceinline__ Magsac hf_loss(const MagsacArgs& p) { return {p.thr2, p.mt2}; }

// T1^-1 X T0 (H) or (T1^T X) T0 (F), unscaled: the first half of denormalise
template <int KIND>
__device__ void to_pixels(const GeoPair& P, const double* X, double* out) {
  double L[9];
  if (KIND == GEO_HOMOGRAPHY) {
    const double r = 1.0 / P.s1;
    const double Li[9] = {r, 0.0, P.cx1, 0.0, r, P.cy1, 0.0, 0.0, 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Li[i];
  } else {
    const double Lt[9] = {P.s1, 0.0, 0.0, 0.0, P.s1, 0.0, -(P.s1 * P.cx1), -(P.s1 * P.cy1), 1.0};
    for (int i = 0; i < 9; ++i) L[i] = Lt[i];
  }
  const double T0[9] = {P.s0, 0.0, -(P.s0 * P.cx0), 0.0, P.s0, -(P.s0 * P.cy0), 0.0, 0.0, 1.0};
  double tmp[9];
  mm3(L, X, tmp);
  mm3(tmp, T0, out);
}

// The columns j != m of the Householder reflection I - (2 / v.v) v v^T, v = e_m - Hn, which maps e_m to Hn: an
// orthonormal basis of the tangent space of the unit sphere at Hn (header step LH7)
__device__ void householder_basis(const double* Hn, double (*B)[9]) {
  int m = 0;
  for (int i = 1; i < 9; ++i)
    if (fabs(Hn[i]) < fabs(Hn[m])) m = i;
  double v[9], vv = 0.0;
  for (int i = 0; i < 9; ++i) v[i] = (i == m ? 1.0 : 0.0) - Hn[i];
  for (int i = 0; i < 9; ++i) vv = vv + v[i] * v[i];
  const double c = 2.0 / vv;
  for (int j = 0, k = 0; j < 9; ++j) {
    if (j == m) continue;
    for (int i = 0; i < 9; ++i) B[k][i] = (i == j ? 1.0 : 0.0) - c * v[i] * v[j];
    ++k;
  }
}

// The schedule hooks of the homography and the fundamental matrix (lo_common.cuh), Model one of the two and Base its
// arguments (GeoArgs or MagsacArgs): L.model is the scaled pixel model, the LM start Model::start of it
template <class Model, class B>
struct HfLo {
  using Base = B;
  using Args = LoArgs<B>;
  using Solver = HfSolver;
  static constexpr int SOLS = 1;

  static __device__ const float4* points(const Args& a, int b) { return a.p.w.pts + (long)b * a.p.M; }
  static __device__ const GeoPair& consts(const Args& a, int b) { return a.p.w.pair[b]; }
  static __device__ auto loss(const Args& a, int) { return hf_loss(a.p); }

  // LH4 / LF4: hypothesis h solved again in double
  static __device__ void seed(LoShared<Model>& s, const Args& a, int b, unsigned hr, long, LoPair& L, int t) {
    if (t == 0) {
      HfSolver::solve(a.p, b, hr >> 4, (double(*)[9])L.model);
      Model::start(s, a.p.w.pair[b], L.model);
    }
  }

  static __device__ void store(LoShared<Model>& s, LoPair& L) {
    for (int i = 0; i < 9; ++i) L.model[i] = s.px[i];
  }

  static __device__ void load(LoShared<Model>& s, const Args& a, int b, const LoPair& L, int t) {
    if (t == 0) Model::start(s, a.p.w.pair[b], L.model);
  }

  static __device__ void restore(LoShared<Model>& s, const Args&, int, const LoPair& L, int t) {
    if (t == 0) {
      for (int i = 0; i < 9; ++i) {
        s.px[i] = L.model[i];
        s.fm[i] = (float)L.model[i];
      }
      s.score = (unsigned long long)L.count * LO_COUNT_ONE + L.score;
    }
    __syncthreads();
  }

  static __device__ void fail(const Args& a, int b, int t) {
    if (t < 9) a.p.out.model[(long)b * 9 + t] = 0.0;
  }

  // LH8 / LF8: the model and its inliers
  static __device__ void write(LoShared<Model>& s, const Args& a, int b, int t) {
    const float4* pts = points(a, b);
    const int* idx = a.p.w.idx + (long)b * a.p.M;
    uint8_t* inl = a.p.out.inliers + (long)b * a.p.M;
    for (int i = t; i < a.p.M; i += RED) inl[i] = 0;
    __syncthreads();
    for (int k = t; k < a.p.w.pair[b].n; k += RED)
      if (Model::err(s.fm, pts[k]) < a.p.thr2) inl[idx[k]] = 1;
    if (t < 9) a.p.out.model[(long)b * 9 + t] = s.px[t];
  }
};

// The policies of a loss: MSAC on GeoArgs with LoHfScore, MAGSAC++ on MagsacArgs with MagsacHfScore
template <class Loss>
struct HfLoss;
template <>
struct HfLoss<Msac> {
  using Base = GeoArgs;
  template <int KIND>
  using Score = LoHfScore<KIND>;
};
template <>
struct HfLoss<Magsac> {
  using Base = MagsacArgs;
  template <int KIND>
  using Score = MagsacHfScore<KIND>;
};

// The homography for lo_common.cuh's LM loop, re-score and schedule over Loss, Self the estimator: x = Hn, the
// unit-norm normalised model (header steps LH7 and MH7)
template <class Self, class Loss>
struct HomographyModel : HfLo<Self, typename HfLoss<Loss>::Base> {
  static constexpr int KIND = GEO_HOMOGRAPHY, S = 4, DOF = 8, TERMS = 45, GROUP = 15, NP = 9, NF = 9;
  using Score = typename HfLoss<Loss>::template Score<KIND>;
  struct Scratch {
    double basis[DOF][9];     // tangent basis at the model being summed or updated
    double Hu[9], G[DOF][9];  // T1^-1 Hn T0 and its derivatives along the basis
  };

  // Hn = T1 H T0^-1 at unit Frobenius norm of a pixel H; thread 0 only
  static __device__ void start(LoShared<Self>& s, const GeoPair& P, const double* H) {
    const double T1[9] = {P.s1, 0.0, -(P.s1 * P.cx1), 0.0, P.s1, -(P.s1 * P.cy1), 0.0, 0.0, 1.0};
    const double r = 1.0 / P.s0;
    const double T0i[9] = {r, 0.0, P.cx0, 0.0, r, P.cy0, 0.0, 0.0, 1.0};
    double tmp[9];
    mm3(T1, H, tmp);
    mm3(tmp, T0i, s.x);
    double f = 0.0;
    for (int i = 0; i < 9; ++i) f = f + s.x[i] * s.x[i];
    f = sqrt(f);
    for (int i = 0; i < 9; ++i) s.x[i] = s.x[i] / f;
  }

  static __device__ void terms(LoShared<Self>& s, const GeoPair& P, const double* X, const float4* pts, int n,
                               double scale, double* out, int tid) {
    if (tid == 0) {
      householder_basis(X, s.m.basis);
      to_pixels<KIND>(P, X, s.m.Hu);
      for (int k = 0; k < DOF; ++k) to_pixels<KIND>(P, s.m.basis[k], s.m.G[k]);
    }
    __syncthreads();
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    const double* h = s.m.Hu;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts[k];
      const double x = p.x, y = p.y, u = p.z, v = p.w;
      const double w = 1.0 / ((h[6] * x + h[7] * y) + h[8]);
      const double px = ((h[0] * x + h[1] * y) + h[2]) * w, py = ((h[3] * x + h[4] * y) + h[5]) * w;
      const double dx = u - px, dy = v - py;
      const double err = dx * dx + dy * dy;
      double cost, wt;
      const bool in = Loss::point(scale, err, cost, wt);
      acc[TERMS - 1] = acc[TERMS - 1] + cost;
      if (!in) continue;
      double jx[DOF], jy[DOF];
#pragma unroll
      for (int q = 0; q < DOF; ++q) {
        const volatile double* g = s.m.G[q];  // re-read per point: held in registers, the 72 entries spill
        const double da = (g[0] * x + g[1] * y) + g[2], db = (g[3] * x + g[4] * y) + g[5];
        const double dc = (g[6] * x + g[7] * y) + g[8];
        jx[q] = -((da - px * dc) * w);
        jy[q] = -((db - py * dc) * w);
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + Loss::weigh(wt, jx[i] * jx[j] + jy[i] * jy[j]);
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[36 + i] = acc[36 + i] + Loss::weigh(wt, jx[i] * dx + jy[i] * dy);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // X' = normalize(X + sum_k d_k basis_k), the basis taken at X
  static __device__ void update(LoShared<Self>& s, const double* X, const double* d, double* out) {
    householder_basis(X, s.m.basis);
    double f = 0.0;
    for (int i = 0; i < 9; ++i) {
      double v = X[i];
      for (int k = 0; k < DOF; ++k) v = v + d[k] * s.m.basis[k][i];
      out[i] = v;
      f = f + v * v;
    }
    f = sqrt(f);
    for (int i = 0; i < 9; ++i) out[i] = out[i] / f;
  }

  static __device__ void pixels(LoShared<Self>&, const GeoPair& P, const double* X, double* out) {
    denormalise(KIND, P, X, out);
  }

  static __device__ __forceinline__ float err(const float* h, float4 p) { return geo_err(KIND, h, p); }
};

struct HomographyLo : HomographyModel<HomographyLo, Msac> {};
struct HomographyMagsac : HomographyModel<HomographyMagsac, Magsac> {};

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Fn_ab = u1_a*v1_b + sig*u2_a*v2_b of x = (U, V, sig)
__device__ void compose(const double* x, double* Fn) {
  const double* U = x;
  const double* V = x + 9;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) Fn[a * 3 + b] = U[a * 3] * V[b * 3] + x[18] * U[a * 3 + 1] * V[b * 3 + 1];
}

// The fundamental matrix for lo_common.cuh's LM loop, re-score and schedule over Loss, Self the estimator: x = U (0-8),
// V (9-17) and sig (18), the orthonormal representation Fn = u1 v1^T + sig u2 v2^T of the normalised model, u_k, v_k
// columns of U, V (header steps LF7 and MF7)
template <class Self, class Loss>
struct FundamentalModel : HfLo<Self, typename HfLoss<Loss>::Base> {
  static constexpr int KIND = GEO_FUNDAMENTAL, S = 8, DOF = 7, TERMS = 36, GROUP = 18, NP = 19, NF = 9;
  using Score = typename HfLoss<Loss>::template Score<KIND>;
  struct Scratch {
    double Fu[9], G[DOF][9];  // T1^T Fn T0 and the directions at Fn in pixels
  };

  // x of a pixel F: Fn = (T1^-T F) T0^-1, then U, V and sig by step 4's one-sided Jacobi; thread 0 only
  static __device__ void start(LoShared<Self>& s, const GeoPair& P, const double* F) {
    const double r1 = 1.0 / P.s1, r0 = 1.0 / P.s0;
    const double T1it[9] = {r1, 0.0, 0.0, 0.0, r1, 0.0, P.cx1, P.cy1, 1.0};
    const double T0i[9] = {r0, 0.0, P.cx0, 0.0, r0, P.cy0, 0.0, 0.0, 1.0};
    double tmp[9], A[9], W[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    mm3(T1it, F, tmp);
    mm3(tmp, T0i, A);
    jacobi_columns3(A, W);
    double nrm[3];
    int m = 0;
    for (int j = 0; j < 3; ++j) {
      double nj = 0.0;
      for (int i = 0; i < 3; ++i) nj = nj + A[i * 3 + j] * A[i * 3 + j];
      nrm[j] = nj;
      if (nj < nrm[m]) m = j;
    }
    int p = m == 0 ? 1 : 0, q = m == 2 ? 1 : 2;
    if (nrm[q] > nrm[p]) {
      const int t = p;
      p = q;
      q = t;
    }
    const double s1 = sqrt(nrm[p]), s2 = sqrt(nrm[q]);
    double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
    for (int r = 0; r < 3; ++r) {
      u1[r] = A[r * 3 + p] / s1;
      u2[r] = A[r * 3 + q] / s2;
      v1[r] = W[r * 3 + p];
      v2[r] = W[r * 3 + q];
    }
    cross3(u1, u2, u3);
    cross3(v1, v2, v3);
    double* U = s.x;
    double* V = s.x + 9;
    for (int r = 0; r < 3; ++r) {
      U[r * 3] = u1[r]; U[r * 3 + 1] = u2[r]; U[r * 3 + 2] = u3[r];
      V[r * 3] = v1[r]; V[r * 3 + 1] = v2[r]; V[r * 3 + 2] = v3[r];
    }
    s.x[18] = s2 / s1;
  }

  static __device__ void terms(LoShared<Self>& s, const GeoPair& P, const double* X, const float4* pts, int n,
                               double scale, double* out, int tid) {
    if (tid == 0) {
      double Fn[9], D[9];
      compose(X, Fn);
      to_pixels<KIND>(P, Fn, s.m.Fu);
      for (int k = 0; k < 3; ++k) {
        const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
        double w[3], c[3];
        for (int j = 0; j < 3; ++j) {  // [e_k]x Fn: column j is e_k x Fn[:, j]
          for (int i = 0; i < 3; ++i) w[i] = Fn[i * 3 + j];
          cross3(e, w, c);
          for (int i = 0; i < 3; ++i) D[i * 3 + j] = c[i];
        }
        to_pixels<KIND>(P, D, s.m.G[k]);
        for (int i = 0; i < 3; ++i) cross3(e, Fn + i * 3, D + i * 3);  // -Fn [e_k]x: row i is e_k x Fn[i, :]
        to_pixels<KIND>(P, D, s.m.G[3 + k]);
      }
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) D[a * 3 + b] = X[a * 3 + 1] * X[9 + b * 3 + 1];
      to_pixels<KIND>(P, D, s.m.G[6]);
    }
    __syncthreads();
    double acc[TERMS];
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc[i] = 0.0;
    const double* f = s.m.Fu;
    for (int k = tid; k < n; k += RED) {
      const float4 p = pts[k];
      const double x = p.x, y = p.y, u = p.z, v = p.w;
      const double a0 = (f[0] * x + f[1] * y) + f[2], a1 = (f[3] * x + f[4] * y) + f[5];
      const double a2 = (f[6] * x + f[7] * y) + f[8];
      const double d = (u * a0 + v * a1) + a2;
      const double b0 = (f[0] * u + f[3] * v) + f[6], b1 = (f[1] * u + f[4] * v) + f[7];
      const double den = ((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1;
      const double err = (d * d) / den;
      double cost, wt;
      const bool in = Loss::point(scale, err, cost, wt);
      acc[TERMS - 1] = acc[TERMS - 1] + cost;
      if (!in) continue;
      const double sq = sqrt(den), r = d / sq;
      double J[DOF];
#pragma unroll
      for (int q = 0; q < DOF; ++q) {
        const volatile double* g = s.m.G[q];  // re-read per point, as the homography's LM does
        const double da0 = (g[0] * x + g[1] * y) + g[2], da1 = (g[3] * x + g[4] * y) + g[5];
        const double da2 = (g[6] * x + g[7] * y) + g[8];
        const double dd = (u * da0 + v * da1) + da2;
        const double db0 = (g[0] * u + g[3] * v) + g[6], db1 = (g[1] * u + g[4] * v) + g[7];
        const double dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1;
        J[q] = (dd - d * dden / den) / sq;
      }
      int e = 0;
#pragma unroll
      for (int i = 0; i < DOF; ++i)
#pragma unroll
        for (int j = i; j < DOF; ++j, ++e) acc[e] = acc[e] + Loss::weigh(wt, J[i] * J[j]);
#pragma unroll
      for (int i = 0; i < DOF; ++i) acc[28 + i] = acc[28 + i] + Loss::weigh(wt, J[i] * r);
    }
    lo_tree_sums<TERMS, GROUP>(acc, s.red, out, tid);
  }

  // U' = Q(d0..2) U, V' = Q(d3..5) V, sig' = sig + d6
  static __device__ void update(LoShared<Self>&, const double* X, const double* d, double* out) {
    double Q[9];
    quat_rotation(d, Q);
    mm3(Q, X, out);
    quat_rotation(d + 3, Q);
    mm3(Q, X + 9, out + 9);
    out[18] = X[18] + d[6];
  }

  static __device__ void pixels(LoShared<Self>&, const GeoPair& P, const double* X, double* out) {
    double Fn[9];
    compose(X, Fn);
    denormalise(KIND, P, Fn, out);
  }

  static __device__ __forceinline__ float err(const float* h, float4 p) { return geo_err(KIND, h, p); }
};

struct FundamentalLo : FundamentalModel<FundamentalLo, Msac> {};
struct FundamentalMagsac : FundamentalModel<FundamentalMagsac, Magsac> {};

// geo_homography_lo and geo_fundamental_lo (GeoArgs from a GeoConfig), geo_homography_magsac and
// geo_fundamental_magsac (MagsacArgs from a GeoMagsacConfig): name for the error strings
template <class Model, class Extra>
int lohf_estimate(const char* name, const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                  size_t workspace_bytes, void* stream_, typename Model::Base g, void (*prepare)(typename Model::Base),
                  Extra extra) {
  int rc = geo_check_config(name, cfg, in, out, GEO_LO_MAX_MATCHES, [&] {
    return cfg->model == Model::KIND          ? nullptr
           : Model::KIND == GEO_HOMOGRAPHY ? "model must be GEO_HOMOGRAPHY"
                                           : "model must be GEO_FUNDAMENTAL";
  }, extra);
  if (rc == GEO_RUN) {
    const GeoOutputs& o = out->geo;
    rc = geo_check_buffers(name, in, {o.model, o.num_inliers, o.success, o.best_hypothesis, o.num_hypotheses,
                                      out->num_local_optimizations, out->cost}, {o.inliers}, {}, in->kpts1,
                           workspace, workspace_bytes, lo_workspace_bytes<Model>(in->B, in->M));
  }
  if (rc != GEO_RUN) return rc;
  g.B = in->B; g.M = in->M; g.N = in->N;
  g.kind = Model::KIND;
  g.s = Model::S;
  g.max_iters = cfg->max_iters;
  g.chunks = geo_chunks(cfg->max_iters);
  g.seed = cfg->seed;
  g.thr2 = (float)(cfg->threshold * cfg->threshold);
  g.confidence = cfg->confidence;
  g.kpts0 = in->kpts0; g.kpts1 = in->kpts1; g.matches0 = in->matches0;
  g.out = out->geo;
  return lo_launch<Model>(g, out->num_local_optimizations, out->cost, workspace, prepare, stream_);
}

template <class Model>
int lohf_lo(const char* name, const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
            size_t workspace_bytes, void* stream) {
  return lohf_estimate<Model>(name, cfg, in, out, workspace, workspace_bytes, stream, GeoArgs{}, geo_prepare_kernel,
                              geo_no_check);
}

// The MAGSAC++ entry points: the checks of the LO ones, with max_threshold's at the place of distance() in
// geo_check_config.  The carve is LO-RANSAC's (MagsacArgs holds the same GeoWs), so the workspace sizes are
// geo_lo_homography_workspace_bytes' and geo_lo_fundamental_workspace_bytes'.
template <class Model>
int lohf_magsac(const char* name, const GeoMagsacConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                size_t workspace_bytes, void* stream) {
  if (!cfg) return geo_error(name, "null argument");
  const double T = cfg->max_threshold;
  MagsacArgs g{};
  g.mt2 = (float)(T * T);
  return lohf_estimate<Model>(name, &cfg->geo, in, out, workspace, workspace_bytes, stream, g, magsac_prepare_kernel,
                              [T]() -> const char* {
                                return T > 0.0 && isfinite(T) ? nullptr : "max_threshold must be positive";
                              });
}

}  // namespace

extern "C" size_t geo_lo_homography_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lo_workspace_bytes<HomographyLo>(B, M);
}

extern "C" size_t geo_lo_fundamental_workspace_bytes(int32_t B, int32_t M, int32_t) {
  return lo_workspace_bytes<FundamentalLo>(B, M);
}

extern "C" int geo_homography_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return lohf_lo<HomographyLo>("geo_homography_lo", cfg, in, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_fundamental_lo(const GeoConfig* cfg, const GeoInputs* in, GeoLoOutputs* out, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return lohf_lo<FundamentalLo>("geo_fundamental_lo", cfg, in, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_homography_magsac(const GeoMagsacConfig* cfg, const GeoInputs* in, GeoLoOutputs* out,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  return lohf_magsac<HomographyMagsac>("geo_homography_magsac", cfg, in, out, workspace, workspace_bytes, stream);
}

extern "C" int geo_fundamental_magsac(const GeoMagsacConfig* cfg, const GeoInputs* in, GeoLoOutputs* out,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  return lohf_magsac<FundamentalMagsac>("geo_fundamental_magsac", cfg, in, out, workspace, workspace_bytes, stream);
}
