// Object detection by 2D-2D matching on the GPU: the reference's LocalFeatureObjectDetector.detect_by_matching
// (local_feature_2D_detector.py:76-147) after its matcher, for B frames against V reference views, without leaving the device.
//   cv2.estimateAffinePartial2D(from, to, RANSAC, ...)         calib3d/src/ptsetreg.cpp                 opb_estimate_affine_partial
//   match_worker + detect_by_matching: per-view match count,   local_feature_2D_detector.py:76-147      opb_boxes_from_matches
//   the view with the most matches, its affine and box
//   the same for (frame, object) pairs, each object's views       DESIGN 5.8                               opb_boxes_from_matches_objects
//   a range of one table of every object's views
//
// The estimator is OpenCV's, stage for stage (the model is tests/affine_ransac_reference.py):
//   samples   cv::RNG((uint64)-1) and getSubset with 2 model points (cv_rng.cuh, the generator of the EPnP loop);
//   model     AffinePartial2DEstimatorCallback::runKernel: the closed-form 2-pair similarity in fp64 from the fp32 points;
//   count     Affine2DEstimatorCallback::computeError: the model rounded to fp32, a = ((F0 x + F1 y) + F2) - X in fp32, a^2 + b^2
//             <= (float)(thr * thr);
//   loop      a win is a count strictly above max(best, 1), then RANSACUpdateNumIters(confidence, outlier ratio, 2, budget);
//             the loop exits at iter >= budget;
//   refine    the winner's inliers, OpenCV's LMSolver on (a, b, tx, ty) (AffinePartial2DRefineCallback) in fp64, its
//             damping schedule and its eigen-decomposition solve (lm_refine).
// Every product and sum of the model and the count is rounded on its own (__dmul_rn, __fadd_rn, ...), so nothing is contracted
// into a fused multiply-add: the samples' models are cv2's bit for bit and the counts exact.  The refinement's reductions run in
// a fixed order (not OpenCV's), so the refined model agrees with cv2's to rounding (DESIGN 5.8).
//
// One block per problem.  Warp 0 draws 32 samples at a time; the block's 8 warps evaluate them, one sample per warp and the
// pairs across its lanes; thread 0 then runs the loop's bookkeeping over the 32 counts in sample order.  Samples past the loop's
// exit are drawn and counted but never read, so the results do not depend on the wave size.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "block.cuh"
#include "cv_rng.cuh"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kAffThreads = 256;
constexpr int kAffWarps = kAffThreads / 32;
constexpr int kAffWave = 32;               // samples per round: one warp_draw call
constexpr int kModelPoints = 2;
constexpr int kMinMatches = 6;             // match_worker: a view with fewer matches gets no affine
constexpr int kMaxViews = 256;
constexpr int kMaxRefPoints = 8192;        // the winning view's pairs live in shared memory, 16 bytes each
constexpr float kFltEps = FLT_EPSILON;     // LMSolver's epsx and epsf

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

struct Pair {
  float x, y, X, Y;                        // from (x, y) -> to (X, Y)
};

struct GlobalPairs {                       // ragged problems: from / to fp32 [n, 2]
  const float* from;
  const float* to;
  __device__ Pair operator()(int i) const {
    const float2 f = __ldg(reinterpret_cast<const float2*>(from) + i), t = __ldg(reinterpret_cast<const float2*>(to) + i);
    return {f.x, f.y, t.x, t.y};
  }
};

struct SharedPairs {                       // the winning view's compacted pairs
  const float4* p;
  __device__ Pair operator()(int i) const {
    const float4 v = p[i];
    return {v.x, v.y, v.z, v.w};
  }
};

struct AffineParams {
  float thr2;                              // (float)(threshold * threshold), as findInliers rounds it
  int max_iters;
  double confidence;
  int refine_iters;
};

struct AffineTrace {                       // test hook: per problem, samples [cap][2], counts [cap], models [cap][6]
  int* samples;
  int* counts;
  double* models;
  int cap;
  __device__ AffineTrace at(int b) const {
    return {samples ? samples + (size_t)b * cap * 2 : nullptr, counts ? counts + (size_t)b * cap : nullptr,
            models ? models + (size_t)b * cap * 6 : nullptr, cap};
  }
};

// AffinePartial2DEstimatorCallback::runKernel on pairs p, q: M row-major 2x3 = [S0 -S1 S2; S1 S0 S3]
__device__ void two_point_model(const Pair& p, const Pair& q, double* M) {
  const double x1 = p.x, y1 = p.y, x2 = q.x, y2 = q.y, X1 = p.X, Y1 = p.Y, X2 = q.X, Y2 = q.Y;
  const double dx = sub(x1, x2), dy = sub(y1, y2), DX = sub(X1, X2), DY = sub(Y1, Y2);
  const double d = __ddiv_rn(1.0, add(mul(dx, dx), mul(dy, dy)));
  const double c = sub(mul(x1, y2), mul(x2, y1));
  const double S0 = mul(d, add(mul(DX, dx), mul(DY, dy)));
  const double S1 = mul(d, sub(mul(DY, dx), mul(DX, dy)));
  const double S2 = mul(d, sub(sub(mul(DY, c), mul(sub(mul(X1, y2), mul(X2, y1)), dy)), mul(sub(mul(X1, x2), mul(X2, x1)), dx)));
  const double S3 = mul(d, sub(sub(mul(-DX, c), mul(sub(mul(Y1, x2), mul(Y2, x1)), dx)), mul(sub(mul(Y1, y2), mul(Y2, y1)), dy)));
  M[0] = S0; M[1] = -S1; M[2] = S2;
  M[3] = S1; M[4] = S0; M[5] = S3;
}

// Affine2DEstimatorCallback::computeError of one pair under the fp32-rounded model F
__device__ __forceinline__ float cv_error(const float* F, const Pair& p) {
  const float a = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(F[0], p.x), __fmul_rn(F[1], p.y)), F[2]), p.X);
  const float b = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(F[3], p.x), __fmul_rn(F[4], p.y)), F[5]), p.Y);
  return __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
}

__device__ __forceinline__ void to_f32(const double* M, float* F) {
#pragma unroll
  for (int k = 0; k < 6; ++k) F[k] = __double2float_rn(M[k]);
}

constexpr int kSums = 9;                   // the first reduction's sums; one max (the largest residual) follows them

struct AffShared {
  int samples[kAffWave * kModelPoints];
  int counts[kAffWave];
  int first, niters, best, win0, win1, done, iter, go;
  double red[kAffWarps][kSums + 1];
  double xd[4];
  double H[6];                             // the result: the model (zeros for none)
  int status;                              // 1: a model, 0: none
};

// v[0 .. N) summed and v[N] maximised (fmax: a NaN is passed over) over the block in a fixed order (lanes by shuffle, then
// warps in index order); thread 0 gets the totals
template <int N>
__device__ void block_reduce(double* v, AffShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k <= N; ++k)
    for (int o = 16; o; o >>= 1) {
      const double u = __shfl_down_sync(0xffffffffu, v[k], o);
      v[k] = k < N ? v[k] + u : fmax(v[k], u);
    }
  if (lane == 0)
    for (int k = 0; k <= N; ++k) sh.red[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k <= N; ++k) {
      double s = sh.red[0][k];
      for (int w = 1; w < kAffWarps; ++w) s = k < N ? s + sh.red[w][k] : fmax(s, sh.red[w][k]);
      v[k] = s;
    }
}

// AffinePartial2DRefineCallback's residuals of pair p at h = (a, b, tx, ty): xi - X, yi - Y
__device__ __forceinline__ void residual(const double* h, const Pair& p, double& r0, double& r1) {
  const double Mx = p.x, My = p.y;
  r0 = sub(add(sub(mul(h[0], Mx), mul(h[1], My)), h[2]), (double)p.X);
  r1 = sub(add(add(mul(h[1], Mx), mul(h[0], My)), h[3]), (double)p.Y);
}

// cv::eigen of the symmetric 4x4 matrix a as OpenCV's JacobiImpl_ runs it: rotations at the largest off-diagonal |a_kl| (found
// through per-row and per-column maxima) until it is <= DBL_EPSILON or after 30 n^2 rotations, then the eigenvalues w in
// descending order with the eigenvectors as the rows of V.  a is overwritten.
__device__ void jacobi4(double (*a)[4], double* w, double (*V)[4]) {
  constexpr int n = 4;
  int ind_r[n], ind_c[n];
  auto row_max = [&](int k) {
    int m = k + 1;
    for (int i = k + 2; i < n; ++i) m = fabs(a[k][m]) < fabs(a[k][i]) ? i : m;
    return m;
  };
  auto col_max = [&](int k) {
    int m = 0;
    for (int i = 1; i < k; ++i) m = fabs(a[m][k]) < fabs(a[i][k]) ? i : m;
    return m;
  };
  for (int k = 0; k < n; ++k) {
    w[k] = a[k][k];
    for (int c = 0; c < n; ++c) V[k][c] = k == c ? 1.0 : 0.0;
    ind_r[k] = k < n - 1 ? row_max(k) : 0;
    ind_c[k] = k > 0 ? col_max(k) : 0;
  }
  for (int iter = 0; iter < 30 * n * n; ++iter) {
    int k = 0, l = ind_r[0];
    double mv = fabs(a[0][ind_r[0]]);
    for (int i = 1; i < n - 1; ++i)
      if (mv < fabs(a[i][ind_r[i]])) { mv = fabs(a[i][ind_r[i]]); k = i; l = ind_r[i]; }
    for (int i = 1; i < n; ++i)
      if (mv < fabs(a[ind_c[i]][i])) { mv = fabs(a[ind_c[i]][i]); k = ind_c[i]; l = i; }
    const double p = a[k][l];
    if (fabs(p) <= DBL_EPSILON) break;
    const double y = mul(sub(w[l], w[k]), 0.5);
    double t = add(fabs(y), hypot(p, y));
    double s = hypot(p, t);
    const double c = __ddiv_rn(t, s);
    s = __ddiv_rn(p, s);
    t = mul(__ddiv_rn(p, t), p);
    if (y < 0) { s = -s; t = -t; }
    a[k][l] = 0.0;
    w[k] = sub(w[k], t);
    w[l] = add(w[l], t);
    auto rot = [&](double& v0, double& v1) {
      const double a0 = v0, b0 = v1;
      v0 = sub(mul(a0, c), mul(b0, s));
      v1 = add(mul(a0, s), mul(b0, c));
    };
    for (int i = 0; i < k; ++i) rot(a[i][k], a[i][l]);
    for (int i = k + 1; i < l; ++i) rot(a[k][i], a[i][l]);
    for (int i = l + 1; i < n; ++i) rot(a[k][i], a[l][i]);
    for (int i = 0; i < n; ++i) rot(V[k][i], V[l][i]);
    for (int idx : {k, l}) {
      if (idx < n - 1) ind_r[idx] = row_max(idx);
      if (idx > 0) ind_c[idx] = col_max(idx);
    }
  }
  for (int k = 0; k < n - 1; ++k) {
    int m = k;
    for (int i = k + 1; i < n; ++i) m = w[m] < w[i] ? i : m;
    if (m != k) {
      const double t = w[k]; w[k] = w[m]; w[m] = t;
      for (int i = 0; i < n; ++i) { const double u = V[k][i]; V[k][i] = V[m][i]; V[m][i] = u; }
    }
  }
}

// SVBkSb's rule: eigenvalue i counts when |w_i| > 2 DBL_EPSILON * sum(w); the others are dropped (a pseudo-inverse)
__device__ __forceinline__ double kept_bound(const double* w) { return mul(add(add(add(w[0], w[1]), w[2]), w[3]), 2.0 * DBL_EPSILON); }

// cv::solve(a, v, d, DECOMP_EIG): d = sum over the kept eigenpairs of V_i (V_i . v) / w_i, in eigenvalue order.  a is overwritten.
__device__ void eig_solve4(double (*a)[4], const double* v, double* d) {
  double w[4], V[4][4];
  jacobi4(a, w, V);
  const double bound = kept_bound(w);
  for (int j = 0; j < 4; ++j) d[j] = 0.0;
  for (int i = 0; i < 4; ++i) {
    if (fabs(w[i]) <= bound) continue;
    double s = 0.0;
    for (int j = 0; j < 4; ++j) s = add(s, mul(V[i][j], v[j]));
    s = mul(s, __ddiv_rn(1.0, w[i]));
    for (int j = 0; j < 4; ++j) d[j] = add(d[j], mul(s, V[i][j]));
  }
}

// max |diag(cv::invert(a, DECOMP_EIG))|, the pseudo-inverse over the kept eigenpairs.  a is overwritten.
__device__ double eig_inverse_diag_max(double (*a)[4]) {
  double w[4], V[4][4], diag[4] = {0.0, 0.0, 0.0, 0.0};
  jacobi4(a, w, V);
  const double bound = kept_bound(w);
  for (int i = 0; i < 4; ++i) {
    if (fabs(w[i]) <= bound) continue;
    const double r = __ddiv_rn(1.0, w[i]);
    for (int j = 0; j < 4; ++j) diag[j] = add(diag[j], mul(V[i][j], mul(r, V[i][j])));
  }
  return fmax(fmax(fabs(diag[0]), fabs(diag[1])), fmax(fabs(diag[2]), fabs(diag[3])));
}

// OpenCV's LMSolver (calib3d/src/levmarq.cpp, eps = FLT_EPSILON) on h = (a, b, tx, ty) over the pairs `inlier` accepts.
// J^T J does not depend on h: rows (x, -y, 1, 0) and (y, x, 0, 1); D is its diagonal.  From lambda = 1 and lc = 0.75, each
// iteration solves (J^T J + lambda D) d = J^T r by eigen decomposition (eig_solve4) and tries h - d.  With the predicted
// decrease dS = d . (2 J^T r - J^T J d) and R = (S - Sd) / dS (dS taken as 1 where |dS| <= DBL_EPSILON): R > 0.75 halves
// lambda, to 0 once it drops below lc; R < 0.25 multiplies it by nu = clamp((Sd - S) / (d . J^T r) + 2, 2, 10), and from
// lambda = 0 first sets lambda = lc = 1 / max |diag((J^T J)^+)| and halves nu.  The step is kept when Sd < S.  Every iteration
// counts; the loop stops after max_iters, or when |d|_inf < eps or when every residual |r_i| of the kept model is below eps
// (not S < eps^2, which takes more steps on sub-pixel fits; tests/affine_ransac_reference.py's lm_refine, the schedule cv2
// 4.13 runs).  h: the same in every thread on entry, the result in thread 0 on exit.
template <class Pairs, class Inlier>
__device__ void lm_refine(const Pairs& P, int n, Inlier inlier, int max_iters, double* h, AffShared& sh) {
  const int tid = threadIdx.x;
  double s[kSums + 1];
  for (int k = 0; k <= kSums; ++k) s[k] = 0.0;
  for (int j = tid; j < n; j += kAffThreads) {        // sums of 1, x, y, x^2 + y^2; then the error and J^T r at h; max |r_i|
    const Pair p = P(j);
    if (!inlier(p)) continue;
    const double Mx = p.x, My = p.y;
    double r0, r1;
    residual(h, p, r0, r1);
    s[0] += 1.0; s[1] += Mx; s[2] += My; s[3] += Mx * Mx + My * My;
    s[4] += r0 * r0 + r1 * r1;
    s[5] += Mx * r0 + My * r1; s[6] += Mx * r1 - My * r0; s[7] += r0; s[8] += r1;
    s[9] = fmax(s[9], fmax(fabs(r0), fabs(r1)));
  }
  block_reduce<kSums>(s, sh);
  double A[4][4], v[4], S = 0.0, rmax = 0.0, lambda = 1.0, lc = 0.75;
  int it = 0;
  if (tid == 0) {
    const double A0[4][4] = {{s[3], 0.0, s[1], s[2]}, {0.0, s[3], -s[2], s[1]}, {s[1], -s[2], s[0], 0.0}, {s[2], s[1], 0.0, s[0]}};
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) A[r][c] = A0[r][c];
    S = s[4];
    rmax = s[9];
    for (int k = 0; k < 4; ++k) v[k] = s[5 + k];
  }
  while (true) {
    double d[4], dmax = 0.0;
    if (tid == 0) {
      double Ap[4][4];
      for (int r = 0; r < 4; ++r) {
        for (int c = 0; c < 4; ++c) Ap[r][c] = A[r][c];
        Ap[r][r] = add(Ap[r][r], mul(lambda, A[r][r]));
      }
      eig_solve4(Ap, v, d);
      for (int k = 0; k < 4; ++k) {
        sh.xd[k] = h[k] - d[k];
        dmax = fmax(dmax, fabs(d[k]));
        if (isnan(d[k])) dmax = NAN;
      }
    }
    __syncthreads();
    const double xd[4] = {sh.xd[0], sh.xd[1], sh.xd[2], sh.xd[3]};
    double t[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = tid; j < n; j += kAffThreads) {
      const Pair p = P(j);
      if (!inlier(p)) continue;
      const double Mx = p.x, My = p.y;
      double r0, r1;
      residual(xd, p, r0, r1);
      t[0] += r0 * r0 + r1 * r1;
      t[1] += Mx * r0 + My * r1; t[2] += Mx * r1 - My * r0; t[3] += r0; t[4] += r1;
      t[5] = fmax(t[5], fmax(fabs(r0), fabs(r1)));
    }
    block_reduce<5>(t, sh);
    if (tid == 0) {
      const double Sd = t[0];
      double dS = 0.0, dv = 0.0;
      for (int r = 0; r < 4; ++r) {
        double Ad = 0.0;
        for (int c = 0; c < 4; ++c) Ad = add(Ad, mul(A[r][c], d[c]));
        dS = add(dS, mul(d[r], sub(mul(2.0, v[r]), Ad)));
        dv = add(dv, mul(d[r], v[r]));
      }
      const double R = __ddiv_rn(sub(S, Sd), fabs(dS) > DBL_EPSILON ? dS : 1.0);
      if (R > 0.75) {
        lambda *= 0.5;
        if (lambda < lc) lambda = 0.0;
      } else if (R < 0.25) {
        double nu = fmin(fmax(add(__ddiv_rn(sub(Sd, S), fabs(dv) > DBL_EPSILON ? dv : 1.0), 2.0), 2.0), 10.0);
        if (lambda == 0.0) {
          double Ai[4][4];
          for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) Ai[r][c] = A[r][c];
          lambda = lc = __ddiv_rn(1.0, fmax(DBL_EPSILON, eig_inverse_diag_max(Ai)));
          nu *= 0.5;
        }
        lambda = mul(lambda, nu);
      }
      if (Sd < S) {
        S = Sd;
        rmax = t[5];
        for (int k = 0; k < 4; ++k) { h[k] = xd[k]; v[k] = t[1 + k]; }
      }
      ++it;
      sh.go = it < max_iters && dmax >= (double)kFltEps && rmax >= (double)kFltEps;
    }
    __syncthreads();
    if (!sh.go) break;
  }
}

// cv2.estimateAffinePartial2D(pairs, RANSAC, ...) by the whole block.  Leaves the model in sh.H, sh.status and the loop's
// iteration count in sh.iter (visible to every thread on return); mask [n] (or NULL) gets the winner's inliers.
template <class Pairs>
__device__ void affine_ransac(const Pairs& P, int n, const AffineParams& prm, const AffineTrace& tr, AffShared& sh, uint8_t* mask) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    sh.first = 0;
    sh.niters = max(prm.max_iters, 1);
    sh.best = 0;
    sh.win0 = sh.win1 = -1;
    sh.done = n <= kModelPoints;
    sh.iter = 0;
    sh.status = 0;
    for (int k = 0; k < 6; ++k) sh.H[k] = 0.0;
    if (n == kModelPoints) {                            // count == modelPoints: the one model, every pair an inlier, no refinement
      sh.win0 = 0;
      sh.win1 = 1;
    }
  }
  __syncthreads();
  unsigned long long s = ~0ull;                         // run() builds RNG rng((uint64)-1); warp 0's copy
  while (!sh.done) {
    const int first = sh.first, count = min(kAffWave, sh.niters - first);
    if (warp == 0)
      cvrng::warp_draw<kModelPoints>(s, first == 0, (unsigned)n, count, sh.samples, kModelPoints, tr.samples, first, tr.cap);
    __syncthreads();
    for (int h = warp; h < count; h += kAffWarps) {
      double M[6];
      float F[6];
      two_point_model(P(sh.samples[2 * h]), P(sh.samples[2 * h + 1]), M);
      to_f32(M, F);
      int c = 0;
      for (int j = lane; j < n; j += 32) c += cv_error(F, P(j)) <= prm.thr2 ? 1 : 0;
      c = __reduce_add_sync(0xffffffffu, c);
      if (lane == 0) {
        sh.counts[h] = c;
        if (first + h < tr.cap) {
          if (tr.counts) tr.counts[first + h] = c;
          if (tr.models)
            for (int k = 0; k < 6; ++k) tr.models[(size_t)(first + h) * 6 + k] = M[k];
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      int niters = sh.niters, best = sh.best;
      for (int h = 0; h < count; ++h) {
        const int i = first + h, c = sh.counts[h];
        if (c > max(best, kModelPoints - 1)) {          // strict: the earliest sample wins a tie
          best = c;
          sh.win0 = sh.samples[2 * h];
          sh.win1 = sh.samples[2 * h + 1];
          niters = cvrng::update_num_iters(prm.confidence, (double)(n - c) / n, kModelPoints, niters);
        }
        if (i + 1 >= niters) {
          sh.done = 1;
          sh.iter = i + 1;
          break;
        }
      }
      sh.niters = niters;
      sh.best = best;
      sh.first = first + count;
    }
    __syncthreads();
  }
  if (sh.win0 < 0) {                                    // no model: run() returns false, the mask is zeros
    if (mask)
      for (int j = tid; j < n; j += kAffThreads) mask[j] = 0;
    return;
  }
  double M[6];
  float F[6];
  two_point_model(P(sh.win0), P(sh.win1), M);
  to_f32(M, F);
  const float thr2 = prm.thr2;
  const bool all = n == kModelPoints;
  if (mask)
    for (int j = tid; j < n; j += kAffThreads) mask[j] = all || cv_error(F, P(j)) <= thr2 ? 1 : 0;
  double h[4] = {M[0], M[3], M[2], M[5]};               // (a, b, tx, ty)
  if (!all && prm.refine_iters > 0)
    lm_refine(P, n, [&](const Pair& p) { return cv_error(F, p) <= thr2; }, prm.refine_iters, h, sh);
  if (tid == 0) {
    sh.H[0] = sh.H[4] = h[0];
    sh.H[1] = -h[1];
    sh.H[3] = h[1];
    sh.H[2] = h[2];
    sh.H[5] = h[3];
    sh.status = 1;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kAffThreads) affine_partial_kernel(const float* __restrict__ from, const float* __restrict__ to,
                                                                     const int* __restrict__ offsets, AffineParams prm, AffineTrace tr,
                                                                     double* __restrict__ affine, uint8_t* __restrict__ mask,
                                                                     int* __restrict__ iterations, int* __restrict__ status) {
  __shared__ AffShared sh;
  const int b = blockIdx.x;
  const int o0 = offsets[b], n = max(offsets[b + 1] - o0, 0);
  affine_ransac(GlobalPairs{from + (size_t)2 * o0, to + (size_t)2 * o0}, n, prm, tr.at(b), sh, mask ? mask + o0 : nullptr);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 6; ++k) affine[(size_t)b * 6 + k] = sh.H[k];
    iterations[b] = sh.iter;
    status[b] = sh.status;
  }
}

// One block per problem b: match_worker's per-view match counts, detect_by_matching's choice, the winner's pairs compacted in
// ascending reference key-point order (numpy's mask order), the estimator on them, and the box of the view's corners.  The
// problem's V views are ref_kp / ref_count / ref_size (already offset to its first view), its matches rows b * v_stride + v of
// matches0, its query key points row q of q_kp / q_count.  Outputs go to row b.
__device__ __forceinline__ void boxes_block(int b, const float* __restrict__ ref_kp, const int* __restrict__ ref_count,
                                            const int* __restrict__ ref_size, int V, int v_stride, int cap_ref, const float* __restrict__ q_kp,
                                            const int* __restrict__ q_count, int q, int cap_q, const void* __restrict__ matches0,
                                            int matches_int64, int qH, int qW, const AffineParams& prm, const AffineTrace& tr,
                                            int32_t* __restrict__ box, int32_t* __restrict__ view, int32_t* __restrict__ n_matches,
                                            double* __restrict__ affine, int32_t* __restrict__ status) {
  extern __shared__ float4 pairs[];
  __shared__ AffShared sh;
  __shared__ int cnt[kMaxViews];
  __shared__ int warp_n[kAffWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long nq = min(max(q_count[q], 0), cap_q);
  auto match = [&](int v, int i) -> long long {
    const size_t o = ((size_t)b * v_stride + v) * cap_ref + i;
    return matches_int64 ? static_cast<const long long*>(matches0)[o] : (long long)static_cast<const int*>(matches0)[o];
  };
  auto n_ref = [&](int v) { return min(max(ref_count[v], 0), cap_ref); };
  for (int v = warp; v < V; v += kAffWarps) {
    const int nr = n_ref(v);
    int c = 0;
    for (int i = lane; i < nr; i += 32) {
      const long long m = match(v, i);
      c += m >= 0 && m < nq ? 1 : 0;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) cnt[v] = c;
  }
  __syncthreads();
  // sorted(..., key=inliers.shape[0], reverse=True)[0]: the most matches among views with >= 6 (shape 0 below), the first on a tie
  int win = 0, key = 0;
  for (int v = 0; v < V; ++v) {
    const int k = cnt[v] >= kMinMatches ? cnt[v] : 0;
    if (k > key) {
      key = k;
      win = v;
    }
  }
  if (tid == 0) {
    view[b] = win;
    n_matches[b] = cnt[win];
  }
  if (key == 0) {                                       // every view below 6: the first view's [0, 0, size[0], size[1]] = [0, 0, H, W]
    if (tid == 0) {
      const int32_t q[4] = {0, 0, qH, qW};
      for (int k = 0; k < 4; ++k) box[(size_t)b * 4 + k] = q[k];
      for (int k = 0; k < 6; ++k) affine[(size_t)b * 6 + k] = 0.0;
      status[b] = 2;
    }
    return;
  }
  const int nr = n_ref(win);
  int n = 0;
  for (int i0 = 0; i0 < nr; i0 += kAffThreads) {
    const int i = i0 + tid;
    const long long m = i < nr ? match(win, i) : -1;
    const bool f = m >= 0 && m < nq;
    int total;
    const int off = n + block_rank(f, warp_n, &total);
    if (f) {
      const float* r = ref_kp + ((size_t)win * cap_ref + i) * 2;
      const float* p = q_kp + ((size_t)q * cap_q + m) * 2;
      pairs[off] = make_float4(r[0], r[1], p[0], p[1]);
    }
    n += total;
  }
  // affine_ransac passes a barrier before it reads pairs
  affine_ransac(SharedPairs{pairs}, n, prm, tr.at(b), sh, nullptr);
  if (tid != 0) return;
  for (int k = 0; k < 6; ++k) affine[(size_t)b * 6 + k] = sh.H[k];
  // (affine @ [[0,0,1],[W,0,1],[0,H,1],[W,H,1]].T).T.astype(np.int32), then min / max; the empty box where the cast is undefined
  const double* H = sh.H;
  const double w = ref_size[win * 2 + 1], h = ref_size[win * 2];
  const double cx[4] = {0.0, w, 0.0, w}, cy[4] = {0.0, 0.0, h, h};
  bool ok = sh.status == 1;
  int32_t lo[2] = {INT32_MAX, INT32_MAX}, hi[2] = {INT32_MIN, INT32_MIN};
  for (int c = 0; c < 4 && ok; ++c)
    for (int r = 0; r < 2; ++r) {
      const double p = add(add(mul(H[r * 3], cx[c]), mul(H[r * 3 + 1], cy[c])), H[r * 3 + 2]);
      ok = ok && p > -2147483649.0 && p < 2147483648.0;   // false for NaN
      const int32_t t = ok ? (int32_t)p : 0;
      lo[r] = min(lo[r], t);
      hi[r] = max(hi[r], t);
    }
  const int32_t out[4] = {lo[0], lo[1], hi[0], hi[1]};
  for (int k = 0; k < 4; ++k) box[(size_t)b * 4 + k] = ok ? out[k] : 0;
  status[b] = ok ? 1 : 0;
}

// One block per frame b against all V views.
__global__ void __launch_bounds__(kAffThreads) boxes_from_matches_kernel(
    const float* __restrict__ ref_kp, const int* __restrict__ ref_count, const int* __restrict__ ref_size, int V, int cap_ref,
    const float* __restrict__ q_kp, const int* __restrict__ q_count, int cap_q, const void* __restrict__ matches0, int matches_int64,
    int qH, int qW, AffineParams prm, AffineTrace tr, int32_t* __restrict__ box, int32_t* __restrict__ view, int32_t* __restrict__ n_matches,
    double* __restrict__ affine, int32_t* __restrict__ status) {
  const int b = blockIdx.x;
  boxes_block(b, ref_kp, ref_count, ref_size, V, V, cap_ref, q_kp, q_count, b, cap_q, matches0, matches_int64, qH, qW, prm, tr, box, view,
              n_matches, affine, status);
}

// One block per (frame, object) pair b: views view_first[b] .. + view_count[b] - 1 of the table of n_views, query row
// query_index[b] of n_query, matches rows [b, 0 .. view_count[b]) of [B, v_stride, cap_ref].  A pair whose view range or query
// row is out of bounds gets status 0, the empty box, view 0, n_matches 0 and a zero affine.
__global__ void __launch_bounds__(kAffThreads) boxes_from_matches_objects_kernel(
    const float* __restrict__ ref_kp, const int* __restrict__ ref_count, const int* __restrict__ ref_size, int n_views, int cap_ref,
    const int* __restrict__ view_first, const int* __restrict__ view_count, int v_stride, const float* __restrict__ q_kp,
    const int* __restrict__ q_count, int n_query, int cap_q, const int* __restrict__ query_index, const void* __restrict__ matches0,
    int matches_int64, int qH, int qW, AffineParams prm, AffineTrace tr, int32_t* __restrict__ box, int32_t* __restrict__ view,
    int32_t* __restrict__ n_matches, double* __restrict__ affine, int32_t* __restrict__ status) {
  const int b = blockIdx.x;
  const int v0 = view_first[b], V = view_count[b], q = query_index[b];
  if (v0 < 0 || V < 1 || V > v_stride || v0 > n_views - V || q < 0 || q >= n_query) {
    if (threadIdx.x == 0) {
      for (int k = 0; k < 4; ++k) box[(size_t)b * 4 + k] = 0;
      for (int k = 0; k < 6; ++k) affine[(size_t)b * 6 + k] = 0.0;
      view[b] = 0;
      n_matches[b] = 0;
      status[b] = 0;
    }
    return;
  }
  boxes_block(b, ref_kp + (size_t)v0 * cap_ref * 2, ref_count + v0, ref_size + (size_t)v0 * 2, V, v_stride, cap_ref, q_kp, q_count, q, cap_q,
              matches0, matches_int64, qH, qW, prm, tr, box, view, n_matches, affine, status);
}

int check_params(const char* fn, double threshold, int32_t max_iters, double confidence, int32_t refine_iters) {
  REQUIRE(fn, isfinite(threshold) && max_iters >= 0 && confidence > 0.0 && confidence < 1.0 && refine_iters >= 0);
  return OPB_OK;
}

AffineParams make_params(double threshold, int32_t max_iters, double confidence, int32_t refine_iters) {
  return {(float)(threshold * threshold), max_iters, confidence, refine_iters};
}

}  // namespace
}  // namespace opb

// test hook: device buffers later calls of the three entry points fill (NULL to stop); see the header
static int32_t* g_aff_trace_samples = nullptr;
static int32_t* g_aff_trace_counts = nullptr;
static double* g_aff_trace_models = nullptr;
static int g_aff_trace_cap = 0;

static opb::AffineTrace aff_trace() { return {g_aff_trace_samples, g_aff_trace_counts, g_aff_trace_models, g_aff_trace_cap}; }

extern "C" int opb_debug_set_affine_trace(int32_t* samples, int32_t* counts, double* models, int32_t capacity) {
  REQUIRE(__func__, capacity > 0 || (capacity == 0 && !samples && !counts && !models));
  g_aff_trace_samples = samples;
  g_aff_trace_counts = counts;
  g_aff_trace_models = models;
  g_aff_trace_cap = capacity;
  return OPB_OK;
}

extern "C" int opb_estimate_affine_partial(const float* from, const float* to, const int32_t* offsets, int32_t B, double threshold,
                                           int32_t max_iters, double confidence, int32_t refine_iters, double* affine, uint8_t* inlier_mask,
                                           int32_t* iterations, int32_t* status, void* stream) {
  REQUIRE(__func__, from && to && offsets && affine && iterations && status && B > 0);
  if (int rc = opb::check_params(__func__, threshold, max_iters, confidence, refine_iters)) return rc;
  LAUNCH_NH(__func__, opb::affine_partial_kernel, (unsigned)B, opb::kAffThreads, 0, (cudaStream_t)stream, from, to, offsets,
            opb::make_params(threshold, max_iters, confidence, refine_iters), aff_trace(), affine, inlier_mask, iterations, status);
  return OPB_OK;
}

extern "C" int opb_boxes_from_matches(const float* ref_keypoints, const int32_t* ref_counts, const int32_t* ref_sizes, int32_t V, int32_t cap_ref,
                                      const float* query_keypoints, const int32_t* query_counts, int32_t cap_query, const void* matches0,
                                      int32_t matches_int64, int32_t B, int32_t query_h, int32_t query_w, int32_t* box, int32_t* view,
                                      int32_t* n_matches, double* affine, int32_t* status, void* stream) {
  REQUIRE(__func__, ref_keypoints && ref_counts && ref_sizes && query_keypoints && query_counts && matches0 && box && view && n_matches && affine &&
                        status);
  REQUIRE(__func__, V > 0 && V <= opb::kMaxViews && cap_ref > 0 && cap_ref <= opb::kMaxRefPoints && cap_query > 0 && B > 0);
  REQUIRE(__func__, (matches_int64 == 0 || matches_int64 == 1) && query_h > 0 && query_w > 0);
  const size_t smem = (size_t)cap_ref * sizeof(float4);
  CK(opb::no_handle_error, cudaFuncSetAttribute(opb::boxes_from_matches_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  LAUNCH_NH(__func__, opb::boxes_from_matches_kernel, (unsigned)B, opb::kAffThreads, smem, (cudaStream_t)stream, ref_keypoints, ref_counts, ref_sizes,
            V, cap_ref, query_keypoints, query_counts, cap_query, matches0, matches_int64, query_h, query_w,
            opb::make_params(6.0, 2000, 0.99, 10), aff_trace(), box, view, n_matches, affine, status);
  return OPB_OK;
}

extern "C" int opb_boxes_from_matches_objects(const float* ref_keypoints, const int32_t* ref_counts, const int32_t* ref_sizes, int32_t n_views,
                                              int32_t cap_ref, const int32_t* view_first, const int32_t* view_count, int32_t V_max,
                                              const float* query_keypoints, const int32_t* query_counts, int32_t n_query, int32_t cap_query,
                                              const int32_t* query_index, const void* matches0, int32_t matches_int64, int32_t B, int32_t query_h,
                                              int32_t query_w, int32_t* box, int32_t* view, int32_t* n_matches, double* affine, int32_t* status,
                                              void* stream) {
  REQUIRE(__func__, ref_keypoints && ref_counts && ref_sizes && view_first && view_count && query_keypoints && query_counts && query_index &&
                        matches0 && box && view && n_matches && affine && status);
  REQUIRE(__func__, n_views > 0 && cap_ref > 0 && cap_ref <= opb::kMaxRefPoints && V_max > 0 && V_max <= opb::kMaxViews);
  REQUIRE(__func__, n_query > 0 && cap_query > 0 && B > 0);
  REQUIRE(__func__, (matches_int64 == 0 || matches_int64 == 1) && query_h > 0 && query_w > 0);
  const size_t smem = (size_t)cap_ref * sizeof(float4);
  CK(opb::no_handle_error, cudaFuncSetAttribute(opb::boxes_from_matches_objects_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  LAUNCH_NH(__func__, opb::boxes_from_matches_objects_kernel, (unsigned)B, opb::kAffThreads, smem, (cudaStream_t)stream, ref_keypoints, ref_counts,
            ref_sizes, n_views, cap_ref, view_first, view_count, V_max, query_keypoints, query_counts, n_query, cap_query, query_index, matches0,
            matches_int64, query_h, query_w, opb::make_params(6.0, 2000, 0.99, 10), aff_trace(), box, view, n_matches, affine, status);
  return OPB_OK;
}
