// Batched RANSAC-PnP on the GPU: the consumer of the matcher's 2D-3D correspondences
// (reference src/utils/eval_utils.py:18-42: cv2.solvePnPRansac(pts_3d, pts_2d, K, 0, reprojectionError=5,
//  iterationsCount=10000, flags=SOLVEPNP_EPNP) per frame on the host -- the step that dominates per-frame latency once
//  matching takes ~1 ms; SURVEY 8f N3).
//
// The reference delegates the arithmetic to OpenCV; parity for this row is the pose itself (the reference's own metric is the
// cm-degree error, src/evaluators/cmd_evaluator.py), not bits: OpenCV draws its minimal samples from its own RNG.  Algorithm:
//   hypotheses  one thread per minimal sample: 3 correspondences -> P3P (Grunert's quartic, coefficients as in Haralick et al.
//               1994; closed-form quartic roots + Newton polish; the second depth ratio from the quadratic of one law-of-cosines
//               equation, then Newton on the three distance equations) -> up to 4 poses, each scored by its inlier count over
//               ALL correspondences of the frame (reprojection error < threshold, point in front of the camera), fp64;
//   selection   per frame: hypothesis with the most inliers (lowest index wins ties: deterministic);
//   refinement  Gauss-Newton on the reprojection error of the inlier set (6 DoF, left rotation update), inlier set re-evaluated
//               between rounds (local optimisation) -- what OpenCV's final EPnP refit on the inliers approximates.
// One launch handles B frames (ragged correspondence lists, offsets[B+1]); everything stays on the device.
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

struct Pose {
  double R[9];   // row-major, world -> camera
  double t[3];
};

// frame b of a batch: correspondences [o0, o0 + n) of the ragged lists, its intrinsics and its first 2D / 3D point
struct Frame {
  int o0, n;
  double Kc[4];   // fx, fy, cx, cy
  const double* p2;
  const double* p3;
};

__device__ __forceinline__ Frame frame_view(int b, const double* Kmat /*[B][9]*/, const double* pts2d, const double* pts3d, const int* offsets) {
  const int o0 = offsets[b];
  const double* K = Kmat + (size_t)b * 9;
  return {o0, offsets[b + 1] - o0, {K[0], K[4], K[2], K[5]}, pts2d + (size_t)o0 * 2, pts3d + (size_t)o0 * 3};
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {   // splitmix64 finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// K distinct indices in [0, n) for sample h of frame b: the k-th splitmix64 draw modulo n - k, shifted past the earlier
// indices in ascending order.  K is a compile-time constant so that the loops unroll and the sorted list stays in registers.
template <int K>
__device__ __forceinline__ void sample_distinct(unsigned long long seed, int b, int h, int n, int* idx) {
  uint64_t r = mix64(seed ^ ((uint64_t)b << 40) ^ (uint64_t)h);
  int srt[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (k > 0) r = mix64(r);
    int v = (int)(r % (uint64_t)(n - k));
#pragma unroll
    for (int e = 0; e < k; ++e)
      if (v >= srt[e]) ++v;
    idx[k] = v;
    srt[k] = v;                                          // insert into the sorted list
#pragma unroll
    for (int e = k; e > 0; --e)
      if (srt[e - 1] > srt[e]) { const int t = srt[e]; srt[e] = srt[e - 1]; srt[e - 1] = t; }
  }
}

// largest real root of z^3 + a2 z^2 + a1 z + a0
__device__ double cubic_largest_real(double a2, double a1, double a0) {
  const double q = (3.0 * a1 - a2 * a2) / 9.0, r = (9.0 * a2 * a1 - 27.0 * a0 - 2.0 * a2 * a2 * a2) / 54.0;
  const double D = q * q * q + r * r;
  if (D >= 0.0) {
    const double sD = sqrt(D);
    return cbrt(r + sD) + cbrt(r - sD) - a2 / 3.0;
  }
  const double th = acos(fmax(-1.0, fmin(1.0, r / sqrt(-q * q * q))));
  return 2.0 * sqrt(-q) * cos(th / 3.0) - a2 / 3.0;
}

// real roots of A4 x^4 + ... + A0 (Ferrari via the resolvent cubic), polished by two Newton steps that are kept only when
// they shrink |f|; returns their number.  A quadratic factor with a negative discriminant still yields its real part, flagged
// in *approx (bit k for x[k]): a double root, as a symmetric P3P sample produces, lands there as often as not, because the
// depressed coefficients lose most of their digits when the roots cluster (narrow views).  The caller verifies those.
__device__ int quartic_real_roots(double A4, double A3, double A2, double A1, double A0, double* x, unsigned* approx) {
  *approx = 0u;
  if (fabs(A4) < 1e-300) return 0;
  const double a = A3 / A4, b = A2 / A4, c = A1 / A4, d = A0 / A4;
  const double p = b - 3.0 * a * a / 8.0, q = c - a * b / 2.0 + a * a * a / 8.0;
  const double r = d - a * c / 4.0 + a * a * b / 16.0 - 3.0 * a * a * a * a / 256.0;
  double y[4];
  int n = 0;
  if (fabs(q) < 1e-14 * fmax(1.0, pow(fabs(p), 1.5))) {        // biquadratic
    const double disc = p * p - 4.0 * r;
    if (disc >= 0.0) {
      const double w[2] = {(-p + sqrt(disc)) / 2.0, (-p - sqrt(disc)) / 2.0};
      for (int k = 0; k < 2; ++k)
        if (w[k] >= 0.0) { y[n++] = sqrt(w[k]); y[n++] = -sqrt(w[k]); }
    }
  } else {
    const double z = cubic_largest_real(2.0 * p, p * p - 4.0 * r, -q * q);
    if (z <= 0.0) return 0;
    const double s = sqrt(z);
    for (int k = 0; k < 2; ++k) {
      const double sg = k ? -1.0 : 1.0;
      const double B = sg * s, C = (p + z - sg * q / s) / 2.0;   // y^2 + B y + C = 0
      const double disc = B * B - 4.0 * C;
      if (disc >= 0.0) { const double sd = sqrt(disc); y[n++] = (-B + sd) / 2.0; y[n++] = (-B - sd) / 2.0; }
      else { *approx |= 1u << n; y[n++] = -B / 2.0; }
    }
  }
  for (int k = 0; k < n; ++k) {
    double v = y[k] - a / 4.0;
    double f = (((A4 * v + A3) * v + A2) * v + A1) * v + A0;
    for (int it = 0; it < 2; ++it) {   // near a double root f' ~ 0 and a full step can leave for another root
      const double df = ((4.0 * A4 * v + 3.0 * A3) * v + 2.0 * A2) * v + A1;
      if (df == 0.0) break;
      const double vn = v - f / df, fn = (((A4 * vn + A3) * vn + A2) * vn + A1) * vn + A0;
      if (!(fabs(fn) < fabs(f))) break;
      v = vn;
      f = fn;
    }
    x[k] = v;
  }
  return n;
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ bool normalize3(double* a) {
  const double n = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  if (!(n > 1e-12)) return false;
  a[0] /= n; a[1] /= n; a[2] /= n;
  return true;
}
// unit bearing (camera frame) of pixel p2
__device__ __forceinline__ void bearing(const double* Kc, const double* p2, double* j) {
  j[0] = (p2[0] - Kc[2]) / Kc[0]; j[1] = (p2[1] - Kc[3]) / Kc[1]; j[2] = 1.0;
  normalize3(j);
}
// orthonormal frame of a triangle: columns e1 = (Q1-Q0)^, e3 = (e1 x (Q2-Q0))^, e2 = e3 x e1; F row-major [3][3] with columns e1,e2,e3
__device__ bool tri_frame(const double Q[3][3], double F[9]) {
  double e1[3] = {Q[1][0] - Q[0][0], Q[1][1] - Q[0][1], Q[1][2] - Q[0][2]};
  double d2[3] = {Q[2][0] - Q[0][0], Q[2][1] - Q[0][1], Q[2][2] - Q[0][2]};
  double e3[3], e2[3];
  if (!normalize3(e1)) return false;
  cross3(e1, d2, e3);
  if (!normalize3(e3)) return false;
  cross3(e3, e1, e2);
  for (int i = 0; i < 3; ++i) { F[i * 3 + 0] = e1[i]; F[i * 3 + 1] = e2[i]; F[i * 3 + 2] = e3[i]; }
  return true;
}

// P3P: world points P[3], unit bearings j[3] (camera frame) -> up to 4 poses
__device__ int p3p(const double P[3][3], const double j[3][3], Pose* out) {
  auto dist2 = [&](int a, int b) {
    const double dx = P[a][0] - P[b][0], dy = P[a][1] - P[b][1], dz = P[a][2] - P[b][2];
    return dx * dx + dy * dy + dz * dz;
  };
  auto dot = [&](int a, int b) { return j[a][0] * j[b][0] + j[a][1] * j[b][1] + j[a][2] * j[b][2]; };
  const double a2 = dist2(1, 2), b2 = dist2(0, 2), c2 = dist2(0, 1);
  if (!(a2 > 1e-18 && b2 > 1e-18 && c2 > 1e-18)) return 0;
  const double ca = dot(1, 2), cb = dot(0, 2), cg = dot(0, 1);
  const double p = (a2 - c2) / b2, q = (a2 + c2) / b2;
  const double A4 = (p - 1.0) * (p - 1.0) - 4.0 * c2 / b2 * ca * ca;
  const double A3 = 4.0 * (p * (1.0 - p) * cb - (1.0 - q) * ca * cg + 2.0 * c2 / b2 * ca * ca * cb);
  const double A2 = 2.0 * (p * p - 1.0 + 2.0 * p * p * cb * cb + 2.0 * ((b2 - c2) / b2) * ca * ca - 4.0 * q * ca * cb * cg + 2.0 * ((b2 - a2) / b2) * cg * cg);
  const double A1 = 4.0 * (-p * (1.0 + p) * cb + 2.0 * a2 / b2 * cg * cg * cb - (1.0 - q) * ca * cg);
  const double A0 = (1.0 + p) * (1.0 + p) - 4.0 * a2 / b2 * cg * cg;
  double v[4];
  unsigned approx;
  const int nr = quartic_real_roots(A4, A3, A2, A1, A0, v, &approx);
  double FP[9];
  if (!tri_frame(P, FP)) return 0;
  double depths[4][3];
  int ns = 0;
  for (int k = 0; k < nr && ns < 4; ++k) {
    if (!(v[k] > 0.0)) continue;
    // depths (s0, u s0, v s0): s0 from the b^2 equation; u from the quadratic of the c^2 equation, u^2 - 2 cg u + 1 -
    // (c2/b2) w = 0, the root that better satisfies the a^2 equation first.  (Grunert's linear back-substitution divides by
    // cg - v ca, which vanishes at the true root of a sample symmetric about a plane through the camera centre; both roots
    // then satisfy the a^2 equation and both are poses.)
    const double w = 1.0 + v[k] * v[k] - 2.0 * v[k] * cb;
    if (!(w > 0.0)) continue;
    const double sd = sqrt(fmax(0.0, cg * cg - 1.0 + c2 / b2 * w));
    double uc[2] = {cg + sd, cg - sd};
    const double e0 = fabs(uc[0] * uc[0] + v[k] * v[k] - 2.0 * uc[0] * v[k] * ca - a2 / b2 * w);
    const double e1 = fabs(uc[1] * uc[1] + v[k] * v[k] - 2.0 * uc[1] * v[k] * ca - a2 / b2 * w);
    if (e1 < e0) { const double tmp = uc[0]; uc[0] = uc[1]; uc[1] = tmp; }
    for (int m = 0; m < 2 && ns < 4; ++m) {
      const bool verify = m == 1 || ((approx >> k) & 1u);   // a candidate that must prove itself a solution
      if (!(uc[m] > 0.0)) continue;
      const double s0 = sqrt(b2 / w);
      double s[3] = {s0, uc[m] * s0, v[k] * s0};
      // Newton on the three distance equations: the quartic root carries its conditioning into u and s, the depths'
      // own system is well conditioned for any sample a P3P can solve
      double F[3];
      for (int it = 0; it < 6; ++it) {   // from a clustered-root start the quadratic phase takes a few steps
        F[0] = s[1] * s[1] + s[2] * s[2] - 2.0 * s[1] * s[2] * ca - a2;
        F[1] = s[0] * s[0] + s[2] * s[2] - 2.0 * s[0] * s[2] * cb - b2;
        F[2] = s[0] * s[0] + s[1] * s[1] - 2.0 * s[0] * s[1] * cg - c2;
        const double J[3][3] = {{0.0, 2.0 * (s[1] - s[2] * ca), 2.0 * (s[2] - s[1] * ca)},
                                {2.0 * (s[0] - s[2] * cb), 0.0, 2.0 * (s[2] - s[0] * cb)},
                                {2.0 * (s[0] - s[1] * cg), 2.0 * (s[1] - s[0] * cg), 0.0}};
        const double C0 = J[1][1] * J[2][2] - J[1][2] * J[2][1], C1 = J[1][2] * J[2][0] - J[1][0] * J[2][2], C2 = J[1][0] * J[2][1] - J[1][1] * J[2][0];
        const double det = J[0][0] * C0 + J[0][1] * C1 + J[0][2] * C2;
        if (!(fabs(det) > 1e-300)) break;
        // s -= J^-1 F (adjugate)
        const double d0 = (C0 * F[0] + (J[0][2] * J[2][1] - J[0][1] * J[2][2]) * F[1] + (J[0][1] * J[1][2] - J[0][2] * J[1][1]) * F[2]) / det;
        const double d1 = (C1 * F[0] + (J[0][0] * J[2][2] - J[0][2] * J[2][0]) * F[1] + (J[0][2] * J[1][0] - J[0][0] * J[1][2]) * F[2]) / det;
        const double d2 = (C2 * F[0] + (J[0][1] * J[2][0] - J[0][0] * J[2][1]) * F[1] + (J[0][0] * J[1][1] - J[0][1] * J[1][0]) * F[2]) / det;
        s[0] -= d0; s[1] -= d1; s[2] -= d2;
      }
      if (!(s[0] > 0.0 && s[1] > 0.0 && s[2] > 0.0)) continue;
      if (verify) {
        F[0] = s[1] * s[1] + s[2] * s[2] - 2.0 * s[1] * s[2] * ca - a2;
        F[1] = s[0] * s[0] + s[2] * s[2] - 2.0 * s[0] * s[2] * cb - b2;
        F[2] = s[0] * s[0] + s[1] * s[1] - 2.0 * s[0] * s[1] * cg - c2;
        const double sm = fmax(s[0], fmax(s[1], s[2]));
        if (!(fmax(fabs(F[0]), fmax(fabs(F[1]), fabs(F[2]))) <= 1e-12 * sm * sm)) continue;
      }
      bool dup = false;                                  // a double root is reported twice
      const double smax = fmax(s[0], fmax(s[1], s[2]));
      for (int o = 0; o < ns; ++o)
        dup |= fmax(fabs(s[0] - depths[o][0]), fmax(fabs(s[1] - depths[o][1]), fabs(s[2] - depths[o][2]))) <= 1e-9 * smax;
      if (dup) continue;
      double X[3][3];
      for (int i = 0; i < 3; ++i)
        for (int d = 0; d < 3; ++d) X[i][d] = s[i] * j[i][d];
      double FX[9];
      if (!tri_frame(X, FX)) continue;
      Pose& o = out[ns];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) o.R[r * 3 + c] = FX[r * 3 + 0] * FP[c * 3 + 0] + FX[r * 3 + 1] * FP[c * 3 + 1] + FX[r * 3 + 2] * FP[c * 3 + 2];   // FX . FP^T
      for (int r = 0; r < 3; ++r) o.t[r] = X[0][r] - (o.R[r * 3 + 0] * P[0][0] + o.R[r * 3 + 1] * P[0][1] + o.R[r * 3 + 2] * P[0][2]);
      for (int i = 0; i < 3; ++i) depths[ns][i] = s[i];
      ++ns;
    }
  }
  return ns;
}

// world point p3 in the camera frame of T
__device__ __forceinline__ void to_camera(const Pose& T, const double* p3, double* X) {
#pragma unroll
  for (int r = 0; r < 3; ++r) X[r] = T.R[r * 3] * p3[0] + T.R[r * 3 + 1] * p3[1] + T.R[r * 3 + 2] * p3[2] + T.t[r];
}

// squared reprojection error of the correspondence p3 -> p2 under T, in fp64
__device__ __forceinline__ double reproj_err2(const Pose& T, const double* Kc /*fx,fy,cx,cy*/, const double* p3, const double* p2) {
  double X[3];
  to_camera(T, p3, X);
  const double du = Kc[0] * X[0] / X[2] + Kc[2] - p2[0], dv = Kc[1] * X[1] / X[2] + Kc[3] - p2[1];
  return du * du + dv * dv;
}

// the P3P path's inlier rule: in front of the camera and squared reprojection error < thr^2.  Not written on reproj_err2:
// that form costs both P3P kernels registers and spills.
__device__ __forceinline__ bool reproj_inlier(const Pose& T, const double* Kc, const double* p3, const double* p2, double thr2) {
  double X[3];
  to_camera(T, p3, X);
  if (!(X[2] > 1e-9)) return false;
  const double du = Kc[0] * X[0] / X[2] + Kc[2] - p2[0], dv = Kc[1] * X[1] / X[2] + Kc[3] - p2[1];
  return du * du + dv * dv < thr2;
}

// hyp: [B][H] records {count, R (9), t (3)} as 13 doubles (the workspace layout of include/onepose_b200.h)
constexpr int kHypStride = 13;
constexpr int kHypThreads = 128;
constexpr int kMaxHypotheses = 65535 * kHypThreads;

__device__ __forceinline__ void store_record(double* rec, double count, const Pose& T) {
  rec[0] = count;
  for (int k = 0; k < 9; ++k) rec[1 + k] = T.R[k];
  for (int k = 0; k < 3; ++k) rec[10 + k] = T.t[k];
}
__device__ __forceinline__ Pose load_record(const double* rec) {   // the record's pose; its count is rec[0]
  Pose T;
  for (int k = 0; k < 9; ++k) T.R[k] = rec[1 + k];
  for (int k = 0; k < 3; ++k) T.t[k] = rec[10 + k];
  return T;
}

__global__ void __launch_bounds__(kHypThreads, 4) pnp_hypotheses(const double* __restrict__ Kmat /*[B][9]*/, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                      const int* __restrict__ offsets, int H, double thr2, unsigned long long seed,
                                                      double* __restrict__ hyp) {
  const int b = blockIdx.x;                          // frames on x: any B; hypothesis blocks on y (at most 65535)
  const int h = blockIdx.y * blockDim.x + threadIdx.x;
  if (h >= H) return;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  double* out = hyp + ((size_t)b * H + h) * kHypStride;
  out[0] = 0.0;
  if (f.n < 4) return;
  int idx[3];
  sample_distinct<3>(seed, b, h, f.n, idx);
  double P[3][3], j[3][3];
  for (int k = 0; k < 3; ++k) {
    const double* p3 = f.p3 + (size_t)idx[k] * 3;
    P[k][0] = p3[0]; P[k][1] = p3[1]; P[k][2] = p3[2];
    bearing(f.Kc, f.p2 + (size_t)idx[k] * 2, j[k]);
  }
  Pose sol[4];
  const int ns = p3p(P, j, sol);
  int best = -1, best_cnt = 0;
  for (int s = 0; s < ns; ++s) {
    int cnt = 0;
    // indexed from the batch's arrays: from the frame's base pointers this loop runs about 1 % slower on an H100
    for (int i = 0; i < f.n; ++i) cnt += reproj_inlier(sol[s], f.Kc, pts3d + (size_t)(f.o0 + i) * 3, pts2d + (size_t)(f.o0 + i) * 2, thr2) ? 1 : 0;
    if (cnt > best_cnt) { best_cnt = cnt; best = s; }
  }
  if (best < 0) return;
  store_record(out, (double)best_cnt, sol[best]);
}

__device__ void rodrigues_left(const double* w, Pose& T) {   // T <- exp([w]x) . T (rotation and translation), small-angle safe
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  const double A = th > 1e-8 ? sin(th) / th : 1.0 - th2 / 6.0, Bc = th > 1e-8 ? (1.0 - cos(th)) / th2 : 0.5 - th2 / 24.0;
  double E[9];
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double w2 = 0;
      for (int k = 0; k < 3; ++k) w2 += W[r * 3 + k] * W[k * 3 + c];
      E[r * 3 + c] = (r == c ? 1.0 : 0.0) + A * W[r * 3 + c] + Bc * w2;
    }
  double Rn[9], tn[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Rn[r * 3 + c] = E[r * 3 + 0] * T.R[c] + E[r * 3 + 1] * T.R[3 + c] + E[r * 3 + 2] * T.R[6 + c];
    tn[r] = E[r * 3 + 0] * T.t[0] + E[r * 3 + 1] * T.t[1] + E[r * 3 + 2] * T.t[2];
  }
  for (int k = 0; k < 9; ++k) T.R[k] = Rn[k];
  for (int k = 0; k < 3; ++k) T.t[k] = tn[k];
}

// block-wide arg-max over frame b's hypothesis records: the most inliers, the lowest index on ties.  Returns the count and
// sets *best_h; every thread of the block gets the same answer.
constexpr int kRefineThreads = 256;
__device__ int best_hypothesis(const double* __restrict__ hyp, int b, int H, unsigned long long* best_key /*shared [kRefineThreads]*/, int* best_h) {
  const int tid = threadIdx.x;
  unsigned long long key = 0ull;
  for (int h = tid; h < H; h += kRefineThreads) {
    const unsigned long long c = (unsigned long long)hyp[((size_t)b * H + h) * kHypStride];
    const unsigned long long k = (c << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)h);
    key = k > key ? k : key;
  }
  best_key[tid] = key;
  __syncthreads();
  for (int s = kRefineThreads / 2; s > 0; s >>= 1) {
    if (tid < s && best_key[tid + s] > best_key[tid]) best_key[tid] = best_key[tid + s];
    __syncthreads();
  }
  const unsigned long long bk = best_key[0];
  *best_h = (int)(0xFFFFFFFFu - (unsigned)(bk & 0xFFFFFFFFull));
  return (int)(bk >> 32);
}

__device__ __forceinline__ void write_pose(const Pose& T, double* dst) {
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) dst[r * 4 + k] = T.R[r * 3 + k];
    dst[r * 4 + 3] = T.t[r];
  }
}
__device__ __forceinline__ void write_identity(double* dst) {
  for (int k = 0; k < 12; ++k) dst[k] = (k == 0 || k == 5 || k == 10) ? 1.0 : 0.0;
}
// a frame without a model, by its whole block: identity pose, no inliers (the reference's except-branch result)
__device__ __forceinline__ void write_no_model(int b, const Frame& f, double* pose_out, int* inlier_mask, int* n_inliers) {
  for (int i = threadIdx.x; i < f.n; i += kRefineThreads) inlier_mask[f.o0 + i] = 0;
  if (threadIdx.x == 0) {
    write_identity(pose_out + (size_t)b * 12);
    n_inliers[b] = 0;
  }
}

// one block per frame: arg-max over hypotheses, local optimisation, outputs
__global__ void __launch_bounds__(kRefineThreads) pnp_select_refine(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                                     const int* __restrict__ offsets, int H, double thr2, const double* __restrict__ hyp,
                                                                     double* __restrict__ pose_out /*[B][12]*/, int* __restrict__ inlier_mask,
                                                                     int* __restrict__ n_inliers /*[B]*/) {
  __shared__ unsigned long long best_key[kRefineThreads];
  __shared__ double red[27][kRefineThreads / 32];
  __shared__ int cnt_w[kRefineThreads / 32];
  __shared__ Pose T;
  __shared__ double delta[6];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  // ---- best hypothesis: max count, lowest index
  int best_h;
  if (best_hypothesis(hyp, b, H, best_key, &best_h) < 4) {
    write_no_model(b, f, pose_out, inlier_mask, n_inliers);
    return;
  }
  if (tid == 0) T = load_record(hyp + ((size_t)b * H + best_h) * kHypStride);
  __syncthreads();
  // ---- Gauss-Newton on the inliers of the current pose; the inlier set is re-evaluated every round
  for (int it = 0; it < 10; ++it) {
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) acc[k] = 0.0;
    const Pose Tl = T;
    for (int i = tid; i < f.n; i += kRefineThreads) {
      const double* p3 = f.p3 + (size_t)i * 3;
      const double* p2 = f.p2 + (size_t)i * 2;
      if (!reproj_inlier(Tl, f.Kc, p3, p2, thr2)) continue;
      double X[3];
      to_camera(Tl, p3, X);
      const double x = X[0], y = X[1], z = X[2];
      const double* Kc = f.Kc;
      const double iz = 1.0 / z;
      const double ru = Kc[0] * x * iz + Kc[2] - p2[0], rv = Kc[1] * y * iz + Kc[3] - p2[1];
      // d(proj)/dX, X' = exp(w) X + dt  =>  dX/dw = -[X]x, dX/dt = I
      const double jux = Kc[0] * iz, juz = -Kc[0] * x * iz * iz, jvy = Kc[1] * iz, jvz = -Kc[1] * y * iz * iz;
      double Ju[6], Jv[6];
      Ju[0] = juz * y;            Ju[1] = jux * z - juz * x;  Ju[2] = -jux * y;           // rotation part: row . (-[X]x)
      Jv[0] = -jvy * z + jvz * y; Jv[1] = -jvz * x;           Jv[2] = jvy * x;
      Ju[3] = jux; Ju[4] = 0.0; Ju[5] = juz;
      Jv[3] = 0.0; Jv[4] = jvy; Jv[5] = jvz;
      int k = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = r; c < 6; ++c) acc[k++] += Ju[r] * Ju[c] + Jv[r] * Jv[c];
#pragma unroll
      for (int r = 0; r < 6; ++r) acc[21 + r] += Ju[r] * ru + Jv[r] * rv;
    }
    // block_sum<27> gives the same sums in the same order, but costs this kernel two registers: thread 0 sums here
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      double v = acc[k];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[k][warp] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double A[6][6], g[6];
      int k = 0;
      for (int r = 0; r < 6; ++r)
        for (int c = r; c < 6; ++c) {
          double v = 0;
          for (int w = 0; w < kRefineThreads / 32; ++w) v += red[k][w];
          A[r][c] = A[c][r] = v;
          ++k;
        }
      for (int r = 0; r < 6; ++r) {
        double v = 0;
        for (int w = 0; w < kRefineThreads / 32; ++w) v += red[21 + r][w];
        g[r] = -v;
      }
      for (int r = 0; r < 6; ++r) A[r][r] *= 1.0 + 1e-9;      // tiny damping against rank deficiency
      // Cholesky solve A d = g
      bool good = true;
      double Lm[6][6] = {};
      for (int r = 0; r < 6 && good; ++r)
        for (int c = 0; c <= r; ++c) {
          double s = A[r][c];
          for (int m = 0; m < c; ++m) s -= Lm[r][m] * Lm[c][m];
          if (r == c) { if (!(s > 1e-300)) { good = false; break; } Lm[r][r] = sqrt(s); }
          else Lm[r][c] = s / Lm[c][c];
        }
      double yv[6], d[6] = {0, 0, 0, 0, 0, 0};
      if (good) {
        for (int r = 0; r < 6; ++r) { double s = g[r]; for (int m = 0; m < r; ++m) s -= Lm[r][m] * yv[m]; yv[r] = s / Lm[r][r]; }
        for (int r = 5; r >= 0; --r) { double s = yv[r]; for (int m = r + 1; m < 6; ++m) s -= Lm[m][r] * d[m]; d[r] = s / Lm[r][r]; }
      }
      for (int r = 0; r < 6; ++r) delta[r] = d[r];
      rodrigues_left(d, T);
      T.t[0] += d[3]; T.t[1] += d[4]; T.t[2] += d[5];
    }
    __syncthreads();
    const double step = fabs(delta[0]) + fabs(delta[1]) + fabs(delta[2]) + fabs(delta[3]) + fabs(delta[4]) + fabs(delta[5]);
    if (step < 1e-12) break;
  }
  // ---- outputs.  A threshold that admits gross outliers lets the refinement leave the model (on 40 % outliers at 1000 px it
  // ends with the object behind the camera): a refined pose with fewer than 4 inliers gives way to the hypothesis it started from.
  int cnt = 0;
  for (int pass = 0; pass < 2; ++pass) {
    cnt = 0;
    for (int i = tid; i < f.n; i += kRefineThreads) {
      const int in = reproj_inlier(T, f.Kc, f.p3 + (size_t)i * 3, f.p2 + (size_t)i * 2, thr2) ? 1 : 0;
      inlier_mask[f.o0 + i] = in;
      cnt += in;
    }
    cnt = block_reduce(cnt, Sum32(), cnt_w);
    if (cnt >= 4) break;
    __syncthreads();                                 // every thread has read T
    if (tid == 0) T = load_record(hyp + ((size_t)b * H + best_h) * kHypStride);
    __syncthreads();
  }
  if (tid == 0) {
    n_inliers[b] = cnt;
    write_pose(T, pose_out + (size_t)b * 12);
  }
}

// ---- EPnP (Lepetit, Moreno-Noguer, Fua, "EPnP: An Accurate O(n) Solution to the PnP Problem", IJCV 2009), fp64.
// Control points: the centroid c0 and c0 + sqrt(lambda_k / n) e_k along the principal axes of the point set (largest first);
// every point is an affine combination (the alphas) of them, so its camera coordinates are the same combination of the
// control points' camera coordinates x (12 unknowns), and each correspondence gives two rows of M x = 0.  x lies near the span
// of the eigenvectors v_0..v_3 of M^T M with the smallest eigenvalues; x = sum beta_k v_k, the betas from the six distance
// constraints |c_a - c_b| (L [6x10] . products of the betas = rho), linearised for N = 1, 2, 3 vectors and refined by
// Gauss-Newton; each candidate gives the points' camera coordinates (depth sign made positive) and R, t by absolute
// orientation; the candidate with the lowest mean reprojection error wins, the first on ties.
// Everything the candidates need from the points is a sum over them (kEpnpSums), so one routine serves a thread that loops
// over a 5-point sample and a block that reduces over a frame.
constexpr int kMtmSums = 78;                           // upper triangle of M^T M (12 x 12)
constexpr int kEpnpSums = kMtmSums + 10 + 4;           // + upper triangle of alpha^T alpha (4 x 4) + alpha sums
constexpr int kEpnpGnIters = 5;

// symmetric eigenproblem by cyclic Jacobi rotations: A [N*N] row-major (its diagonal ends as the eigenvalues), V [N*N]
// (columns = eigenvectors).  Fixed sweep order: deterministic.
template <int N>
__device__ void jacobi_eigen(double* A, double* V) {
  for (int i = 0; i < N * N; ++i) V[i] = (i % (N + 1)) == 0 ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    double off = 0.0, dia = 0.0;
    for (int p = 0; p < N; ++p) {
      dia += A[p * N + p] * A[p * N + p];
      for (int q = p + 1; q < N; ++q) off += A[p * N + q] * A[p * N + q];
    }
    if (!(off > 1e-34 * dia)) break;
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p * N + q];
        if (apq == 0.0) continue;
        const double th = (A[q * N + q] - A[p * N + p]) / (2.0 * apq);
        const double t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {               // A <- A J
          const double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {               // A <- J^T A
          const double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {               // V <- V J
          const double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
  }
}

// least squares min |A x - b| of a 6 x k system (k <= 5) by Householder QR; a [6*5] row-major (first k columns) and b are
// destroyed.  False when a column is rank deficient.
__device__ bool lstsq6(double* a, double* b, int k, double* x) {
  for (int j = 0; j < k; ++j) {
    double nrm = 0.0;
    for (int r = j; r < 6; ++r) nrm += a[r * 5 + j] * a[r * 5 + j];
    nrm = sqrt(nrm);
    if (!(nrm > 0.0)) return false;
    const double alpha = a[j * 5 + j] > 0.0 ? -nrm : nrm;
    double v[6], vv = 0.0;
    for (int r = j; r < 6; ++r) v[r] = a[r * 5 + j];
    v[j] -= alpha;
    for (int r = j; r < 6; ++r) vv += v[r] * v[r];
    if (vv > 0.0) {
      for (int c = j; c < k; ++c) {
        double s = 0.0;
        for (int r = j; r < 6; ++r) s += v[r] * a[r * 5 + c];
        s *= 2.0 / vv;
        for (int r = j; r < 6; ++r) a[r * 5 + c] -= s * v[r];
      }
      double s = 0.0;
      for (int r = j; r < 6; ++r) s += v[r] * b[r];
      s *= 2.0 / vv;
      for (int r = j; r < 6; ++r) b[r] -= s * v[r];
    }
  }
  for (int j = k - 1; j >= 0; --j) {
    double s = b[j];
    for (int c = j + 1; c < k; ++c) s -= a[j * 5 + c] * x[c];
    x[j] = s / a[j * 5 + j];
  }
  return true;
}

constexpr double kEpnpFlat = 1e-10;                   // an axis whose eigenvalue is below this fraction of the largest is flat

struct EpnpBasis {
  double c[4][3];    // world control points
  double ax[3][3];   // c[k+1] - c[0]
  double il2[3];     // 1 / |ax_k|^2
  int planar;        // the third axis is flat: its control point is placed at full length along the plane's normal
};

// centroid sum[3] and scatter sc[6] = {xx, xy, xz, yy, yz, zz} about the centroid of m points -> control points.
// Each axis is an eigenvector of the scatter with its largest-magnitude component made positive (the first such component on
// ties), so that the control points -- and, on noisy data, EPnP's algebraic least squares, which depends on them -- do not
// depend on the sign an eigen-solver happens to return.  A flat third axis (a planar set) gets the length of the first, so
// that its control point stays a distinct point: the points' coordinates along it are then (near) 0 and its camera
// coordinates are fixed by the distance constraints alone.  False for coincident or collinear points.
__device__ bool epnp_basis(const double* sum, const double* sc, int m, EpnpBasis& E) {
  double A[9] = {sc[0], sc[1], sc[2], sc[1], sc[3], sc[4], sc[2], sc[4], sc[5]}, V[9];
  jacobi_eigen<3>(A, V);
  int ord[3] = {0, 1, 2};                              // descending eigenvalues
  for (int i = 1; i < 3; ++i)
    for (int j = i; j > 0 && A[ord[j] * 4] > A[ord[j - 1] * 4]; --j) { const int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; }
  const double l0 = A[ord[0] * 4];
  if (!(l0 > 0.0) || !(A[ord[1] * 4] > kEpnpFlat * l0)) return false;
  E.planar = A[ord[2] * 4] > kEpnpFlat * l0 ? 0 : 1;
  for (int d = 0; d < 3; ++d) E.c[0][d] = sum[d] / m;
  for (int k = 0; k < 3; ++k) {
    const double lam = (k == 2 && E.planar) ? l0 : A[ord[k] * 4];
    int big = 0;
    for (int d = 1; d < 3; ++d)
      if (fabs(V[d * 3 + ord[k]]) > fabs(V[big * 3 + ord[k]])) big = d;
    const double s = (V[big * 3 + ord[k]] < 0.0 ? -1.0 : 1.0) * sqrt(lam / m);
    double l2 = 0.0;
    for (int d = 0; d < 3; ++d) {
      E.c[k + 1][d] = E.c[0][d] + s * V[d * 3 + ord[k]];
      E.ax[k][d] = E.c[k + 1][d] - E.c[0][d];
      l2 += E.ax[k][d] * E.ax[k][d];
    }
    if (!(l2 > 0.0)) return false;
    E.il2[k] = 1.0 / l2;
  }
  return true;
}

__device__ __forceinline__ void epnp_alphas(const EpnpBasis& E, const double* p, double* a) {
  const double d[3] = {p[0] - E.c[0][0], p[1] - E.c[0][1], p[2] - E.c[0][2]};
  for (int k = 0; k < 3; ++k) a[k + 1] = (E.ax[k][0] * d[0] + E.ax[k][1] * d[1] + E.ax[k][2] * d[2]) * E.il2[k];
  a[0] = 1.0 - a[1] - a[2] - a[3];
}

// one correspondence's contribution to the kEpnpSums sums
__device__ __forceinline__ void epnp_accumulate(const double* a, const double* uv, const double* Kc, double* acc) {
  double r1[12], r2[12];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    r1[3 * j] = a[j] * Kc[0]; r1[3 * j + 1] = 0.0; r1[3 * j + 2] = a[j] * (Kc[2] - uv[0]);
    r2[3 * j] = 0.0; r2[3 * j + 1] = a[j] * Kc[1]; r2[3 * j + 2] = a[j] * (Kc[3] - uv[1]);
  }
  int k = 0;
#pragma unroll
  for (int r = 0; r < 12; ++r)
#pragma unroll
    for (int c = r; c < 12; ++c) acc[k++] += r1[r] * r1[c] + r2[r] * r2[c];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = r; c < 4; ++c) acc[k++] += a[r] * a[c];
#pragma unroll
  for (int r = 0; r < 4; ++r) acc[k++] += a[r];
}

__device__ __forceinline__ void beta_products(const double* be, double* p) {
  p[0] = be[0] * be[0]; p[1] = be[0] * be[1]; p[2] = be[1] * be[1]; p[3] = be[0] * be[2]; p[4] = be[1] * be[2];
  p[5] = be[2] * be[2]; p[6] = be[0] * be[3]; p[7] = be[1] * be[3]; p[8] = be[2] * be[3]; p[9] = be[3] * be[3];
}

// beta0, beta1 from the linearised b00, b01, b11
__device__ __forceinline__ void two_betas(double b00, double b01, double b11, double* be) {
  if (b00 < 0.0) { be[0] = sqrt(-b00); be[1] = b11 < 0.0 ? sqrt(-b11) : 0.0; }
  else { be[0] = sqrt(b00); be[1] = b11 > 0.0 ? sqrt(b11) : 0.0; }
  if (b01 < 0.0) be[0] = -be[0];
}

// the three candidates' poses from the sums of m points
__device__ void epnp_candidates(const double* sums, const EpnpBasis& E, int m, Pose* cand) {
  double A[144], V[144];
  {
    int k = 0;
    for (int r = 0; r < 12; ++r)
      for (int c = r; c < 12; ++c) { A[r * 12 + c] = A[c * 12 + r] = sums[k]; ++k; }
  }
  jacobi_eigen<12>(A, V);
  int ord[12];
  for (int i = 0; i < 12; ++i) ord[i] = i;
  for (int i = 1; i < 12; ++i)                          // ascending eigenvalues, stable
    for (int j = i; j > 0 && A[ord[j] * 13] < A[ord[j - 1] * 13]; --j) { const int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; }
  if (E.planar) {
    // the flat axis's control point is unconstrained by M (its columns are (near) zero), so three of the four smallest
    // eigenvalues belong to vectors that live on its columns and tie with the true one: the vector with the least weight
    // there goes first (stable), the one the N = 1 .. 3 approximations build on
    double w[4];
    for (int k = 0; k < 4; ++k) w[k] = V[9 * 12 + ord[k]] * V[9 * 12 + ord[k]] + V[10 * 12 + ord[k]] * V[10 * 12 + ord[k]] + V[11 * 12 + ord[k]] * V[11 * 12 + ord[k]];
    for (int i = 1; i < 4; ++i)
      for (int j = i; j > 0 && w[j] < w[j - 1]; --j) {
        const double tw = w[j]; w[j] = w[j - 1]; w[j - 1] = tw;
        const int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t;
      }
  }
  double v[4][12];
  for (int k = 0; k < 4; ++k)
    for (int i = 0; i < 12; ++i) v[k][i] = V[i * 12 + ord[k]];
  const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
  double L[6][10], rho[6];
  for (int r = 0; r < 6; ++r) {
    double dv[4][3];
    for (int k = 0; k < 4; ++k)
      for (int d = 0; d < 3; ++d) dv[k][d] = v[k][3 * pa[r] + d] - v[k][3 * pb[r] + d];
    auto dot = [&](int i, int j) { return dv[i][0] * dv[j][0] + dv[i][1] * dv[j][1] + dv[i][2] * dv[j][2]; };
    L[r][0] = dot(0, 0); L[r][1] = 2.0 * dot(0, 1); L[r][2] = dot(1, 1); L[r][3] = 2.0 * dot(0, 2); L[r][4] = 2.0 * dot(1, 2);
    L[r][5] = dot(2, 2); L[r][6] = 2.0 * dot(0, 3); L[r][7] = 2.0 * dot(1, 3); L[r][8] = 2.0 * dot(2, 3); L[r][9] = dot(3, 3);
    double r2 = 0.0;
    for (int d = 0; d < 3; ++d) r2 += (E.c[pa[r]][d] - E.c[pb[r]][d]) * (E.c[pa[r]][d] - E.c[pb[r]][d]);
    rho[r] = r2;
  }
  const double* G = sums + kMtmSums;                  // alpha^T alpha, upper triangle
  const double* as = sums + kMtmSums + 10;            // alpha sums
  double Gm[4][4];
  {
    int k = 0;
    for (int r = 0; r < 4; ++r)
      for (int c = r; c < 4; ++c) { Gm[r][c] = Gm[c][r] = G[k]; ++k; }
  }
  const int cols[3][5] = {{0, 1, 3, 6, 0}, {0, 1, 2, 0, 0}, {0, 1, 2, 3, 4}};
  const int ncols[3] = {4, 3, 5};
  for (int N = 0; N < 3; ++N) {
    double a[30], bb[6], x[5] = {0, 0, 0, 0, 0}, be[4] = {0, 0, 0, 0};
    for (int r = 0; r < 6; ++r) {
      for (int c = 0; c < ncols[N]; ++c) a[r * 5 + c] = L[r][cols[N][c]];
      bb[r] = rho[r];
    }
    if (!lstsq6(a, bb, ncols[N], x)) {                // no betas: the candidate is not a pose
      for (int k = 0; k < 9; ++k) cand[N].R[k] = NAN;
      for (int k = 0; k < 3; ++k) cand[N].t[k] = NAN;
      continue;
    }
    {
      if (N == 0) {
        be[0] = sqrt(fabs(x[0]));
        const double sg = x[0] < 0.0 ? -1.0 : 1.0;
        for (int k = 1; k < 4; ++k) be[k] = sg * x[k] / be[0];
      } else {
        two_betas(x[0], x[1], x[2], be);
        if (N == 2) be[2] = be[0] != 0.0 ? x[3] / be[0] : 0.0;
      }
    }
    for (int it = 0; it < kEpnpGnIters; ++it) {         // Gauss-Newton on all four betas
      double pr[10];
      beta_products(be, pr);
      for (int r = 0; r < 6; ++r) {
        const double* l = L[r];
        a[r * 5 + 0] = 2.0 * l[0] * be[0] + l[1] * be[1] + l[3] * be[2] + l[6] * be[3];
        a[r * 5 + 1] = l[1] * be[0] + 2.0 * l[2] * be[1] + l[4] * be[2] + l[7] * be[3];
        a[r * 5 + 2] = l[3] * be[0] + l[4] * be[1] + 2.0 * l[5] * be[2] + l[8] * be[3];
        a[r * 5 + 3] = l[6] * be[0] + l[7] * be[1] + l[8] * be[2] + 2.0 * l[9] * be[3];
        double s = 0.0;
        for (int c = 0; c < 10; ++c) s += l[c] * pr[c];
        bb[r] = rho[r] - s;
      }
      double d[5];
      if (!lstsq6(a, bb, 4, d)) break;
      for (int k = 0; k < 4; ++k) be[k] += d[k];
    }
    // camera control points, the sign that puts the points' depths (their sum) in front, centroids and the cross-covariance
    // sum_i (pw_i - pw~)(pc_i - pc~)^T = sum_jk G_jk (cw_j - pw~)(cc_k - pc~)^T (alphas sum to 1) -> Horn's quaternion
    double cc[4][3];
    for (int j = 0; j < 4; ++j)
      for (int d = 0; d < 3; ++d) cc[j][d] = be[0] * v[0][3 * j + d] + be[1] * v[1][3 * j + d] + be[2] * v[2][3 * j + d] + be[3] * v[3][3 * j + d];
    double zs = 0.0;
    for (int j = 0; j < 4; ++j) zs += as[j] * cc[j][2];
    if (zs < 0.0)
      for (int j = 0; j < 4; ++j)
        for (int d = 0; d < 3; ++d) cc[j][d] = -cc[j][d];
    double pw[3], pc[3];
    for (int d = 0; d < 3; ++d) {
      double sw = 0.0, sc = 0.0;
      for (int j = 0; j < 4; ++j) { sw += as[j] * E.c[j][d]; sc += as[j] * cc[j][d]; }
      pw[d] = sw / m;
      pc[d] = sc / m;
    }
    double S[3][3] = {};
    for (int j = 0; j < 4; ++j)
      for (int k = 0; k < 4; ++k)
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) S[r][c] += Gm[j][k] * (E.c[j][r] - pw[r]) * (cc[k][c] - pc[c]);
    double Nq[16] = {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0],
                     S[1][2] - S[2][1], S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2],
                     S[2][0] - S[0][2], S[0][1] + S[1][0], -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1],
                     S[0][1] - S[1][0], S[2][0] + S[0][2], S[1][2] + S[2][1], -S[0][0] - S[1][1] + S[2][2]};
    double Vq[16];
    jacobi_eigen<4>(Nq, Vq);
    int top = 0;
    for (int i = 1; i < 4; ++i)
      if (Nq[i * 5] > Nq[top * 5]) top = i;
    const double w = Vq[0 * 4 + top], x1 = Vq[1 * 4 + top], y = Vq[2 * 4 + top], z = Vq[3 * 4 + top];
    double* R = cand[N].R;
    R[0] = w * w + x1 * x1 - y * y - z * z; R[1] = 2.0 * (x1 * y - w * z);           R[2] = 2.0 * (x1 * z + w * y);
    R[3] = 2.0 * (x1 * y + w * z);           R[4] = w * w - x1 * x1 + y * y - z * z; R[5] = 2.0 * (y * z - w * x1);
    R[6] = 2.0 * (x1 * z - w * y);           R[7] = 2.0 * (y * z + w * x1);           R[8] = w * w - x1 * x1 - y * y + z * z;
    for (int r = 0; r < 3; ++r) cand[N].t[r] = pc[r] - (R[r * 3] * pw[0] + R[r * 3 + 1] * pw[1] + R[r * 3 + 2] * pw[2]);
  }
}

// the reprojection distance that picks an EPnP candidate
__device__ __forceinline__ double reproj_dist(const Pose& T, const double* Kc, const double* p3, const double* p2) {
  return sqrt(reproj_err2(T, Kc, p3, p2));
}

// the lowest error sum (mean x m), the first on ties; a non-finite error never wins
__device__ __forceinline__ int epnp_pick(const double* err) {
  int best = 0;
  double be = isfinite(err[0]) ? err[0] : INFINITY;
  for (int c = 1; c < 3; ++c)
    if (isfinite(err[c]) && err[c] < be) { be = err[c]; best = c; }
  return best;
}

__device__ __forceinline__ bool pose_finite(const Pose& T) {
  bool f = true;
  for (int k = 0; k < 9; ++k) f &= isfinite(T.R[k]);
  for (int k = 0; k < 3; ++k) f &= isfinite(T.t[k]);
  return f;
}

// OpenCV's RANSAC inlier rule: squared reprojection error <= thr^2, no depth test.  A non-finite error (a pair with a NaN or
// an infinity) is never an inlier, not even at thr = inf.
__device__ __forceinline__ bool epnp_inlier(const Pose& T, const double* Kc, const double* p3, const double* p2, double thr2) {
  const double e = reproj_err2(T, Kc, p3, p2);
  return e <= thr2 && e < INFINITY;
}

// correspondence i of a frame, rounded to fp32 first when kRound (as OpenCV's solvePnPRansac converts its inputs)
template <bool kRound>
__device__ __forceinline__ void load_pair(const double* pts2d, const double* pts3d, size_t i, double* p2, double* p3) {
  for (int d = 0; d < 2; ++d) p2[d] = kRound ? (double)(float)pts2d[i * 2 + d] : pts2d[i * 2 + d];
  for (int d = 0; d < 3; ++d) p3[d] = kRound ? (double)(float)pts3d[i * 3 + d] : pts3d[i * 3 + d];
}

// point p's contribution to the scatter sc[6] = {xx, xy, xz, yy, yz, zz} about c0
__device__ __forceinline__ void add_scatter(const double* p, const double* c0, double* sc) {
  const double d[3] = {p[0] - c0[0], p[1] - c0[1], p[2] - c0[2]};
  sc[0] += d[0] * d[0]; sc[1] += d[0] * d[1]; sc[2] += d[0] * d[2]; sc[3] += d[1] * d[1]; sc[4] += d[1] * d[2]; sc[5] += d[2] * d[2];
}

// EPnP of m <= 5 points by one thread (the RANSAC hypotheses)
__device__ bool epnp_points(const double (*P)[3], const double (*uv)[2], int m, const double* Kc, Pose& out) {
  double sum[3] = {0, 0, 0}, sc[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < m; ++i)
    for (int d = 0; d < 3; ++d) sum[d] += P[i][d];
  const double c0[3] = {sum[0] / m, sum[1] / m, sum[2] / m};
  for (int i = 0; i < m; ++i) add_scatter(P[i], c0, sc);
  EpnpBasis E;
  if (!epnp_basis(sum, sc, m, E)) return false;
  double acc[kEpnpSums];
  for (int k = 0; k < kEpnpSums; ++k) acc[k] = 0.0;
  for (int i = 0; i < m; ++i) {
    double a[4];
    epnp_alphas(E, P[i], a);
    epnp_accumulate(a, uv[i], Kc, acc);
  }
  Pose cand[3];
  epnp_candidates(acc, E, m, cand);
  double err[3] = {0, 0, 0};
  for (int i = 0; i < m; ++i)
    for (int c = 0; c < 3; ++c) err[c] += reproj_dist(cand[c], Kc, P[i], uv[i]);
  out = cand[epnp_pick(err)];
  return pose_finite(out);
}

// block-wide fixed-order sum of K per-thread values into out[K] (shared); every thread returns with out complete
constexpr int kEpnpThreads = kRefineThreads;
template <int K>
__device__ void block_sum(double* v, double (*red)[kEpnpThreads / 32], double* out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = v[k];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[k][warp] = s;
  }
  __syncthreads();
  for (int k = tid; k < K; k += kEpnpThreads) {
    double s = 0.0;
    for (int w = 0; w < kEpnpThreads / 32; ++w) s += red[k][w];
    out[k] = s;
  }
  __syncthreads();
}

struct EpnpShared {
  double red[kEpnpSums][kEpnpThreads / 32];
  double sums[kEpnpSums];
  EpnpBasis E;
  Pose cand[3];
  int ok;
};

// EPnP of the frame's correspondences i in [0, n) with use(i) by the whole block; the pose lands in *out (shared).  Returns
// the number of points used, or 0 for a degenerate set (then, as with fewer than 4 points, *out is not written).
template <bool kRound, class Use>
__device__ int epnp_block(const double* pts2d, const double* pts3d, int n, const double* Kc, Use use, EpnpShared& sh, Pose* out) {
  const int tid = threadIdx.x;
  double v[4] = {0, 0, 0, 0};
  for (int i = tid; i < n; i += kEpnpThreads) {
    if (!use(i)) continue;
    double p2[2], p3[3];
    load_pair<kRound>(pts2d, pts3d, i, p2, p3);
    v[0] += p3[0]; v[1] += p3[1]; v[2] += p3[2]; v[3] += 1.0;
  }
  block_sum<4>(v, sh.red, sh.sums);
  const int m = (int)sh.sums[3];
  if (m < 4) return m;
  const double sum[3] = {sh.sums[0], sh.sums[1], sh.sums[2]};
  const double c0[3] = {sum[0] / m, sum[1] / m, sum[2] / m};
  double sc[6] = {0, 0, 0, 0, 0, 0};
  for (int i = tid; i < n; i += kEpnpThreads) {
    if (!use(i)) continue;
    double p2[2], p3[3];
    load_pair<kRound>(pts2d, pts3d, i, p2, p3);
    add_scatter(p3, c0, sc);
  }
  block_sum<6>(sc, sh.red, sh.sums);
  if (tid == 0) sh.ok = epnp_basis(sum, sh.sums, m, sh.E) ? 1 : 0;
  __syncthreads();
  if (!sh.ok) return 0;
  double acc[kEpnpSums];
#pragma unroll
  for (int k = 0; k < kEpnpSums; ++k) acc[k] = 0.0;
  for (int i = tid; i < n; i += kEpnpThreads) {
    if (!use(i)) continue;
    double p2[2], p3[3], a[4];
    load_pair<kRound>(pts2d, pts3d, i, p2, p3);
    epnp_alphas(sh.E, p3, a);
    epnp_accumulate(a, p2, Kc, acc);
  }
  block_sum<kEpnpSums>(acc, sh.red, sh.sums);
  if (tid == 0) epnp_candidates(sh.sums, sh.E, m, sh.cand);
  __syncthreads();
  double err[3] = {0, 0, 0};
  for (int i = tid; i < n; i += kEpnpThreads) {
    if (!use(i)) continue;
    double p2[2], p3[3];
    load_pair<kRound>(pts2d, pts3d, i, p2, p3);
    for (int c = 0; c < 3; ++c) err[c] += reproj_dist(sh.cand[c], Kc, p3, p2);
  }
  block_sum<3>(err, sh.red, sh.sums);
  if (tid == 0) *out = sh.cand[epnp_pick(sh.sums)];
  __syncthreads();
  return m;
}

// the end of both EPnP selectors: the winner's pose W, its inlier set (inlier(p3, p2) on the fp32-rounded pairs) as the mask,
// EPnP on that set; a degenerate set keeps W.  count: the mask's count, which the winner's own count is (the same test).
template <class Inlier>
__device__ __forceinline__ void refit_tail(int b, const Frame& f, const Pose& W, Inlier inlier, int count, EpnpShared& sh, Pose* T,
                                           double* pose_out, int* inlier_mask, int* n_inliers) {
  auto use = [&](int i) {
    double p2[2], p3[3];
    load_pair<true>(f.p2, f.p3, i, p2, p3);
    return inlier(p3, p2);
  };
  for (int i = threadIdx.x; i < f.n; i += kEpnpThreads) inlier_mask[f.o0 + i] = use(i) ? 1 : 0;
  const int m = epnp_block<true>(f.p2, f.p3, f.n, f.Kc, use, sh, T);
  if (threadIdx.x == 0) {
    write_pose(m >= 4 && pose_finite(*T) ? *T : W, pose_out + (size_t)b * 12);
    n_inliers[b] = count;
  }
}

// one block per frame: EPnP on all of its correspondences (cv2.solvePnP(..., flags=SOLVEPNP_EPNP) for B frames)
__global__ void __launch_bounds__(kEpnpThreads) epnp_frames(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                            const int* __restrict__ offsets, double* __restrict__ pose_out, int* __restrict__ status) {
  __shared__ EpnpShared sh;
  __shared__ Pose T;
  const int b = blockIdx.x;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  const int m = f.n >= 4 ? epnp_block<false>(f.p2, f.p3, f.n, f.Kc, [](int) { return true; }, sh, &T) : 0;
  if (threadIdx.x == 0) {
    const bool ok = m >= 4 && pose_finite(T);
    if (ok) write_pose(T, pose_out + (size_t)b * 12);
    else write_identity(pose_out + (size_t)b * 12);
    status[b] = ok ? 1 : 0;
  }
}

// the model of a frame of exactly 4 correspondences (fp32-rounded): P3P on 0-2, the solution that best reprojects 3
__device__ __forceinline__ bool four_pair_model(const double* f2, const double* f3, const double* Kc, Pose& T) {
  double P[4][3], uv[4][2], j[3][3];
  for (int k = 0; k < 4; ++k) load_pair<true>(f2, f3, k, uv[k], P[k]);
  for (int k = 0; k < 3; ++k) bearing(Kc, uv[k], j[k]);
  Pose sol[4];
  const int ns = p3p(P, j, sol);
  double be = INFINITY;
  bool ok = false;
  for (int s = 0; s < ns; ++s) {
    const double e = reproj_dist(sol[s], Kc, P[3], uv[3]);
    if (e < be) { be = e; T = sol[s]; ok = true; }
  }
  return ok;
}

// EPnP-RANSAC hypotheses: one thread per sample of five distinct correspondences (fp32-rounded), EPnP on them, inliers over
// all n by OpenCV's rule; a frame of exactly 4 correspondences uses P3P on 0-2, the solution that best reprojects 3
__global__ void __launch_bounds__(kHypThreads) epnp_hypotheses(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                               const int* __restrict__ offsets, int H, double thr2, unsigned long long seed,
                                                               double* __restrict__ hyp) {
  const int b = blockIdx.x;
  const int h = blockIdx.y * blockDim.x + threadIdx.x;
  if (h >= H) return;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  double* out = hyp + ((size_t)b * H + h) * kHypStride;
  out[0] = 0.0;
  if (f.n < 4) return;
  Pose T;
  bool ok = false;
  if (f.n == 4) {
    ok = four_pair_model(f.p2, f.p3, f.Kc, T);
  } else {
    int idx[5];
    sample_distinct<5>(seed, b, h, f.n, idx);
    double P[5][3], uv[5][2];
    for (int k = 0; k < 5; ++k) load_pair<true>(f.p2, f.p3, idx[k], uv[k], P[k]);
    ok = epnp_points(P, uv, 5, f.Kc, T);
  }
  if (!ok || !pose_finite(T)) return;
  int cnt = 0;
  for (int i = 0; i < f.n; ++i) {
    double p2[2], p3[3];
    load_pair<true>(f.p2, f.p3, i, p2, p3);
    cnt += epnp_inlier(T, f.Kc, p3, p2, thr2) ? 1 : 0;
  }
  if (cnt == 0) return;
  store_record(out, (double)cnt, T);
}

// one block per frame: the best hypothesis, its inlier set (the reported mask), EPnP on that set
__global__ void __launch_bounds__(kEpnpThreads) epnp_select_refit(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                                  const int* __restrict__ offsets, int H, double thr2, const double* __restrict__ hyp,
                                                                  double* __restrict__ pose_out, int* __restrict__ inlier_mask, int* __restrict__ n_inliers) {
  __shared__ unsigned long long best_key[kRefineThreads];
  __shared__ EpnpShared sh;
  __shared__ Pose W, T;
  const int b = blockIdx.x;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  int best_h;
  const int best_cnt = best_hypothesis(hyp, b, H, best_key, &best_h);
  if (best_cnt < 4) {
    write_no_model(b, f, pose_out, inlier_mask, n_inliers);
    return;
  }
  if (threadIdx.x == 0) W = load_record(hyp + ((size_t)b * H + best_h) * kHypStride);
  __syncthreads();
  const Pose Wl = W;
  refit_tail(b, f, W, [&](const double* p3, const double* p2) { return epnp_inlier(Wl, f.Kc, p3, p2, thr2); }, best_cnt, sh, &T, pose_out,
             inlier_mask, n_inliers);
}

// ---- EPnP-RANSAC as OpenCV runs it (RANSACPointSetRegistrator::run, calib3d/src/ptsetreg.cpp): OpenCV's sample sequence,
// its fp32 inlier count and its confidence-driven stopping rule, evaluated in waves of W samples per frame.
//   cv_scan (wave -1)  per frame: the state below, and wave 0's samples;
//   cv_wave (wave w)   one thread per sample w*W + h below the frame's budget: EPnP (epnp_points) and the fp32 count;
//   cv_scan (wave w)   per frame, in sample order: the loop's bookkeeping, then wave w+1's samples unless the loop ended;
//   cv_select_refit    the winner's inlier set as the mask, EPnP on it.
// A frame whose loop ended skips every later launch at its first instruction.
constexpr int kCvModelPoints = 5;
constexpr int kCvScanThreads = 32;

struct CvState {                                       // per frame, 16 doubles at the end of the workspace
  Pose pose;                                           // the winning sample's R (9) and t (3)
  unsigned long long rng;                              // cv::RNG state after the samples drawn so far
  int niters;                                          // the loop's budget (only ever lowered)
  int iter;                                            // the iter at which the loop exited, once done
  int best;                                            // maxGoodCount
  int winner;                                          // index of the winning sample, -1 for none
  int done;
  int pad;
};
static_assert(sizeof(CvState) == 16 * sizeof(double), "CvState is 16 doubles");

// PnPRansacCallback::computeError of one fp32-rounded pair: projectPoints in fp64 (x * (1/z), then * f + c; OpenCV's
// distortion and tilt terms are exact no-ops for zero coefficients) rounded to fp32, the squared distance in fp32.  Explicit
// roundings: no FMA contraction, as in OpenCV's x86 build, and the same value in every kernel that asks.
__device__ __forceinline__ float cv_error(const Pose& T, const double* Kc, const double* p3, const double* p2) {
  double X[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    X[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.R[r * 3], p3[0]), __dmul_rn(T.R[r * 3 + 1], p3[1])), __dmul_rn(T.R[r * 3 + 2], p3[2])), T.t[r]);
  const double iz = X[2] != 0.0 ? __ddiv_rn(1.0, X[2]) : 1.0;
  const float u = (float)__dadd_rn(__dmul_rn(__dmul_rn(X[0], iz), Kc[0]), Kc[2]);
  const float v = (float)__dadd_rn(__dmul_rn(__dmul_rn(X[1], iz), Kc[1]), Kc[3]);
  const float du = __fsub_rn((float)p2[0], u), dv = __fsub_rn((float)p2[1], v);
  return __fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv));
}

// OpenCV's fp32 inlier rule on cv_error; a non-finite error is never an inlier (OpenCV counts an infinite one at thr = inf)
__device__ __forceinline__ bool cv_inlier(float e, float thr2f) { return e <= thr2f && e < INFINITY; }

// samples first .. first + W - 1 of frame b, those below its budget niters, into the wave's records (one warp).  Every lane
// passes its own copy of the budget: lane 0's store to S.niters need not be what the other lanes read back.
__device__ void draw_wave(CvState& S, double* r, int n, int W, int first, int niters, int b, int* trace_samples, int trace_cap) {
  const int count = min(W, niters - first);
  unsigned long long s = S.rng;
  if (count > 0)
    cvrng::warp_draw<kCvModelPoints>(s, first == 0, (unsigned)n, count, reinterpret_cast<int*>(r), kHypStride * 2, trace_samples + (trace_samples ? (size_t)b * trace_cap * kCvModelPoints : 0),
              first, trace_cap);
  if ((threadIdx.x & 31) == 0) S.rng = s;
}

// wave < 0: initialise frame b's state and draw wave 0.  wave >= 0: run the loop over wave w's counts, then draw wave w+1.
// A frame of 4 or 5 pairs (model_points == npoints in solvePnPRansac) has one model, of every pair, and no loop.
// One warp per frame: the loop reads 32 counts at a time and finds the next sample that wins or ends the loop by a ballot
// (wins are rare); every lane keeps the same copy of the loop's state.  Lane 0 draws the samples.
__global__ void __launch_bounds__(kCvScanThreads) epnp_cv_scan(const int* __restrict__ offsets, int H, int W, int wave, double confidence,
                                                              CvState* __restrict__ st, double* __restrict__ rec, int* __restrict__ trace_samples,
                                                              int trace_cap) {
  const int b = blockIdx.x, lane = threadIdx.x;
  CvState& S = st[b];
  const int n = offsets[b + 1] - offsets[b];
  double* r = rec + (size_t)b * W * kHypStride;
  if (wave >= 0 && n > kCvModelPoints) {
    if (S.done) return;
    const int base = wave * W;
    int niters = S.niters, best = S.best, winner = S.winner, done = 0, iter = 0;
    for (int h0 = 0; h0 < W && !done; h0 += kCvScanThreads) {
      const int h = h0 + lane;
      const int c = h < W ? (int)r[(size_t)h * kHypStride] : -1;
      int from = 0;                                    // lanes below it are done with
      while (true) {
        const bool event = lane >= from && h < W && (c > max(best, kCvModelPoints - 1) || base + h + 1 >= niters);
        const unsigned mask = __ballot_sync(0xffffffffu, event);
        if (!mask) break;
        const int e = __ffs(mask) - 1, i = base + h0 + e;
        const int ce = __shfl_sync(0xffffffffu, c, e);
        if (ce > max(best, kCvModelPoints - 1)) {      // strict: the earliest sample wins a tie
          best = ce;
          winner = i;
          if (lane == 0) S.pose = load_record(r + (size_t)(h0 + e) * kHypStride);
          niters = cvrng::update_num_iters(confidence, (double)(n - ce) / n, kCvModelPoints, niters);
        }
        if (i + 1 >= niters) { done = 1; iter = i + 1; break; }
        from = e + 1;
      }
    }
    if (lane == 0) {
      S.niters = niters;
      S.best = best;
      S.winner = winner;
      S.done = done;
      S.iter = iter;
    }
    if (done) return;
    __syncwarp();
    draw_wave(S, r, n, W, base + W, niters, b, trace_samples, trace_cap);
    return;
  }
  if (wave < 0) {
    if (lane == 0) {
      S.rng = ~0ull;                                   // run() builds RNG rng((uint64)-1) on every call
      S.niters = n <= kCvModelPoints ? 1 : H;          // 4 or 5 pairs: one model, sample 0 = every pair in order
      S.iter = 0;
      S.best = 0;
      S.winner = -1;
      S.done = n < 4 ? 1 : 0;
      if (n >= 4 && n <= kCvModelPoints) {
        int* si = reinterpret_cast<int*>(r);
        for (int k = 0; k < kCvModelPoints; ++k) si[k] = k;
      }
    }
    if (n <= kCvModelPoints) return;
    __syncwarp();                                      // lane 0's state is visible to the warp
    draw_wave(S, r, n, W, 0, H, b, trace_samples, trace_cap);
    return;
  }
  if (lane != 0 || S.done) return;                     // wave >= 0, 4 or 5 pairs: take the one model
  const int c = (int)r[0];
  if (c >= 0) {
    S.winner = 0;
    S.best = n;
    S.pose = load_record(r);
  }
  S.done = 1;
}

// one thread per sample of the wave: its five indices (written over by its record), EPnP, OpenCV's count.  Record count -1:
// no model (OpenCV's runKernel failing), which never wins.  Samples at or past the frame's budget are not needed.
__global__ void __launch_bounds__(kHypThreads) epnp_cv_wave(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                            const int* __restrict__ offsets, int W, int wave, float thr2f, const CvState* __restrict__ st,
                                                            double* __restrict__ rec, int* __restrict__ trace_counts, int trace_cap) {
  const int b = blockIdx.x;
  const int h = blockIdx.y * blockDim.x + threadIdx.x;
  if (h >= W) return;
  const CvState& S = st[b];
  const int i = wave * W + h;
  if (S.done || i >= S.niters) return;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  double* out = rec + ((size_t)b * W + h) * kHypStride;
  Pose T;
  bool ok;
  if (f.n == 4) {
    ok = four_pair_model(f.p2, f.p3, f.Kc, T);
  } else {
    const int* si = reinterpret_cast<const int*>(out);
    double P[5][3], uv[5][2];
    for (int k = 0; k < 5; ++k) load_pair<true>(f.p2, f.p3, si[k], uv[k], P[k]);
    ok = epnp_points(P, uv, 5, f.Kc, T);
  }
  int cnt = -1;
  if (ok && pose_finite(T)) {
    cnt = 0;
    for (int j = 0; j < f.n; ++j) {
      double p2[2], p3[3];
      load_pair<true>(f.p2, f.p3, j, p2, p3);
      cnt += cv_inlier(cv_error(T, f.Kc, p3, p2), thr2f) ? 1 : 0;
    }
  }
  store_record(out, (double)cnt, T);
  if (trace_counts && i < trace_cap) trace_counts[(size_t)b * trace_cap + i] = cnt;
}

// one block per frame: the winner's inlier set as the mask, EPnP on it, the iteration count.  A frame of 4 or 5 pairs keeps
// its one model (solvePnP(P3P) / solvePnP(EPNP) on every pair in solvePnPRansac), every pair an inlier, with no refit.
__global__ void __launch_bounds__(kEpnpThreads) epnp_cv_select_refit(const double* __restrict__ Kmat, const double* __restrict__ pts2d, const double* __restrict__ pts3d,
                                                                     const int* __restrict__ offsets, float thr2f, const CvState* __restrict__ st,
                                                                     double* __restrict__ pose_out, int* __restrict__ inlier_mask, int* __restrict__ n_inliers,
                                                                     int* __restrict__ iterations, int* __restrict__ trace_winner) {
  __shared__ EpnpShared sh;
  __shared__ Pose T;
  const int b = blockIdx.x, tid = threadIdx.x;
  const Frame f = frame_view(b, Kmat, pts2d, pts3d, offsets);
  const CvState& S = st[b];
  const int winner = S.winner;
  if (tid == 0) {
    iterations[b] = S.iter;
    if (trace_winner) trace_winner[b] = winner;
  }
  if (winner < 0) {                                    // run() returns false
    write_no_model(b, f, pose_out, inlier_mask, n_inliers);
    return;
  }
  const Pose Wl = S.pose;
  if (f.n <= kCvModelPoints) {
    for (int i = tid; i < f.n; i += kEpnpThreads) inlier_mask[f.o0 + i] = 1;
    if (tid == 0) {
      write_pose(Wl, pose_out + (size_t)b * 12);
      n_inliers[b] = f.n;
    }
    return;
  }
  refit_tail(b, f, Wl, [&](const double* p3, const double* p2) { return cv_inlier(cv_error(Wl, f.Kc, p3, p2), thr2f); }, S.best, sh, &T, pose_out,
             inlier_mask, n_inliers);
}

// the first `count` samples of a frame of n pairs, by the generator epnp_cv_scan uses (one warp), in calls of `chunk`
__global__ void epnp_cv_subsets(int n, int count, int chunk, int* __restrict__ out) {
  unsigned long long s = ~0ull;
  for (int i = 0; i < count; i += chunk)
    cvrng::warp_draw<kCvModelPoints>(s, i == 0, (unsigned)n, min(chunk, count - i), out + (size_t)i * kCvModelPoints, kCvModelPoints, nullptr, 0, 0);
}

// ---- matched pairs -> the ragged correspondence lists above (reference inference.py:147-152: valid = matches > -1;
// mkpts2d = kpts2d[valid]; mkpts3d = kpts3d[matches[valid]]).  Three launches, no workspace: per-frame counts into
// offsets[1..B], an in-place scan of offsets, then a per-frame ordered compaction (ascending n, numpy boolean-mask order).
// Frames of different objects: frame b's 3D key points are rows [kp3_first[b], kp3_first[b] + kp3_count[b]) of the concatenated
// keypoints3d; kp3_first == nullptr: one object of M rows for every frame.
constexpr int kGatherThreads = 256;

__device__ __forceinline__ bool is_match(int64_t m, int M) { return m >= 0 && m < (int64_t)M; }
__device__ __forceinline__ int frame_kp3_count(const int* kp3_count, int b, int M) { return kp3_count ? kp3_count[b] : M; }

__global__ void __launch_bounds__(kGatherThreads) gather_count(const int64_t* __restrict__ matches0, int N, int M_all,
                                                               const int* __restrict__ kp3_count, int* __restrict__ offsets) {
  __shared__ int cnt_w[kGatherThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int M = frame_kp3_count(kp3_count, b, M_all);
  const int64_t* m0 = matches0 + (size_t)b * N;
  int cnt = 0;
  for (int n = tid; n < N; n += kGatherThreads) cnt += is_match(m0[n], M) ? 1 : 0;
  cnt = block_reduce(cnt, Sum32(), cnt_w);
  if (tid == 0) {
    offsets[b + 1] = cnt;
    if (b == 0) offsets[0] = 0;
  }
}

// one block: inclusive scan of offsets[1..B] in place (offsets[0] = 0), tiles of 1024 with a running carry
constexpr int kScanThreads = 1024;
__global__ void __launch_bounds__(kScanThreads) gather_scan(int B, int* __restrict__ offsets) {
  __shared__ int sh[kScanThreads / 32];
  int carry = 0;
  for (int base = 0; base < B; base += kScanThreads) {
    const int i = base + (int)threadIdx.x;
    const int v = i < B ? offsets[i + 1] : 0;
    int total;
    const int exc = block_scan(v, Sum32(), 0, sh, &total);
    if (i < B) offsets[i + 1] = carry + exc + v;
    carry += total;
  }
}

// one block per frame: ordered compaction over tiles of kGatherThreads entries; keypoints2d rows are read for matches only
__global__ void __launch_bounds__(kGatherThreads) gather_compact(const int64_t* __restrict__ matches0, const float* __restrict__ mscores0,
                                                                 const float* __restrict__ kp2d, const float* __restrict__ kp3d_all, int N, int M_all,
                                                                 const int* __restrict__ kp3_first, const int* __restrict__ kp3_count,
                                                                 const int* __restrict__ offsets, double* __restrict__ pts2d, double* __restrict__ pts3d,
                                                                 float* __restrict__ mconf, int* __restrict__ query_index) {
  __shared__ int sh[kGatherThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int M = frame_kp3_count(kp3_count, b, M_all);
  const float* kp3d = kp3d_all + (kp3_first ? (size_t)kp3_first[b] * 3 : 0);
  const size_t row0 = (size_t)b * N;
  int pos = offsets[b];
  for (int base = 0; base < N; base += kGatherThreads) {
    const int n = base + tid;
    const int64_t m = n < N ? matches0[row0 + n] : -1;
    const bool valid = is_match(m, M);
    int total;
    const int rank = block_rank(valid, sh, &total);
    if (valid) {
      const size_t o = (size_t)(pos + rank);
      const float* k2 = kp2d + (row0 + n) * 2;
      const float* k3 = kp3d + (size_t)m * 3;
      pts2d[o * 2 + 0] = (double)k2[0];
      pts2d[o * 2 + 1] = (double)k2[1];
      pts3d[o * 3 + 0] = (double)k3[0];
      pts3d[o * 3 + 1] = (double)k3[1];
      pts3d[o * 3 + 2] = (double)k3[2];
      if (mconf) mconf[o] = mscores0[row0 + n];
      if (query_index) query_index[o] = n;
    }
    pos += total;
  }
}

}  // namespace
}  // namespace opb

// The gather of both entry points: kp3_first / kp3_count == nullptr means one object of M key points for every frame.
static int gather_matches_impl(const char* fn, const int64_t* matches0, const float* mscores0, const float* keypoints2d, const float* keypoints3d,
                               int32_t B, int32_t N, int32_t M, const int32_t* kp3_first, const int32_t* kp3_count, double* pts2d, double* pts3d,
                               float* mconf, int32_t* query_index, int32_t* offsets, void* stream) {
  REQUIRE(fn, N == 0 || (matches0 && keypoints2d && pts2d && pts3d));
  REQUIRE(fn, !mconf || mscores0);
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) {
    CK(opb::no_handle_error, cudaMemsetAsync(offsets, 0, sizeof(int32_t) * ((size_t)B + 1), st));
    return OPB_OK;
  }
  LAUNCH_NH(fn, opb::gather_count, (unsigned)B, opb::kGatherThreads, 0, st, matches0, N, M, kp3_count, offsets);
  LAUNCH_NH(fn, opb::gather_scan, 1, opb::kScanThreads, 0, st, B, offsets);
  LAUNCH_NH(fn, opb::gather_compact, (unsigned)B, opb::kGatherThreads, 0, st, matches0, mscores0, keypoints2d, keypoints3d, N, M, kp3_first, kp3_count,
            offsets, pts2d, pts3d, mconf, query_index);
  return OPB_OK;
}

extern "C" int opb_gather_matches(const int64_t* matches0, const float* mscores0, const float* keypoints2d, const float* keypoints3d,
                                  int32_t B, int32_t N, int32_t M, double* pts2d, double* pts3d, float* mconf, int32_t* query_index,
                                  int32_t* offsets, void* stream) {
  REQUIRE(__func__, B > 0 && N >= 0 && M > 0 && keypoints3d && offsets && (int64_t)B * N <= (int64_t)INT32_MAX);
  return gather_matches_impl(__func__, matches0, mscores0, keypoints2d, keypoints3d, B, N, M, nullptr, nullptr, pts2d, pts3d, mconf, query_index,
                             offsets, stream);
}

extern "C" int opb_gather_matches_objects(const int64_t* matches0, const float* mscores0, const float* keypoints2d, const float* keypoints3d,
                                          const int32_t* kp3_first, const int32_t* kp3_count, int32_t B, int32_t N, double* pts2d, double* pts3d,
                                          float* mconf, int32_t* query_index, int32_t* offsets, void* stream) {
  REQUIRE(__func__, B > 0 && N >= 0 && keypoints3d && kp3_first && kp3_count && offsets && (int64_t)B * N <= (int64_t)INT32_MAX);
  return gather_matches_impl(__func__, matches0, mscores0, keypoints2d, keypoints3d, B, N, 0, kp3_first, kp3_count, pts2d, pts3d, mconf, query_index,
                             offsets, stream);
}

// the arguments every RANSAC entry point takes
static int check_ransac_args(const char* fn, const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B,
                             int32_t hypotheses, double reproj_error, const double* workspace, const double* pose_out, const int32_t* inlier_mask,
                             const int32_t* n_inliers) {
  REQUIRE(fn, K && pts2d && pts3d && offsets && workspace && pose_out && inlier_mask && n_inliers);
  REQUIRE(fn, B > 0 && hypotheses > 0 && hypotheses <= opb::kMaxHypotheses && reproj_error > 0.0);
  return OPB_OK;
}

// a RANSAC of a fixed number of hypotheses: one thread per hypothesis record, then one block per frame selects
template <class HypothesesKernel, class SelectKernel>
static int ransac_fixed(const char* fn, HypothesesKernel hypotheses_kernel, SelectKernel select_kernel, const double* K, const double* pts2d,
                        const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses, double reproj_error, uint64_t seed,
                        double* workspace, double* pose_out, int32_t* inlier_mask, int32_t* n_inliers, void* stream) {
  if (int rc = check_ransac_args(fn, K, pts2d, pts3d, offsets, B, hypotheses, reproj_error, workspace, pose_out, inlier_mask, n_inliers)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const double thr2 = reproj_error * reproj_error;
  LAUNCH_NH(fn, hypotheses_kernel, dim3((unsigned)B, (unsigned)((hypotheses + opb::kHypThreads - 1) / opb::kHypThreads)), opb::kHypThreads, 0, st,
            K, pts2d, pts3d, offsets, hypotheses, thr2, (unsigned long long)seed, workspace);
  LAUNCH_NH(fn, select_kernel, (unsigned)B, opb::kRefineThreads, 0, st, K, pts2d, pts3d, offsets, hypotheses, thr2, workspace, pose_out, inlier_mask,
            n_inliers);
  return OPB_OK;
}

extern "C" int opb_ransac_pnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                              double reproj_error, uint64_t seed, double* workspace, double* pose_out, int32_t* inlier_mask, int32_t* n_inliers,
                              void* stream) {
  return ransac_fixed(__func__, opb::pnp_hypotheses, opb::pnp_select_refine, K, pts2d, pts3d, offsets, B, hypotheses, reproj_error, seed, workspace,
                      pose_out, inlier_mask, n_inliers, stream);
}

extern "C" int opb_epnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, double* pose_out,
                        int32_t* status, void* stream) {
  REQUIRE(__func__, K && pts2d && pts3d && offsets && pose_out && status && B > 0);
  LAUNCH_NH(__func__, opb::epnp_frames, (unsigned)B, opb::kEpnpThreads, 0, (cudaStream_t)stream, K, pts2d, pts3d, offsets, pose_out, status);
  return OPB_OK;
}

extern "C" int opb_ransac_epnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                               double reproj_error, uint64_t seed, double* workspace, double* pose_out, int32_t* inlier_mask, int32_t* n_inliers,
                               void* stream) {
  return ransac_fixed(__func__, opb::epnp_hypotheses, opb::epnp_select_refit, K, pts2d, pts3d, offsets, B, hypotheses, reproj_error, seed, workspace,
                      pose_out, inlier_mask, n_inliers, stream);
}

// test hooks of opb_ransac_epnp_cv (host-side settings read at launch; the launch sequence does not change)
static int g_cv_wave = 0;                               // samples per frame and wave; 0 = chosen from B
static int32_t* g_cv_trace_samples = nullptr;
static int32_t* g_cv_trace_counts = nullptr;
static int32_t* g_cv_trace_winner = nullptr;
static int g_cv_trace_cap = 0;

extern "C" int opb_debug_set_cv_wave(int32_t wave) {
  REQUIRE(__func__, wave >= 0);
  g_cv_wave = wave;
  return OPB_OK;
}

extern "C" int opb_debug_set_cv_trace(int32_t* samples, int32_t* counts, int32_t* winner, int32_t capacity) {
  REQUIRE(__func__, capacity > 0 || (capacity == 0 && !samples && !counts));
  g_cv_trace_samples = samples;
  g_cv_trace_counts = counts;
  g_cv_trace_winner = winner;
  g_cv_trace_cap = capacity;
  return OPB_OK;
}

extern "C" int opb_debug_cv_subsets(int32_t n, int32_t count, int32_t chunk, int32_t* out, void* stream) {
  REQUIRE(__func__, n >= 5 && count > 0 && chunk > 0 && out);
  LAUNCH_NH(__func__, opb::epnp_cv_subsets, 1, 32, 0, (cudaStream_t)stream, n, count, chunk, out);
  return OPB_OK;
}

// samples per frame and wave: B x W about one 128-thread block per SM.  A wave's time is one thread's EPnP latency (about
// 2.5 ms on an H100) up to roughly that many threads, and grows with the thread count beyond it (tools/epnp_cv_bench.py,
// DESIGN 5.4): smaller waves add waves without saving time, larger ones evaluate samples the loop may never need.  Whole
// blocks, at most the budget.  OPB_E_CUDA if the device query fails.
static int cv_wave_size(int B, int H) {
  int w = g_cv_wave;
  if (w == 0) {
    int dev = 0, sms = 0;
    CK(opb::no_handle_error, cudaGetDevice(&dev));
    CK(opb::no_handle_error, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int target = sms * opb::kHypThreads;
    w = (target / B + opb::kHypThreads - 1) / opb::kHypThreads * opb::kHypThreads;
    w = w < opb::kHypThreads ? opb::kHypThreads : w;
  }
  return w < H ? w : H;
}

extern "C" int opb_ransac_epnp_cv(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                                  double reproj_error, double confidence, double* workspace, double* pose_out, int32_t* inlier_mask,
                                  int32_t* n_inliers, int32_t* iterations, void* stream) {
  if (int rc = check_ransac_args(__func__, K, pts2d, pts3d, offsets, B, hypotheses, reproj_error, workspace, pose_out, inlier_mask, n_inliers))
    return rc;
  REQUIRE(__func__, iterations && confidence >= 0.0 && confidence <= 1.0);
  cudaStream_t st = (cudaStream_t)stream;
  // solvePnPRansac takes a float reprojectionError; findInliers squares it in double (exact) and rounds to float: the fp32
  // square of the fp32 threshold, which differs from (float)(reproj_error^2) by an ulp for about half of all thresholds
  const float thr_f = (float)reproj_error;
  const float thr2f = thr_f * thr_f;
  const int W = cv_wave_size(B, hypotheses);
  if (W < 0) return W;
  const int waves = (hypotheses + W - 1) / W;
  opb::CvState* state = reinterpret_cast<opb::CvState*>(workspace + (size_t)B * hypotheses * opb::kHypStride);
  int* ts = g_cv_trace_samples;
  int* tc = g_cv_trace_counts;
  const int cap = g_cv_trace_cap;
  LAUNCH_NH(__func__, opb::epnp_cv_scan, (unsigned)B, opb::kCvScanThreads, 0, st, offsets, hypotheses, W, -1, confidence, state, workspace, ts, cap);
  for (int w = 0; w < waves; ++w) {
    LAUNCH_NH(__func__, opb::epnp_cv_wave, dim3((unsigned)B, (unsigned)((W + opb::kHypThreads - 1) / opb::kHypThreads)), opb::kHypThreads, 0, st,
              K, pts2d, pts3d, offsets, W, w, thr2f, state, workspace, tc, cap);
    LAUNCH_NH(__func__, opb::epnp_cv_scan, (unsigned)B, opb::kCvScanThreads, 0, st, offsets, hypotheses, W, w, confidence, state, workspace, ts, cap);
  }
  LAUNCH_NH(__func__, opb::epnp_cv_select_refit, (unsigned)B, opb::kEpnpThreads, 0, st, K, pts2d, pts3d, offsets, thr2f, state, pose_out, inlier_mask,
            n_inliers, iterations, g_cv_trace_winner);
  return OPB_OK;
}
