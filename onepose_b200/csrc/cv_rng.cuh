// OpenCV's RANSAC sample sequence on the device (RANSACPointSetRegistrator::run and getSubset, calib3d/src/ptsetreg.cpp),
// for any number K of model points: cv::RNG((uint64)-1), K distinct indices uniform(0, n) per sample (an index repeating an
// earlier one of the sample is redrawn), and RANSACUpdateNumIters.  Used by the EPnP loop (pnp_ransac.cu, K = 5) and the
// partial-affine loop (detect.cu, K = 2); the numpy model is tests/opencv_ransac_reference.py.
#pragma once

#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

namespace opb {
namespace cvrng {

constexpr unsigned kMwcA = 4164903690u;                                                   // cv::RNG's multiplier (CV_RNG_COEFF)
constexpr unsigned long long kMwcM = (unsigned long long)kMwcA * 4294967296ull - 1ull;   // the LCG modulus of the MWC

__device__ __forceinline__ unsigned mwc_next(unsigned long long& s) {   // cv::RNG::next
  s = (unsigned long long)(unsigned)s * kMwcA + (s >> 32);
  return (unsigned)s;
}

// x % n for 32-bit x by a 64-bit reciprocal m = 2^64 / n rounded up (Lemire, Kaser, Kurz 2019): exact for every 32-bit x, n
__device__ __forceinline__ unsigned fast_mod(unsigned x, unsigned long long m, unsigned n) { return (unsigned)__umul64hi(m * x, n); }
__host__ __device__ __forceinline__ unsigned long long fast_mod_m(unsigned n) { return ~0ull / n + 1; }

// K draws uniform(0, n) from state t (advanced) into v; true when they are distinct
template <int K>
__device__ __forceinline__ bool draw(unsigned long long& t, unsigned long long m, unsigned n, int* v) {
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = (int)fast_mod(mwc_next(t), m, n);
  bool distinct = true;
#pragma unroll
  for (int a = 0; a < K; ++a)
#pragma unroll
    for (int c = a + 1; c < K; ++c) distinct &= v[a] != v[c];
  return distinct;
}

// getSubset with a checkSubset that accepts every sample: K indices uniform(0, n), an index repeating an earlier one of the
// sample redrawn.  K distinct draws in a row (the common case for large n) take one branch-free pass.
template <int K>
__device__ __forceinline__ void subset(unsigned long long& s, unsigned n, unsigned long long m, int* idx) {
  unsigned long long t = s;
  int v[K];
  if (draw<K>(t, m, n, v)) {
    s = t;
#pragma unroll
    for (int k = 0; k < K; ++k) idx[k] = v[k];
    return;
  }
  for (int i = 0; i < K; ++i) {
    int u;
    bool rep;
    do {
      u = (int)fast_mod(mwc_next(s), m, n);
      rep = false;
      for (int e = 0; e < i; ++e) rep |= idx[e] == u;
    } while (rep);
    idx[i] = u;
  }
}

// RANSACUpdateNumIters: clamps, DBL_MIN guards and cvRound (round half to even) as OpenCV has them
__device__ inline int update_num_iters(double p, double ep, int model_points, int max_iters) {
  p = fmin(fmax(p, 0.0), 1.0);
  ep = fmin(fmax(ep, 0.0), 1.0);
  double num = fmax(1.0 - p, DBL_MIN);
  double denom = 1.0 - pow(1.0 - ep, (double)model_points);
  if (denom < DBL_MIN) return 0;
  num = log(num);
  denom = log(denom);
  return denom >= 0.0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
}

__device__ __forceinline__ unsigned long long mwc_mulmod(unsigned long long x, unsigned long long y) {
  return (unsigned long long)(((unsigned __int128)x * y) % kMwcM);
}

// `count` consecutive samples from generator state s (updated), by one warp: every lane calls with the same arguments.
// The MWC step is state -> state * kMwcA mod kMwcM on residues, so lane l jumps K l steps ahead and draws the K indices a
// sample takes when it needs no redraw; the samples before the first lane that saw a repeat are OpenCV's, and that lane's
// sample is drawn serially (with its redraws) before the next 32.  fresh: s is the start state 2^64 - 1, which, like the
// state after it, lies above the modulus (its low word is not its residue's): the first sample is drawn serially.
// Sample h goes to dst[h * stride .. + K - 1] (and trace[(trace_first + h) * K ..] while below trace_cap).
template <int K>
__device__ void warp_draw(unsigned long long& s, bool fresh, unsigned n, int count, int* dst, int stride, int* trace, int trace_first,
                          int trace_cap) {
  const int lane = threadIdx.x & 31;
  const unsigned long long m = fast_mod_m(n);
  auto put = [&](int h, const int* idx) {
    for (int k = 0; k < K; ++k) dst[(size_t)h * stride + k] = idx[k];
    if (trace && trace_first + h < trace_cap)
      for (int k = 0; k < K; ++k) trace[(size_t)(trace_first + h) * K + k] = idx[k];
  };
  int h = 0;
  if (fresh && count > 0) {
    int idx[K];
    subset<K>(s, n, m, idx);
    if (lane == 0) put(0, idx);
    h = 1;
  }
  unsigned long long jump = 1, sq = kMwcA;             // kMwcA^(K lane) mod kMwcM
  for (int e = K * lane; e; e >>= 1) {
    if (e & 1) jump = mwc_mulmod(jump, sq);
    sq = mwc_mulmod(sq, sq);
  }
  while (h < count) {
    const unsigned long long start = mwc_mulmod(s, jump);
    unsigned long long t = start;
    int v[K];
    const bool distinct = draw<K>(t, m, n, v);
    const int avail = min(32, count - h);
    const unsigned bad = __ballot_sync(0xffffffffu, lane < avail && !distinct);
    const int k = bad ? __ffs(bad) - 1 : avail;
    if (lane < k) put(h + lane, v);
    if (k == avail) {
      s = __shfl_sync(0xffffffffu, t, k - 1);
      h += k;
    } else {
      unsigned long long u = __shfl_sync(0xffffffffu, start, k);
      int idx[K];
      subset<K>(u, n, m, idx);
      if (lane == 0) put(h + k, idx);
      s = u;
      h += k + 1;
    }
  }
}

}  // namespace cvrng
}  // namespace opb
