// Shared device/host helpers for the GATsSPG matcher kernels (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace opb {

constexpr int kD = 256;        // descriptor_dim
constexpr int kHeads = 4;
constexpr int kDh = 64;        // per-head dim
constexpr int kSegPad = 256;   // segments are padded to this: 2 row tiles / one 256-wide score tile
// fp16-split operand format: every plane pair carries a fixed 2^6 pre-scale,
//   hi = fp16(64 x),  lo = fp16(64 x - hi)      =>  x = (hi + lo) / 64  to ~2^-22 relative
// (the pre-scale keeps `lo` out of the fp16 subnormal range for |x| > ~2e-3; |x| < 1023 is
// representable).  A product of two such operands carries 2^12, removed in the GEMM epilogue.
constexpr float kPre = 64.0f;
constexpr float kPreInv = 1.0f / 64.0f;
constexpr float kProdInv = 1.0f / 4096.0f;
// Smallest pre-scaled value whose hi plane rounds to fp16 inf (65504 + half an ulp): a split of 64 x at or above it stores
// hi = inf, lo = -inf, and the next product turns into NaN.
constexpr float kSplitLimit = 65520.0f;
// Range guard of the extractor's producers of split planes: `peak` is the largest pre-scaled |value| a thread split.  A
// running fmaxf ignores NaN, so NaN is excluded where it could enter instead: the weights are checked on the host
// (opb_sp_finalize_weights) and the image in sp_conv1a; from finite in-range operands a convolution can only produce finite
// values, which the peak sees.
__host__ __device__ __forceinline__ bool split_out_of_range(float peak) { return !(peak < kSplitLimit); }

// Activation layout of one forward chunk: frame b owns rows
//   [b*R, b*R + n_pad)           query segment   (N valid)
//   [b*R + n_pad, (b+1)*R)       3D-point segment (M_b valid: the rows of frame b's object)
// with R = n_pad + m_pad, both multiples of kSegPad.  A "segment" is the unit of
// InstanceNorm statistics and of the linear-attention KV state
// (reference GATs_SuperGlue.py:126 and :77-78 reduce over the point dimension).
// Frames of one chunk may use different objects: M is the largest M_b of the chunk, rows [M_b, m_pad) of a 3D segment are
// zero and masked out of every reduction, as the query rows past n_of(b).
struct Layout {
  int B, N, M, n_pad, m_pad, R;
  const int* nlen;   // device int32 [B]: valid query rows of each frame (ragged batch, every entry in [0, N]) or nullptr: N everywhere
  const int* mlen;   // device int32 [B]: valid 3D rows of each frame (frames of different objects, entries in [1, M]) or nullptr: M everywhere
  __host__ __device__ int rows() const { return B * R; }
  __host__ __device__ int segs() const { return 2 * B; }
  __host__ __device__ int seg_of_row(int row) const {
    int b = row / R;
    return 2 * b + ((row - b * R) >= n_pad ? 1 : 0);
  }
  __host__ __device__ int seg_start(int seg) const { return (seg >> 1) * R + ((seg & 1) ? n_pad : 0); }
  __host__ __device__ int seg_padded(int seg) const { return (seg & 1) ? m_pad : n_pad; }
#ifdef __CUDACC__
  // valid query rows of frame b / valid rows of a segment (device only: nlen lives in device memory)
  __device__ int n_of(int b) const { return nlen ? min(max(__ldg(nlen + b), 0), N) : N; }
  __device__ int m_of(int b) const { return mlen ? __ldg(mlen + b) : M; }
  __device__ int seg_valid(int seg) const { return (seg & 1) ? m_of(seg >> 1) : n_of(seg >> 1); }
#endif
  // attention source segment: 'self' -> itself, 'cross' -> the other side of the frame
  // (reference GATs_SuperGlue.py:57-58, :62-63)
  __host__ __device__ int src_seg(int seg, int cross) const { return cross ? (seg ^ 1) : seg; }
};

__host__ __device__ inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

#ifdef __CUDACC__
// exp / elu+1 on the bare hardware exponential: ex2.approx.ftz (max rel. error ~2^-22, the order of the fp16 split every
// consumer applies next).  __expf wraps the same instruction in denormal-range handling that costs ~10 predicated
// instructions per element -- measured 4x on the element-wise epilogues.
__device__ __forceinline__ float ex2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// Programmatic dependent launch (every kernel of the path is launched with programmatic stream serialization): wait until the
// previous launch of the stream has completed and its writes are visible, then allow the next launch to begin its own set-up.
// Nothing before this call may touch global memory.
__device__ __forceinline__ void griddep_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ float exp_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}
__device__ __forceinline__ float elu1_fast(float x) {
  const float e = exp_fast(x);
  return x > 0.f ? x + 1.f : e;
}
#endif

__host__ __device__ __forceinline__ void split_f32(float x, __half& hi, __half& lo) {
  const float xs = x * kPre;
  hi = __float2half_rn(xs);
  lo = __float2half_rn(xs - __half2float(hi));
}
// split_f32 of two elements at once, two per conversion instruction; `scaled` is already x kPre
__device__ __forceinline__ void split_f32x2(float2 scaled, __half2& hi, __half2& lo) {
  hi = __float22half2_rn(scaled);
  const float2 back = __half22float2(hi);
  lo = __float22half2_rn(make_float2(scaled.x - back.x, scaled.y - back.y));
}
__host__ __device__ __forceinline__ float join_f32(__half hi, __half lo) {
  return (__half2float(hi) + __half2float(lo)) * kPreInv;
}

struct Planes {      // one fp16-split tensor [rows, ld]
  __half* hi;
  __half* lo;
  int ld;
};
struct CPlanes {
  const __half* hi;
  const __half* lo;
  int ld;
};

}  // namespace opb
