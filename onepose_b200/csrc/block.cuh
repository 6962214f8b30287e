// Block-wide integer primitives the library's kernels share: a reduction, an exclusive scan (forward or reverse) and a kept
// thread's slot in an ordered compaction.  Each passes a barrier before it writes sh, so a loop may call it again with the same sh.
#pragma once
#include <stdint.h>

namespace opb {
namespace {

template <typename T, typename Op>
__device__ T block_reduce(T v, Op op, T* sh) {                // every thread gets the result; sh holds 32 values
  for (int d = 16; d; d >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, d));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = sh[0];
  for (int w = 1; w < nw; ++w) v = op(v, sh[w]);
  return v;
}

// Exclusive scan of v over the block in thread order, or from the last thread when reverse; *total gets the whole.  Every
// thread calls it; blockDim.x is a multiple of 32 and sh holds 32 values.
template <typename T, typename Op>
__device__ T block_scan(T v, Op op, T identity, T* sh, T* total, bool reverse = false) {
  const int nw = blockDim.x >> 5;
  const int r = reverse ? blockDim.x - 1 - threadIdx.x : threadIdx.x;   // rank in scan order
  const int lane = r & 31, warp = r >> 5;
  T inc = v;
  for (int d = 1; d < 32; d <<= 1) {
    const T u = reverse ? __shfl_down_sync(0xffffffffu, inc, d) : __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc = op(inc, u);
  }
  T exc = reverse ? __shfl_down_sync(0xffffffffu, inc, 1) : __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) exc = identity;
  __syncthreads();
  if (lane == 31) sh[warp] = inc;
  __syncthreads();
  T carry = identity, all = identity;
  for (int w = 0; w < nw; ++w) {
    if (w < warp) carry = op(carry, sh[w]);
    all = op(all, sh[w]);
  }
  if (total) *total = all;
  return op(carry, exc);
}

// The number of threads before this one, in thread order, whose keep is true; *total gets the block's count on every thread.
// Every thread calls it; blockDim.x is a multiple of 32 and sh holds blockDim.x / 32 values.
__device__ __forceinline__ int block_rank(bool keep, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  __syncthreads();
  if (lane == 0) sh[warp] = __popc(m);
  __syncthreads();
  const int c = lane < (int)(blockDim.x >> 5) ? sh[lane] : 0;    // lane w holds warp w's count
  *total = __reduce_add_sync(0xffffffffu, c);
  return __reduce_add_sync(0xffffffffu, lane < warp ? c : 0) + __popc(m & ((1u << lane) - 1u));
}

struct Max { __device__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; } };
struct Min { __device__ int32_t operator()(int32_t a, int32_t b) const { return a < b ? a : b; } };
struct Sum32 { __device__ int32_t operator()(int32_t a, int32_t b) const { return a + b; } };
struct Sum64 { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };
struct SumS64 { __device__ long long operator()(long long a, long long b) const { return a + b; } };

}  // namespace
}  // namespace opb
