// wgmma / TMA GEMM core (sm_90a) -- declarations.  See gemm_tc.cu.
#pragma once
#include <cuda.h>

#include "gemm_common.cuh"

namespace opb {
// C (+ fused epilogue, GemmProblem::epi) = A . B^T on the Hopper tensor cores with the 3-pass fp16-split
// scheme.  Returns 0, -1 (bad shape / unsupported combination) or -2 (CUDA error).
int launch_gemm_tc(const GemmProblem& p, cudaStream_t stream);
// 2-D row-major tensor map [rows, ld] (columns used: `cols`), box = box_cols x box_rows; swizzle follows the box row width
// (128 B -> SWIZZLE_128B, 64 B -> SWIZZLE_64B).  Cached per (pointer, shape, box, dtype).
bool make_tensor_map_2d(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows, bool f32);
// Raises the dynamic shared-memory limit of kernel `func` to `bytes` on the current device.  The attribute belongs to a device's
// context, so it is set once per (kernel, device) -- again only for a larger size; thread-safe.
cudaError_t ensure_smem_limit(const void* func, int bytes);
// Programmatic dependent launch switch shared by every launch site (default on; opb_debug_set_pdl).
bool pdl_enabled();
void set_pdl_enabled(bool on);
// 3x3 convolutions on narrow column tiles (EPI_CONV): 1 (default) = halo boxes -- one (BM + 2)-row A box per kernel row serves the three
// horizontal taps through row-offset wgmma descriptors; 0 = nine row-shifted boxes per tile (A/B switch: opb_debug_set_conv_halo).
void set_conv_halo_mode(int mode);
}  // namespace opb
