// Linear-attention state on the Hopper tensor cores (wgmma).
//
//   per segment s, head h:   KV[h][d][q] = sum_rows elu1(K[r,h,d]) * V[r,h,q],   Ksum[h][d] = sum_rows elu1(K[r,h,d])
//   (reference GATs_SuperGlue.py:71-78; the 1/m of :75 is applied by kv_state_reduce)
//
// The k,v projection epilogue (EPI_QKV) leaves  kvh[rows, 512] = fp16(64 * [elu1(K) | V])  with pad rows zero, so the state
// is ONE tensor-core pass over operands that TMA lands directly in the MN-major SWIZZLE_128B layout wgmma reads (reduction
// index = row).  Rounding K and V to fp16 perturbs each product by <= 2^-11 relative with zero mean; the state is a MEAN over the
// segment's rows, so the perturbation of the mean is ~2^-12/sqrt(rows) -- measured end to end in tools/kv_precision.py
// (cosine error unchanged at 7e-7 down to 16-row segments).
#include <cuda.h>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "host_util.cuh"
#include "kv_state_tc.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace opb {
namespace {

// One CTA per ROW GROUP = `slabs_per_group` consecutive 256-row slabs of one segment (groups never straddle a segment; the
// host picks the group size so that the grid is about two CTAs per SM -- fewer, larger groups mean fewer partial states to
// write and re-read).  256 threads:
//   warp 0       TMA producer: 32-row stages = 8 boxes of 64 channels x 32 rows (4 K blocks, 4 V blocks), 3-stage ring
//   warps 4-7    one warpgroup: per stage and head h, wgmma m64n64k16 with A = K_h^T and B = V_h read MN-major straight from
//                the TMA boxes (reduction index = row), 2 k-steps of 16 rows, the four head accumulators in registers over the
//                whole group; while the MMAs run it sums the K columns of the same stage (the K mean of the attention
//                normaliser), then writes the state.
constexpr int kHRows = 32;                                 // rows per stage
constexpr int kHStages = 3;
constexpr int kHBlockBytes = kHRows * 128;                 // one 64-channel x 32-row box = 4 KB
constexpr int kHStageBytes = 8 * kHBlockBytes;             // 32 KB
constexpr int kHSmemBytes = kHStages * kHStageBytes + 1024 + 128;
constexpr int kHThreads = 256;

// MN-major SWIZZLE_128B descriptor (sm_90): LBO = bytes between 64-element blocks along M / N (one block per head here),
// SBO = 1024 bytes between 8-row groups along the reduction
__device__ __forceinline__ uint64_t make_desc_mn_h(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(kHBlockBytes >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;                                  // SWIZZLE_128B
  return d;
}

__global__ void __launch_bounds__(kHThreads, 1) kv_state_h_kernel(const __grid_constant__ CUtensorMap kv_map, Layout L, KvGroups G, float* __restrict__ partial) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kHStages * kHStageBytes);   // [3] stage landed
  uint64_t* empty_bar = full_bar + kHStages;                                          // [3] stage consumed (MMAs retired + sums read)

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform for the compiler (wgmma issue path)
  // row group -> (frame, side, group index inside the segment)
  const int per_frame = G.gq + G.gd;
  const int b = blockIdx.x / per_frame, g = blockIdx.x - b * per_frame;
  const int side = g >= G.gq ? 1 : 0, gi = side ? g - G.gq : g;
  const int seg = 2 * b + side;
  const int group_rows = G.slabs * 256;
  const int row0 = L.seg_start(seg) + gi * group_rows;
  float* out = partial + (long long)blockIdx.x * kHeads * (kDh * kDh + kDh);
  griddep_sync();                                          // kvh of the preceding GEMM is visible from here on
  const int n_valid = min(group_rows, L.seg_valid(seg) - gi * group_rows);
  if (n_valid <= 0) {                                      // group entirely in the padding: never read by the reduction, defined anyway
    for (int i = tid; i < kHeads * (kDh * kDh + kDh); i += kHThreads) out[i] = 0.f;
    return;
  }
  const int n_stages = (n_valid + kHRows - 1) / kHRows;    // rows past n_valid inside the last stage are zero (EPI_QKV zeroes pad rows)
  if (tid == 0) {
    for (int s = 0; s < kHStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&kv_map) : "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      for (int s = 0; s < n_stages; ++s) {
        const int buf = s % kHStages;
        if (s >= kHStages) mbar_wait(&empty_bar[buf], ((s / kHStages) - 1) & 1);
        mbar_expect_tx(&full_bar[buf], kHStageBytes);
        uint8_t* st = smem + buf * kHStageBytes;
#pragma unroll
        for (int blk = 0; blk < 8; ++blk) tma_load_2d(st + blk * kHBlockBytes, &kv_map, &full_bar[buf], blk * 64, row0 + s * kHRows);
      }
    }
  } else if (warp >= 4) {
    float acc[kHeads][32];                                  // head h: KV_h [64 x 64] fragment (wgmma.cuh)
#pragma unroll
    for (int h = 0; h < kHeads; ++h)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
    // ---- K column sums: thread = (8-channel chunk j of the 256 K channels, row group g of 4)
    const int t = tid - 128;
    const int j = t & 31, g = t >> 5;
    float ks[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int prev = -1;
    for (int s = 0; s < n_stages; ++s) {
      const int buf = s % kHStages;
      mbar_wait(&full_bar[buf], (s / kHStages) & 1);
      const uint32_t kb = smem_u32(smem) + buf * kHStageBytes, vb = kb + 4 * kHBlockBytes;
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < kHeads; ++h)
#pragma unroll
        for (int k = 0; k < kHRows / 16; ++k)
          wgmma_m64n64k16_mn(acc[h], make_desc_mn_h(kb + h * kHBlockBytes + k * 2048), make_desc_mn_h(vb + h * kHBlockBytes + k * 2048));
      wgmma_commit();
      const uint32_t base = kb + (j >> 3) * kHBlockBytes;
#pragma unroll
      for (int i = 0; i < kHRows / 4; ++i) {
        const int r = g + 4 * i;
        uint4 v;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(base + r * 128 + (((j & 7) ^ (r & 7)) << 4)));
        const __half2* hp = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(hp[e]);
          ks[2 * e] += f.x;
          ks[2 * e + 1] += f.y;
        }
      }
      wgmma_wait<1>();                                      // the previous stage's MMAs have retired
      // The arrive releases the stage to the TMA producer and must not overtake the loads of its K sums: ptxas sinks the
      // FADDs that consume them below the arrive, so nothing in issue order guarantees they have returned.  Without the fence
      // the K sums could pick up rows of the NEXT use of the stage.
      __threadfence_block();
      __syncwarp();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = buf;
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < kHeads; ++h) fence_regs<32>(acc[h]);
    // ---- epilogue: KV_h[d][q] (d = K channel = fragment row, q = V channel = fragment column)
    const int wq = warp - 4;
#pragma unroll
    for (int h = 0; h < kHeads; ++h) {
      float* o = out + (long long)h * (kDh * kDh + kDh);
#pragma unroll
      for (int gg = 0; gg < 8; ++gg) {
        const int d = 16 * wq + (lane >> 2), qc = 8 * gg + 2 * (lane & 3);
        *reinterpret_cast<float2*>(o + d * kDh + qc) = make_float2(acc[h][4 * gg] * kProdInv, acc[h][4 * gg + 1] * kProdInv);
        *reinterpret_cast<float2*>(o + (d + 8) * kDh + qc) = make_float2(acc[h][4 * gg + 2] * kProdInv, acc[h][4 * gg + 3] * kProdInv);
      }
    }
    // K sums: combine the 4 row groups through the (now idle) stage memory
    float* red = reinterpret_cast<float*>(smem);
    asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
    for (int e = 0; e < 8; ++e) red[g * 256 + j * 8 + e] = ks[e];
    asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
    for (int c = t; c < 256; c += 128)
      out[(long long)(c >> 6) * (kDh * kDh + kDh) + kDh * kDh + (c & 63)] = (red[c] + red[256 + c] + red[512 + c] + red[768 + c]) * kPreInv;
  }
}

}  // namespace

}  // namespace opb

namespace opb {
KvGroups kv_groups_for(const Layout& L, int num_sms) {
  const int total_slabs = L.rows() / 256;
  int slabs = total_slabs / (2 * num_sms);                 // about two CTAs per SM (two waves of the one-CTA-per-SM kernel)
  slabs = slabs < 1 ? 1 : (slabs > 8 ? 8 : slabs);
  KvGroups G;
  G.slabs = slabs;
  G.gq = (L.n_pad / 256 + slabs - 1) / slabs;
  G.gd = (L.m_pad / 256 + slabs - 1) / slabs;
  return G;
}

cudaError_t launch_kv_state_h(const __half* kvh, const Layout& L, const KvGroups& G, float* partial, cudaStream_t stream) {
  if (const cudaError_t e = ensure_smem_limit((const void*)kv_state_h_kernel, kHSmemBytes)) return e;
  CUtensorMap map;
  if (!make_tensor_map_2d(&map, kvh, L.rows(), 512, 512, 64, kHRows, false)) return cudaErrorInvalidValue;
  return launch_k(pdl_enabled(), kv_state_h_kernel, dim3((unsigned)(L.B * (G.gq + G.gd))), dim3(kHThreads), kHSmemBytes, stream, map, L, G, partial);
}
}  // namespace opb
