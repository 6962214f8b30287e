// wgmma / TMA GEMM core for sm_90a -- persistent, warp-specialised, register accumulators.
//
//   C[128 x BN tile] = sum_k A_tile . B_tile^T     A, B: fp16-split planes (hi, lo; common.cuh), K-major
//
// Each logical product runs as THREE tensor-core passes into ONE fp32 accumulator
//     D += A_hi.B_hi + A_hi.B_lo + A_lo.B_hi            (x 2^-12 in the epilogue)
// which reproduces fp32 products to ~2^-22 relative (tools/precision_ladder.py); the reference
// computes in fp32 (GATs_SuperGlue.py:191-193) and the contract is 1e-4 abs on conf.
//
// Persistent grid (at most one CTA per SM), static round-robin tile schedule (n-tile fastest so CTAs that share an A row tile
// run together).  Two consumer schedules:
//   ping-pong (PP: EPI_F32 / EPI_F32_STATS / EPI_SCORE_SUMS)  128 x 128 tiles; warpgroup w owns the
//                CTA's units w, w + 2, ... whole (two m64n128 accumulators: rows [0, 64) and [64, 128), 128 registers per
//                thread).  An order barrier (two mbarriers) hands the tensor pipe to the other warpgroup once a warpgroup has
//                issued its tile's last MMAs, so one warpgroup's epilogue runs under the other's main loop.  The epilogue
//                walks the tile in 32-column chunks through the warpgroup's own 16 KB staging box: fragment -> box ->
//                thread = row -> fused op -> staged in place -> TMA store.  Ring: 3 stages of 64 KB.
//   cooperative  every other variant.  EPI_L2NORM needs a row's 256 columns; the epilogues of EPI_QKV, EPI_QSCALE and
//                EPI_SCORE_CONF need more registers than a live 128-register accumulator leaves (they spill as PP).  The
//                converter (mlp.3), EPI_BIAS_PLANES and the extractor's narrow EPI_CONV / EPI_F32 tiles were not measured as PP.
// 384 threads = 12 warps:
//   warps 0-7    two consumer warpgroups.  Cooperative: warpgroup w issues wgmma.m64nBNk16 for rows [64 w, 64 w + 64) of the tile and keeps
//                that accumulator in registers (BN = 256: 128 registers per thread).  At the end of a tile both warpgroups
//                park their accumulators in shared memory and the same 8 warps run the fused epilogue as two groups of 4
//                warps: thread = tile row, group g = half g of the tile's columns, smem -> registers -> fused op -> swizzled
//                smem staging -> TMA store.  Every epilogue that writes fp16-split planes goes through one store path
//                (store_planes32: 32 columns, two SWIZZLE_64B buffers).  BN 256 parks in the last k-block's ring stage and
//                the staging buffers and stages every chunk in place (kStagePark), so the next tile's first k-block loads
//                into the other stage during the epilogue; narrow tiles park over the ring and load the next tile after it.
//   warp 8       TMA producer   cp.async.bulk.tensor 2D, SWIZZLE_128B boxes -> a 192 KB shared-memory ring of 2-4 stages
//   warps 9-11   converters (ACV_NORM_RELU only; in every other variant they go straight to the final __syncthreads)
// (The registers of a block are allocated in whole warpgroups, so the third warpgroup costs no registers: 168 per thread.)
// Converter variant (ACV_NORM_RELU): the producer lands the RAW fp32 A tile, the converter warps rewrite all 128 rows into the
// (hi, lo) planes in place and arrive on the stage's conv_bar; the consumers wait on conv_bar instead of full_bar, so their
// k-blocks are the same branch-free MMA chain as every other variant's and the conversion of stage s + 1 runs under the MMAs
// of stage s.
// Every kernel starts with griddepcontrol.wait after its on-chip set-up (programmatic dependent launch: the set-up of launch
// i+1 overlaps the tail of launch i).
#include <cuda.h>

#include <cstdlib>

#include <map>
#include <mutex>
#include <tuple>

#include "gemm_tc.cuh"
#include "host_util.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace opb {
namespace {

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int MMA_K = 16;
constexpr int kABytes = BM * BK * 2;             // one plane of the A tile (16 KB)
constexpr int kRingBytes = 192 * 1024;           // load ring; also holds the parked fp32 accumulator tile between main loops
constexpr int kStagingBytes = 16384;             // one 128-row x 128-B swizzled epilogue buffer
constexpr int kNumStaging = 2;
constexpr int kParkBoxBytes = 128 * 128;         // BN 256: one 128-row x 32-column fp32 box of the parked accumulator
constexpr int kExtraBytes = 1024;                // per-tile scratch of the score epilogue (inverse column sums of the tile)
constexpr int kMaxStages = 4;
constexpr int kSmemBytes = kRingBytes + kNumStaging * kStagingBytes + 1024 /*align*/ + 256 /*barriers*/ + kExtraBytes;
static_assert(kSmemBytes <= 227 * 1024, "exceeds the 227 KB of shared memory an H100 block can have");
constexpr int kThreads = 384;                    // warpgroups 0, 1: MMA + epilogue; warp 8: TMA producer; warps 9-11: converters
constexpr int kProducerWarp = 8;
constexpr int kConvWarps = 3;

// ------------------------------------------------------------------ PTX wrappers (mbarrier / TMA loads: tma.cuh)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c_inner, int c_outer) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(smem_u32(smem_src)),
               "r"(c_inner), "r"(c_outer)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(smem_u32(smem_src)),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void epi_bar_id(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }   // the 4 warps of one warpgroup
__device__ __forceinline__ void consumers_bar() { asm volatile("bar.sync 3, 256;" ::: "memory"); }                // both consumer warpgroups

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90):
//   start address >> 4 | LBO (unused for swizzled K-major; 1) | SBO = 1024 bytes between 8-row groups | swizzle mode 1 = 128B
// A k-step of 16 elements inside the 128-byte swizzle row moves the start address by 32 bytes, a row offset by 128 bytes per
// row: the swizzle XOR is a function of the absolute shared-memory address bits, so both TMA and the tensor core see the same
// layout from any such start (the 3x3 halo convolution reads one (BM + 2)-row box at row offsets 0 / 1 / 2).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
  return d;
}
// One k-step of a consumer warpgroup: its 64 rows x N columns += A (64 x 16) . B (N x 16)^T
template <int N>
__device__ __forceinline__ void mma_k16(float* d, uint64_t a, uint64_t b) {
  if (N == 256) wgmma_m64n256k16(d, a, b);
  else if (N == 128) wgmma_m64n128k16(d, a, b);
  else wgmma_m64n64k16(d, a, b);
}

// byte offset of 16-byte chunk j of row r inside a 128-row x 128-B SWIZZLE_128B staging buffer
__device__ __forceinline__ uint32_t stg_off(int r, int j) { return (uint32_t)(r * 128 + ((j ^ (r & 7)) << 4)); }
// same for a 128-row x 64-B SWIZZLE_64B buffer (16-byte chunk j in 0..3): Swizzle<2,4,3> = address bits [4,6) ^= bits [7,9)
__device__ __forceinline__ uint32_t stg64_off(int r, int j) { return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4)); }

struct TcParams {
  int K1, K2;            // reduction split (multiples of BK)
  int b2_per_seg;
  int n_out;
  int m_tiles, n_tiles, batch;
  long long a_batch_rows, b_batch_rows;
  int c_batch_rows;      // output rows per batch (C is [batch*rows, ldc])
  int seg_rows;          // rows are rows of the activation layout L (segment-aware masking); 0: plain matrix
  Layout L;
  const float* bias;
  // fused epilogues
  const float* kmean;    // EPI_QSCALE
  int cross;
  float* statpart;       // EPI_F32_STATS
  // A-operand converters (ACV)
  const float* mu;       // ACV_NORM_RELU: [S][512]
  const float* rstd;
  // EPI_SCORE_*
  float inv_scale;
  float* rowsum_part;
  float* colsum_part;
  const float* inv_rowsum;
  const float* inv_colsum;
  float* conf;
  int conf_tma;          // 1: conf goes out through the 3-D tensor map (conf_ld % 4 == 0), 0: plain stores from the staged chunk
  int conf_ld;           // columns of a conf row (GemmProblem::conf_ld)
  unsigned long long* rowbest;
  unsigned long long* colbest;
  // implicit-GEMM convolution (GemmProblem::taps) and the EPI_CONV geometry
  int taps, kb_per_tap;
  int tap_off[9];
  int cv_w2, cv_h, cv_w, cv_ppad, relu;
  int* range_flag;       // GemmProblem::range_flag
  int halo;              // 3x3 convolution with one (BM + 2)-row A box per (kernel row, 64-channel block)
};

struct Maps {
  CUtensorMap a1h, a1l, a2h, a2l, b1h, b1l, b2h, b2l;   // loads
  CUtensorMap out_f32;                                    // store: fp32 [rows, ldc], box 32 x 128 (SWIZZLE_128B)
  CUtensorMap out_hi, out_lo;                             // store: fp16-split planes, box 32 x 128 (SWIZZLE_64B)
  CUtensorMap a_raw;                                      // load: fp32 source of a converted A operand, box 32 x 128 (SWIZZLE_128B)
                                                          // (halo convolution: a1h / a1l have boxes of BM + 2 rows)
};

// A-operand conversion: instead of fp16-split planes prepared by a separate kernel, the TMA producer lands the RAW fp32
// tile (128 rows x 64 columns = exactly the 32 KB of the stage's A_hi + A_lo planes) and the converter warps rewrite it
// IN PLACE as the (hi, lo) planes the MMA descriptors expect -- the pointwise op between two GEMMs runs on data that is
// already on the SM, and its 4 KB/row HBM round trip disappears:
//   ACV_NORM_RELU  A  = ReLU((hid - mu_seg) * rstd_seg)          mlp.3 reads mlp.0's fp32 output (GATs_SuperGlue.py:126-127)
enum { ACV_NONE = 0, ACV_NORM_RELU = 1 };

// HI: the A operand enters with its hi plane only (k,v projection, GemmProblem::a_hi_only): two passes, A_hi + B_hi + B_lo per stage.
// BN_: column-tile width (256 for every matcher GEMM; 64 / 128 for the narrow convolution layers of the extractor: the stage
// shrinks and the ring deepens to three / four stages).
// ACV and the K2 block: the converter exists for mlp.3 only, whose K2 block is its residual as an identity K-block
// (GemmProblem::b2_lo_zero; launch_gemm_tc requires it with the converter and refuses it without).  The identity's lo plane is
// zero, so with ACV the K2 k-blocks run a chain of their own without the A_hi.B_lo pass (it would add exact zeros).  The
// template, not a branch inside the chain, selects it: a branch between two wgmmas makes ptxas insert a warpgroup.arrive in
// front of the MMAs that follow it.  The identity runs at full width: N = 64 MMAs on its diagonal blocks are slower on an
// H100 (DESIGN.md 5.1).

// PP: the ping-pong schedule (BN_ 128; see the top of the file).
template <int EPI, int ACV = ACV_NONE, bool HI = false, int BN_ = 256, bool PP = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ Maps maps, TcParams p) {
  constexpr int BN = BN_;
  static_assert(!PP || (BN_ == 128 && ACV == ACV_NONE && !HI && (EPI == EPI_F32 || EPI == EPI_F32_STATS || EPI == EPI_SCORE_SUMS)),
                "ping-pong: 128-column tiles of the variants that move");
  constexpr int kBBytes = BN * BK * 2;             // one plane of the B tile
  constexpr int kBOff = HI ? kABytes : 2 * kABytes;      // offset of the B planes inside a stage
  constexpr int kStageBytes = kBOff + 2 * kBBytes;
  constexpr int kStages = kRingBytes / kStageBytes;      // BN 256: 2, BN 128: 3, BN 64: 4
  static_assert(ACV == ACV_NONE || (BN_ == 256 && EPI == EPI_BIAS_PLANES), "the converter: mlp.3 only");
  static_assert(EPI != EPI_SCORE_SUMS || PP, "score sums: one row sum per 128-column ping-pong tile");
  static_assert(PP || (EPI == EPI_CONV ? BN_ == 64 || BN_ == 128 : EPI == EPI_F32 ? BN_ == 128 || BN_ == 256 : BN_ == 256),
                "tile widths: EPI_CONV 64 / 128, EPI_F32 128 / 256, every other cooperative epilogue 256");
  static_assert(BN_ == 256 || ACV == ACV_NONE && !HI, "narrow tiles: no converter, both A planes");
  static_assert(!HI || ACV == ACV_NONE, "converters need the full stage");
  static_assert(kStages >= 2 && kStages <= kMaxStages, "ring depth");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // halo convolution (EPI_CONV, TcParams::halo; 64-column tiles -- a 128-column halo stage would leave room for one stage only):
  // a stage = one (kernel row, 64-channel block) group = A_hi / A_lo boxes of BM + 2 rows (the three horizontal taps read it at
  // row offsets 0 / 1 / 2) + the B tiles of the three taps
  constexpr int kHaloRows = BM + 2;
  constexpr int kHaloABytes = (kHaloRows * 128 + 1023) / 1024 * 1024;         // 17408
  constexpr int kHaloStageBytes = 2 * kHaloABytes + 6 * kBBytes;
  constexpr int kHaloStages = (EPI == EPI_CONV && BN_ == 64) ? kRingBytes / kHaloStageBytes : 0;
  static_assert(kHaloStages == 0 || (kHaloStages >= 2 && kHaloStages <= kMaxStages), "halo ring depth");
  const bool halo = kHaloStages > 0 && p.halo != 0;
  // Split accumulators (narrow tiles only).  The two correction passes (A_hi.B_lo, A_lo.B_hi: 2^-11 of the main term) get an
  // accumulator of their own, and with 64-wide tiles the main term is further split by kernel row; the partial sums are added
  // with round-to-nearest when the tile is parked -- fewer accumulate steps at full magnitude per fp32 accumulator.
  constexpr bool kSplitAcc = BN_ != 256 && !PP;
  constexpr int kMainAcc = BN_ == 64 ? 3 : 1;                    // accumulators of the A_hi.B_hi term (3: one per kernel row of a 3x3 convolution)
  const int n_main = (kMainAcc > 1 && EPI == EPI_CONV && p.taps == 9) ? kMainAcc : 1;
  constexpr int kHaloStagesDiv = kHaloStages ? kHaloStages : 1;  // (modulus of the halo ring; never used when there is none)
  constexpr int kAccLd = BN + 4;                                 // row stride (floats) of the parked accumulator: conflict-free row reads
  static_assert(BM * kAccLd * 4 <= kRingBytes, "parked accumulator exceeds the ring");
  // BN 256: the accumulator is parked as eight 128-row x 32-column fp32 SWIZZLE_128B boxes (box b = tile columns [32 b, +32)),
  // the first kStageBoxes in the ring stage of the tile's last k-block, the rest behind the ring (the staging buffers).  The
  // other stage stays free, so the next tile's first k-block loads under this tile's epilogue.  The epilogue stages each
  // chunk's stores in place, in the box it was read from.
  constexpr bool kStagePark = BN_ == 256;
  constexpr int kStageBoxes = kStageBytes / kParkBoxBytes;
  static_assert(!kStagePark || (kStageBytes % kParkBoxBytes == 0 &&
                                (8 - kStageBoxes) * kParkBoxBytes <= kRingBytes + kNumStaging * kStagingBytes - kStages * kStageBytes),
                "the parked tile fits one stage and the bytes behind the ring");
  uint8_t* staging = smem + kRingBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + kNumStaging * kStagingBytes);
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* acc_free_bar = empty_bar + kMaxStages;   // the parked accumulator has been read: the ring may be refilled
  uint64_t* conv_bar = acc_free_bar + 1;             // ACV: the stage's A tile has been converted (every k-block of the stage arrives)
  uint64_t* order_bar = conv_bar + kMaxStages;       // PP: order_bar[w] = the other warpgroup has issued its tile's last MMAs
  float* extra = reinterpret_cast<float*>(staging + kNumStaging * kStagingBytes + 256);   // kExtraBytes of per-tile scratch
  float* acc_smem = reinterpret_cast<float*>(smem);  // parked accumulator [BM][kAccLd]

  constexpr int kColsPerGroup = PP ? BN : BN / 2;    // columns of a tile that one epilogue group (warpgroup) writes
  // warp index through a shuffle: provably warp-uniform, so the wgmma issue paths below are not treated as divergent
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int nkb1 = p.K1 / BK, nkb = (p.K1 + p.K2) / BK;
  const int units_per_batch = p.m_tiles * p.n_tiles;
  const int total_units = units_per_batch * p.batch;

  if (threadIdx.x == 0) {
    // full: the TMA transaction arrive; empty: one arrive per consumer warp that reads the stage; conv: one arrive per
    // converter warp; order: one arrive per warp of the other warpgroup
    for (int s = 0; s < kMaxStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], PP ? 4 : 8); mbar_init(&conv_bar[s], kConvWarps); }
    mbar_init(acc_free_bar, 1);
    mbar_init(&order_bar[0], 4);
    mbar_init(&order_bar[1], 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&maps.a1h); prefetch_tmap(&maps.a1l); prefetch_tmap(&maps.b1h); prefetch_tmap(&maps.b1l);
    if (p.K2) { prefetch_tmap(&maps.a2h); prefetch_tmap(&maps.a2l); prefetch_tmap(&maps.b2h); prefetch_tmap(&maps.b2l); }
    if (ACV) prefetch_tmap(&maps.a_raw);
    if (EPI == EPI_F32 || EPI == EPI_F32_STATS || EPI == EPI_SCORE_CONF) prefetch_tmap(&maps.out_f32);
    if (EPI == EPI_QKV || EPI == EPI_QSCALE || EPI == EPI_L2NORM || EPI == EPI_BIAS_PLANES || EPI == EPI_CONV) { prefetch_tmap(&maps.out_hi); prefetch_tmap(&maps.out_lo); }
  }
  __syncthreads();
  griddep_sync();                      // results of the previous launch are visible from here on; let the next launch set up

  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t it = 0, tc = 0;   // k-block counter across all tiles of this CTA, tile counter
      for (int u = blockIdx.x; u < total_units; u += gridDim.x, ++tc) {
        if (!kStagePark && !PP && tc) mbar_wait(acc_free_bar, (tc - 1) & 1);   // the previous tile's parked accumulator has been read
        const int z = u / units_per_batch, rem = u - z * units_per_batch;
        const int m_tile = rem / p.n_tiles, n_tile = rem % p.n_tiles;
        const int row0 = m_tile * BM;
        const int a_row = (int)(z * p.a_batch_rows) + row0;
        const int b_row1 = (int)(z * p.b_batch_rows) + n_tile * BN;
        const int seg = p.b2_per_seg ? p.L.seg_of_row(row0) : 0;     // a row tile lies inside one segment (segments are 256-row aligned)
        const int b_row2 = (p.b2_per_seg ? seg * p.n_out : 0) + n_tile * BN;
        if (halo) {
          const int ngroups = 3 * p.kb_per_tap;
          for (int g = 0; g < ngroups; ++g, ++it) {
            const int s = it % kHaloStagesDiv;
            mbar_wait(&empty_bar[s], ((it / kHaloStagesDiv) & 1) ^ 1);
            uint8_t* st = smem + s * kHaloStageBytes;
            mbar_expect_tx(&full_bar[s], 2 * kHaloRows * 128 + 6 * kBBytes);
            const int dy = g / p.kb_per_tap, cb = g - dy * p.kb_per_tap;
            const int arow = a_row + (dy - 1) * p.cv_w2 - 1;          // first row of the box: tap (dy, dx = 0); may be < 0 (zero fill)
            tma_load_2d(st, &maps.a1h, &full_bar[s], cb * BK, arow);
            tma_load_2d(st + kHaloABytes, &maps.a1l, &full_bar[s], cb * BK, arow);
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
              const int kcb = ((dy * 3 + dx) * p.kb_per_tap + cb) * BK;
              tma_load_2d(st + 2 * kHaloABytes + dx * 2 * kBBytes, &maps.b1h, &full_bar[s], kcb, b_row1);
              tma_load_2d(st + 2 * kHaloABytes + dx * 2 * kBBytes + kBBytes, &maps.b1l, &full_bar[s], kcb, b_row1);
            }
          }
          continue;
        }
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % kStages;
          // kStagePark: k-block 0 goes to the stage the previous tile did not park in; k-block 1 refills the parked stage once
          // the parked tile has been read.  (One k-block per tile: wait before k-block 0, so that the tile's epilogue cannot
          // complete a second acc_free phase before this wait.)
          if (kStagePark && tc && kb == (nkb > 1 ? 1 : 0)) mbar_wait(acc_free_bar, (tc - 1) & 1);
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          uint8_t* st = smem + s * kStageBytes;
          const bool first = kb < nkb1;
          const bool conv = ACV == ACV_NORM_RELU && first;           // this k-block's A tile comes in raw
          mbar_expect_tx(&full_bar[s], kStageBytes);
          int kc = (first ? kb * BK : (kb - nkb1) * BK);
          int arow = a_row, kcb = kc;                                   // A rows / B columns of this k-block
          if (EPI == EPI_CONV && p.taps) {                              // implicit-GEMM convolution: tap t = row-shifted A, B columns follow kb
            const int t = kb / p.kb_per_tap;
            kcb = kb * BK;
            kc = (kb - t * p.kb_per_tap) * BK;
            arow = a_row + p.tap_off[t];                                // may leave [0, rows): the tensor map zero-fills
          }
          const CUtensorMap* mah = first ? &maps.a1h : &maps.a2h;
          const CUtensorMap* mal = first ? &maps.a1l : &maps.a2l;
          const CUtensorMap* mbh = first ? &maps.b1h : &maps.b2h;
          const CUtensorMap* mbl = first ? &maps.b1l : &maps.b2l;
          const int brow = first ? b_row1 : b_row2;
          if (conv) {
            // raw fp32 [128 x 64] = two 32-column boxes, landing where the hi / lo planes will be written
            tma_load_2d(st, &maps.a_raw, &full_bar[s], kc, a_row);
            tma_load_2d(st + kABytes, &maps.a_raw, &full_bar[s], kc + 32, a_row);
          } else {
            tma_load_2d(st, mah, &full_bar[s], kc, arow);
            if (!HI) tma_load_2d(st + kABytes, mal, &full_bar[s], kc, arow);
          }
          tma_load_2d(st + kBOff, mbh, &full_bar[s], kcb, brow);
          tma_load_2d(st + kBOff + kBBytes, mbl, &full_bar[s], kcb, brow);
        }
      }
    }
  } else if (warp > kProducerWarp) {
    // ===================== converters: raw fp32 tile -> (hi, lo) planes, in place =====================
    // Converter warp cw rewrites the 16-row groups cw, cw + 3, cw + 6 of every hidden k-block.  Row r of the raw boxes and row r
    // of the planes are the same two 128-byte slots, so a lane group reads a row before any lane writes it (__syncwarp between).
    // Lane = (row 4i + lane/8, 8-column group c = lane%8): every shared-memory instruction touches each bank group once per
    // wavefront.  Every k-block arrives on conv_bar (the identity k-blocks need no conversion), so conv_bar runs through the
    // same phases as full_bar.
    if (ACV != ACV_NONE) {
      constexpr int kLPR = BK / 8;               // lanes per row = 8-column groups per k-block
      constexpr int kRPI = 32 / kLPR;            // rows per shared-memory instruction
      constexpr int kRowIters = 16 / kRPI;
      const int cw = warp - kProducerWarp - 1;
      const int c = lane % kLPR, rsub = lane / kLPR;
      uint32_t it = 0;
      for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
        const int m_tile = (u % units_per_batch) / p.n_tiles;
        const int seg_a = p.L.seg_of_row(m_tile * BM);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % kStages;
          if (kb < nkb1) {
            const int kcol = kb * BK + 8 * c;      // first of this lane's 8 source columns
            float pa[8], pb[8];                    // per-column parameters: (-64 mu rstd, 64 rstd)
            {
              const float* base_a = p.mu + (long long)seg_a * 512 + kcol;
              const float4 a0 = __ldg(reinterpret_cast<const float4*>(base_a)), a1 = __ldg(reinterpret_cast<const float4*>(base_a) + 1);
              pa[0] = a0.x; pa[1] = a0.y; pa[2] = a0.z; pa[3] = a0.w; pa[4] = a1.x; pa[5] = a1.y; pa[6] = a1.z; pa[7] = a1.w;
              const float* base_b = p.rstd + (long long)seg_a * 512 + kcol;
              const float4 b0 = __ldg(reinterpret_cast<const float4*>(base_b)), b1 = __ldg(reinterpret_cast<const float4*>(base_b) + 1);
              pb[0] = b0.x; pb[1] = b0.y; pb[2] = b0.z; pb[3] = b0.w; pb[4] = b1.x; pb[5] = b1.y; pb[6] = b1.z; pb[7] = b1.w;
              // 64 * ReLU((h - mu) * rstd) = max(h * (64 rstd) - 64 mu rstd, 0): one FFMA + one FMNMX per element, pre-scale included
#pragma unroll
              for (int j = 0; j < 8; ++j) { pb[j] *= kPre; pa[j] = -pa[j] * pb[j]; }
            }
            mbar_wait(&full_bar[s], (it / kStages) & 1);
            const uint32_t stu = smem_u32(smem + s * kStageBytes);
            const uint32_t rawbox = stu + ((2 * c) >> 3) * (BM * 128);
            for (int g = cw; g < BM / 16; g += kConvWarps) {
#pragma unroll
              for (int i = 0; i < kRowIters; ++i) {
                const int r = g * 16 + kRPI * i + rsub;
                const float4 ra = lds128(rawbox + r * 128 + ((((2 * c) & 7) ^ (r & 7)) << 4));
                const float4 rb = lds128(rawbox + r * 128 + ((((2 * c + 1) & 7) ^ (r & 7)) << 4));
                __syncwarp();                      // every lane holds its raw values of these rows before any lane overwrites them
                float v[8] = {ra.x, ra.y, ra.z, ra.w, rb.x, rb.y, rb.z, rb.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], pb[j], pa[j]), 0.f);     // already x 2^6
                uint4 oh, ol;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                  split_f32x2(make_float2(v[2 * j], v[2 * j + 1]), reinterpret_cast<__half2*>(&oh)[j], reinterpret_cast<__half2*>(&ol)[j]);
                sts128(stu + stg_off(r, c), oh);
                sts128(stu + kABytes + stg_off(r, c), ol);
              }
            }
            fence_async_smem();                    // generic-proxy writes -> visible to the tensor core (async proxy)
          } else {
            mbar_wait(&full_bar[s], (it / kStages) & 1);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&conv_bar[s]);
        }
      }
    }
  } else {
    // ===================== consumers: MMA main loop, then the epilogue =====================
    // cooperative: warpgroup wg = rows [64 wg, +64) of the MMA, columns half wg of the epilogue; PP: every row and column of
    // its own tiles
    const int wg = warp >> 2;
    const int q = warp & 3;                   // warp within the warpgroup
    const uint32_t a_off = PP ? 0u : (uint32_t)wg * 64 * 128; // this warpgroup's rows inside an A box (8-row groups of 1024 B)
    constexpr uint32_t kHalfOff = 64 * 128;         // PP: rows [64, 128) of an A box
    constexpr int kRegs = PP ? BN : BN / 2;         // accumulator registers per thread (PP: two m64n128 accumulators)
    float acc[kRegs];                               // main term (BN 64, 3x3 convolution: kernel row 0)
    float acc_c[kSplitAcc ? kRegs : 1];             // split accumulators: correction passes
    float acc_m1[kMainAcc > 1 ? kRegs : 1], acc_m2[kMainAcc > 1 ? kRegs : 1];   // BN 64: kernel rows 1, 2
    auto mma_main = [&](int am, uint64_t a, uint64_t b) {
      if (kMainAcc == 1 || am == 0) mma_k16<BN>(acc, a, b);
      else if (am == 1) mma_k16<BN>(acc_m1, a, b);
      else mma_k16<BN>(acc_m2, a, b);
    };
    auto release = [&](int s) {                     // this warp's MMAs reading stage s have completed
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    };
    const int grp = wg;                             // epilogue group: columns [grp*kColsPerGroup, +kColsPerGroup) of every tile
    const int r_in_tile = q * 32 + lane;
    const int t_in_grp = threadIdx.x - grp * 128;
    const bool leader = t_in_grp == 0;
    const int c_begin = PP ? 0 : grp * kColsPerGroup, c_end = c_begin + kColsPerGroup;
    auto epi_bar = [grp]() { epi_bar_id(1 + grp); };
    // one staging buffer per group (the other group's chain overlaps); before the group rewrites it, the store that last
    // read it must be done with it.  Staging rows are written with st.shared on 32-bit addresses (sts128): through generic
    // pointers, ptxas keeps the tile-invariant 64-bit row addresses live across the main loop and spills them there.
    auto stage_wait = [leader]() {                  // (kStagePark: no buffer is reused within a tile)
      if (!kStagePark && leader) tma_store_wait_read<0>();
    };
    // kStagePark: box b of the parked tile (the first kStageBoxes in the parked stage, the rest behind the ring).  PP: every
    // chunk goes through the warpgroup's own staging box (PP epilogues write no planes: store_planes32 never sees it).
    uint8_t* park_stage = smem;
    auto park_box = [&](int b) {
      if (PP) return staging + grp * kStagingBytes;
      return b < kStageBoxes ? park_stage + b * kParkBoxBytes : smem + kStages * kStageBytes + (b - kStageBoxes) * kParkBoxBytes;
    };
    // staging buffer of the chunk at tile column ct: the group's buffer, or (kStagePark, PP) the chunk's own box
    auto chunk_buf = [&](int ct) { return kStagePark || PP ? park_box(ct >> 5) : staging + grp * kStagingBytes; };
    // fp16-split planes out, one 32-column chunk at (col, row), tile column ct: pair(j) returns the pre-scaled (x 2^6) values
    // of the chunk's columns 2 j, 2 j + 1 for this thread's row; it runs after the staging buffers are free, in column order
    auto store_planes32 = [&](int ct, int col, int row, auto&& pair) {
      // this group's 8 KB halves of the two staging buffers, or the two halves of the chunk's box
      uint8_t* sh = kStagePark ? park_box(ct >> 5) : staging + grp * 8192;
      uint8_t* sl = kStagePark ? sh + 8192 : staging + kStagingBytes + grp * 8192;
      stage_wait();                                 // the store that last read these buffers is done with them
      epi_bar();                                    // (kStagePark: the group's threads have read every row of the box)
#pragma unroll
      for (int j8 = 0; j8 < 4; ++j8) {
        uint4 oh, ol;
#pragma unroll
        for (int e = 0; e < 4; ++e) split_f32x2(pair(4 * j8 + e), reinterpret_cast<__half2*>(&oh)[e], reinterpret_cast<__half2*>(&ol)[e]);
        sts128(smem_u32(sh) + stg64_off(r_in_tile, j8), oh);
        sts128(smem_u32(sl) + stg64_off(r_in_tile, j8), ol);
      }
      fence_async_smem();
      epi_bar();
      if (leader) {
        tma_store_2d(&maps.out_hi, sh, col, row);
        tma_store_2d(&maps.out_lo, sl, col, row);
        tma_store_commit();
      }
    };
    // PP: warpgroup wg runs the CTA's units tl = wg, wg + 2, ...; k-block kb of unit tl is ring position tl * nkb + kb
    const int unit_step = PP ? 2 * gridDim.x : gridDim.x;
    uint32_t it = PP ? wg * nkb : 0;
    for (int u = blockIdx.x + (PP ? wg * gridDim.x : 0), tl = PP ? wg : 0; u < total_units; u += unit_step, tl += PP ? 2 : 1) {
      const int z = u / units_per_batch, rem = u - z * units_per_batch;
      const int m_tile = rem / p.n_tiles, n_tile = rem % p.n_tiles;
      // PP: the other warpgroup has issued the MMAs of unit tl - 1 (its ((tl - 1) >> 1)-th arrival on order_bar[wg]).  Only
      // then are the full barriers of this unit's k-blocks at most one phase behind the one awaited.
      if (PP && tl > 0) mbar_wait(&order_bar[wg], ((tl - 1) >> 1) & 1);
#pragma unroll
      for (int i = 0; i < kRegs; ++i) {
        acc[i] = 0.f;
        if (kSplitAcc) acc_c[i] = 0.f;
        if (kMainAcc > 1) { acc_m1[i] = 0.f; acc_m2[i] = 0.f; }
      }
      int prev_s = -1;
      if (halo) {
        const int ngroups = 3 * p.kb_per_tap;
        for (int g = 0; g < ngroups; ++g, ++it) {
          const int s = it % kHaloStagesDiv;
          mbar_wait(&full_bar[s], (it / kHaloStagesDiv) & 1);
          const uint32_t sa_h = smem_u32(smem + s * kHaloStageBytes) + a_off, sa_l = sa_h + kHaloABytes;
          const uint32_t sb0 = smem_u32(smem + s * kHaloStageBytes) + 2 * kHaloABytes;
          const int am = (g / p.kb_per_tap) % n_main;             // kernel row -> main accumulator
          wgmma_fence();
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const uint32_t sb_h = sb0 + dx * 2 * kBBytes, sb_l = sb_h + kBBytes;
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k) {
              const uint32_t koff = k * MMA_K * 2;
              const uint64_t ah = make_desc(sa_h + dx * 128 + koff), al = make_desc(sa_l + dx * 128 + koff);
              const uint64_t bh = make_desc(sb_h + koff), bl = make_desc(sb_l + koff);
              mma_main(am, ah, bh);
              mma_k16<BN>(acc_c, ah, bl);
              mma_k16<BN>(acc_c, al, bh);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev_s >= 0) release(prev_s);
          prev_s = s;
        }
      } else {
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(ACV != ACV_NONE ? &conv_bar[s] : &full_bar[s], (it / kStages) & 1);
          uint8_t* st = smem + s * kStageBytes;
          const uint32_t sa_h = smem_u32(st) + a_off;
          const uint32_t sa_l = sa_h + kABytes, sb_h = smem_u32(st) + kBOff, sb_l = sb_h + kBBytes;
          wgmma_fence();
          if (ACV != ACV_NONE && kb >= nkb1) {
            // the identity K-block, B_lo == 0: the A_hi.B_lo pass would add exact zeros.  A chain of its own, so that no branch
            // sits between MMAs.
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k) {
              const uint32_t koff = k * MMA_K * 2;
              const uint64_t bh = make_desc(sb_h + koff), ah = make_desc(sa_h + koff), al = make_desc(sa_l + koff);
              mma_k16<BN>(acc, ah, bh);
              mma_k16<BN>(acc, al, bh);
            }
            wgmma_commit();
          } else {
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k) {
              const uint32_t koff = k * MMA_K * 2;   // bytes inside the swizzle row
              const uint64_t ah = make_desc(sa_h + koff), al = make_desc(sa_l + koff);
              const uint64_t bh = make_desc(sb_h + koff), bl = make_desc(sb_l + koff);
              if (kSplitAcc) {                                        // narrow tiles: never HI / K2 blocks (launch_gemm_tc)
                const int dy = (EPI == EPI_CONV && p.taps == 9) ? kb / (3 * p.kb_per_tap) : 0;
                mma_main(dy % n_main, ah, bh);
                mma_k16<BN>(acc_c, ah, bl);
                mma_k16<BN>(acc_c, al, bh);
                continue;
              }
              mma_k16<BN>(acc, ah, bh);
              mma_k16<BN>(acc, ah, bl);
              if (!HI) mma_k16<BN>(acc, al, bh);
              if (PP) {                                               // rows [64, 128) of the tile: the second accumulator
                const uint64_t ah1 = make_desc(sa_h + kHalfOff + koff), al1 = make_desc(sa_l + kHalfOff + koff);
                float* acc1 = acc + (PP ? 64 : 0);
                mma_k16<BN>(acc1, ah1, bh);
                mma_k16<BN>(acc1, ah1, bl);
                mma_k16<BN>(acc1, al1, bh);
              }
            }
            wgmma_commit();
          }
          wgmma_wait<1>();                                           // the previous k-block's MMAs are done: free its stage
          if (prev_s >= 0) release(prev_s);
          prev_s = s;
        }
      }
      if (PP) {                                                       // hand the tensor pipe to the other warpgroup
        it += nkb;                                                    // (skip the other warpgroup's unit tl + 1)
        __syncwarp();
        if (lane == 0) mbar_arrive(&order_bar[wg ^ 1]);
      }
      wgmma_wait<0>();
      fence_regs<kRegs>(acc);
      if (kSplitAcc) fence_regs<kRegs>(acc_c);
      if (kMainAcc > 1) { fence_regs<kRegs>(acc_m1); fence_regs<kRegs>(acc_m2); }
      if (prev_s >= 0) release(prev_s);
      // ---- park the accumulator: fragment -> the eight boxes (BN 256), or acc_smem [BM][kAccLd] (narrow tiles: split
      // accumulators summed with round-to-nearest); PP parks chunk by chunk in ld32
      if (!PP) consumers_bar();                                       // both warpgroups' MMAs have finished reading the ring
      if (kStagePark) {
        park_stage = smem + prev_s * kStageBytes;                     // the last k-block's stage
        const int r = 64 * wg + 16 * q + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int g = 0; g < BN / 8; ++g) {                            // columns 8 g + cq, + 1 of rows r, r + 8
          float* p0 = reinterpret_cast<float*>(park_box(g >> 2) + stg_off(r, 2 * (g & 3) + (cq >> 2))) + (cq & 3);
          *reinterpret_cast<float2*>(p0) = make_float2(acc[4 * g], acc[4 * g + 1]);
          *reinterpret_cast<float2*>(p0 + 8 * 32) = make_float2(acc[4 * g + 2], acc[4 * g + 3]);   // stg_off(r + 8, j) = + 1024 B
        }
      } else if (!PP) {
        const int r = 64 * wg + 16 * q + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int g = 0; g < BN / 8; ++g) {
          float v[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            v[e] = acc[4 * g + e];
            if (kSplitAcc) v[e] += acc_c[4 * g + e];
            if (kMainAcc > 1 && n_main > 1) { v[e] += acc_m1[4 * g + e]; v[e] += acc_m2[4 * g + e]; }
          }
          *reinterpret_cast<float2*>(acc_smem + r * kAccLd + 8 * g + cq) = make_float2(v[0], v[1]);
          *reinterpret_cast<float2*>(acc_smem + (r + 8) * kAccLd + 8 * g + cq) = make_float2(v[2], v[3]);
        }
      }
      if (!PP) consumers_bar();
      // 32 accumulator columns of this thread's row starting at column c (a multiple of 32)
      auto ld32 = [&](int c, uint32_t (&v)[32]) {
        if (PP) {
          // fragment columns [c, c + 32) of both accumulators -> the group's box, once the store that last read the box is
          // done with it and every thread has finished with its previous contents
          const uint32_t box = smem_u32(park_box(0));
          if (leader) tma_store_wait_read<0>();
          epi_bar();
          const int cq = 2 * (lane & 3);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = 64 * h + 16 * q + (lane >> 2);
#pragma unroll
            for (int g = 0; g < BN / 8; ++g) {                          // columns 8 g + cq, + 1 of rows r, r + 8
              if ((g >> 2) != (c >> 5)) continue;
              const float* a = acc + 64 * h + 4 * g;
              const uint32_t p0 = box + stg_off(r, 2 * (g & 3) + (cq >> 2)) + (cq & 3) * 4;
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p0), "f"(a[0]), "f"(a[1]) : "memory");
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p0 + 1024), "f"(a[2]), "f"(a[3]) : "memory");   // row r + 8
            }
          }
          epi_bar();
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 f = lds128(box + stg_off(r_in_tile, j));
            v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y); v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
          }
          return;
        }
        if (kStagePark) {
          const uint32_t box = smem_u32(park_box(c >> 5));
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 f = lds128(box + stg_off(r_in_tile, j));
            v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y); v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
          }
          return;
        }
        const float* src = acc_smem + r_in_tile * kAccLd + c;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 f = *reinterpret_cast<const float4*>(src + 4 * j);
          v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y); v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
        }
      };
      // PP: the chunk loops are unrolled, so that the fragment registers of a chunk are free once it has been parked (the
      // whole accumulator would otherwise stay live through the epilogue and spill)
      constexpr int kChunkUnroll = PP ? 4 : 1;
      const int out_row0 = z * p.c_batch_rows + m_tile * BM;
      const int row0 = m_tile * BM;                               // within the batch
      int n_valid = BM;                                           // valid rows of this tile (segment-aware launches)
      int seg = 0;
      if (p.seg_rows) {
        seg = p.L.seg_of_row(row0);
        n_valid = p.L.seg_valid(seg) - (row0 - p.L.seg_start(seg));
      }
      if (EPI == EPI_F32 || EPI == EPI_F32_STATS) {
        // ---- fp32 tile out through swizzled staging + TMA store, 32 columns per chunk
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 32) {
          uint32_t v[32];
          ld32(c0, v);
          const int col0 = n_tile * BN + c0;
          uint8_t* sb = chunk_buf(c0);
          stage_wait();                             // the store that last read this buffer is done with it
          epi_bar();
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float4 o;
            o.x = __uint_as_float(v[4 * j + 0]) * kProdInv;
            o.y = __uint_as_float(v[4 * j + 1]) * kProdInv;
            o.z = __uint_as_float(v[4 * j + 2]) * kProdInv;
            o.w = __uint_as_float(v[4 * j + 3]) * kProdInv;
            if (p.bias) {
              const float4 bb = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + 4 * j));
              o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w;
            }
            sts128(smem_u32(sb) + stg_off(r_in_tile, j), make_uint4(__float_as_uint(o.x), __float_as_uint(o.y), __float_as_uint(o.z), __float_as_uint(o.w)));
          }
          fence_async_smem();
          epi_bar();
          if (leader) {
            tma_store_2d(&maps.out_f32, sb, col0, out_row0);
            tma_store_commit();
          }
          if (EPI == EPI_F32_STATS) {
            // InstanceNorm partials straight from the staged tile: thread = (32-row quarter, column); the sum and the sum of
            // squared deviations from the quarter's mean, two passes over the 32 staged values (the one-pass sum(x^2) - n mean^2
            // cancels catastrophically when a channel's mean is large against its spread)
            const int t = t_in_grp, qq = t >> 5, cc = t & 31;
            const int r_end = min(32, n_valid - qq * 32);
            const uint32_t sbu = smem_u32(sb) + (cc & 3) * 4;
            auto staged = [&](int i) {
              float x;
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(sbu + stg_off(qq * 32 + i, cc >> 2)));
              return x;
            };
            float sum = 0.f, m2 = 0.f;
            for (int i = 0; i < r_end; ++i) sum += staged(i);
            const float mq = r_end > 0 ? sum / (float)r_end : 0.f;
            for (int i = 0; i < r_end; ++i) {
              const float d = staged(i) - mq;
              m2 = fmaf(d, d, m2);
            }
            float2* dst = reinterpret_cast<float2*>(p.statpart) + ((long long)(out_row0 / 32 + qq) * p.n_out + col0 + cc);
            *dst = make_float2(sum, m2);
          }
        }
      } else if (EPI == EPI_QKV) {
        // ---- [K | V] tiles of the k,v projection -> one fp16 plane (x 2^6), 64 columns per chunk (128-byte staging rows).
        // elu+1 on K (GATs_SuperGlue.py:71-72); pad rows are zeroed so the state kernel needs no row masks.
        const bool is_k = n_tile == 0;
        const bool row_ok = r_in_tile < n_valid;
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 64) {
          uint32_t v0[32], v1[32];
          ld32(c0, v0);
          ld32(c0 + 32, v1);
          const int col0 = n_tile * BN + c0;
          uint8_t* sb = chunk_buf(c0);
          stage_wait();
          epi_bar();
#pragma unroll
          for (int j8 = 0; j8 < 8; ++j8) {
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + j8 * 8));
            const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + j8 * 8 + 4));
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            float x[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int jj = j8 * 8 + e;
              x[e] = fmaf(__uint_as_float(jj < 32 ? v0[jj & 31] : v1[jj & 31]), kProdInv, bb[e]);
              if (is_k) x[e] = elu1_fast(x[e]);
              x[e] = row_ok ? x[e] * kPre : 0.f;
            }
            uint4 o;
#pragma unroll
            for (int e = 0; e < 4; ++e) reinterpret_cast<__half2*>(&o)[e] = __float22half2_rn(make_float2(x[2 * e], x[2 * e + 1]));
            sts128(smem_u32(sb) + stg_off(r_in_tile, j8), o);
          }
          fence_async_smem();
          epi_bar();
          if (leader) {
            tma_store_2d(&maps.out_hi, sb, col0, out_row0);
            tma_store_commit();
          }
        }
      } else if (EPI == EPI_SCORE_SUMS) {
        // ---- dual-softmax tail, pass 1 (reference GATs_SuperGlue.py:217-218).  Unit-norm operands: cos <= 1, so with the
        // fixed shift  e = exp((cos - 1)/scale)  softmax(s,1)*softmax(s,2) = e^2 / (colsum*rowsum)  needs no running max.
        // Nothing is stored but the partial sums: row sums per (tile half, row) in registers; column sums over the warp's 32
        // rows by a transposing butterfly (31 shuffles per 32 x 32 block, no shared memory, no barriers).
        const int Nz = p.L.n_of(z), M = p.L.m_of(z);
        const int row = row0 + r_in_tile;                          // query index inside frame z
        const bool row_ok = row < Nz;
        const float ea = kProdInv * p.inv_scale * 1.4426950408889634f, eb = -p.inv_scale * 1.4426950408889634f;
        float rs = 0.f;
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 32) {
          uint32_t v[32];
          ld32(c0, v);
          const int col0 = n_tile * BN + c0;
          float e[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const bool ok = row_ok && (col0 + j) < M;
            e[j] = ok ? ex2_fast(fmaf(__uint_as_float(v[j]), ea, eb)) : 0.f;
            rs += e[j];
          }
          // after the butterfly lane l holds the sum over the warp's 32 rows of column col0 + l
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < off; ++i) {
              const float keep = up ? e[i + off] : e[i];
              const float send = up ? e[i] : e[i + off];
              e[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
          }
          p.colsum_part[((long long)z * (p.m_tiles * 4) + m_tile * 4 + q) * p.L.m_pad + col0 + lane] = e[0];
        }
        // one row sum per 128-column tile of the score matrix
        p.rowsum_part[((long long)z * p.n_tiles + n_tile) * p.L.n_pad + row] = rs;
      } else if (EPI == EPI_SCORE_CONF) {
        // ---- dual-softmax tail, pass 2: conf = (e / rowsum) * (e / colsum) recomputed from the accumulator (the cos matrix is
        // never materialised), optional conf store, packed row / column arg-max (reference :218-220).  The 32-column chunk is
        // staged once in shared memory: it feeds the TMA store of conf and the per-column scan of the arg-max.
        // M: valid columns of frame z; conf rows are conf_ld wide (columns [M, conf_ld) hold 0), colbest rows L.M wide
        const int Nz = p.L.n_of(z), M = p.L.m_of(z), ldm = p.conf_ld;
        const int row = row0 + r_in_tile;
        const bool row_ok = row < Nz;
        const float ea = kProdInv * p.inv_scale * 1.4426950408889634f, eb = -p.inv_scale * 1.4426950408889634f;
        const int t = t_in_grp, qq = t >> 5, cc = t & 31;          // column-scan role: (32-row quarter, column)
        const float irs = row_ok ? __ldg(p.inv_rowsum + (long long)z * p.L.n_pad + row) : 0.f;
        float* ics = extra + grp * kColsPerGroup;                   // this tile half's inverse column sums
        epi_bar();                                                  // every thread of the group is done with the previous tile's values
        ics[t] = __ldg(p.inv_colsum + (long long)z * p.L.m_pad + n_tile * BN + c_begin + t);
        epi_bar();
        // running row arg-max as (value, column): columns are visited in ascending order and only a STRICTLY larger value
        // replaces the best, so the first maximum wins like torch.max; packed once per tile for the 64-bit atomicMax
        float rbest_v = 0.f;
        int rbest_c = -1;
        const bool store_plain = p.conf != nullptr && !p.conf_tma;
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 32) {
          uint32_t v[32];
          ld32(c0, v);
          const int col0 = n_tile * BN + c0;
          uint8_t* sb = chunk_buf(c0);
          float o[32];
#pragma unroll
          for (int j4 = 0; j4 < 8; ++j4) {
            const float4 ic4 = *reinterpret_cast<const float4*>(ics + (c0 - c_begin) + 4 * j4);   // broadcast read
            const float icv[4] = {ic4.x, ic4.y, ic4.z, ic4.w};
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * j4 + jj;
              const bool ok = row_ok && (col0 + j) < M;
              const float e = ok ? ex2_fast(fmaf(__uint_as_float(v[j]), ea, eb)) : 0.f;
              const float c = (e * irs) * (e * icv[jj]);
              o[j] = c;
              if (c > rbest_v) { rbest_v = c; rbest_c = col0 + j; }
            }
          }
          if (!kStagePark && p.conf_tma && leader) tma_store_wait_read<0>();   // the store that last read this group's buffer is done with it
          epi_bar();                                                // ... and every thread has finished scanning the previous chunk
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(sb + stg_off(r_in_tile, j)) = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
          if (p.conf_tma) fence_async_smem();
          epi_bar();
          if (p.conf_tma && leader) {
            tma_store_3d(&maps.out_f32, sb, col0, row0, z);         // rows >= N and columns >= M are clipped by the tensor map
            tma_store_commit();
          }
          // column scan over the staged 128 x 32 chunk: thread (qq, cc) = rows [32 qq, +32) of column col0 + cc.  Fully unrolled
          // (invalid rows hold 0 and can never win): 32 independent shared-memory loads in flight instead of a latency chain.
          const int col = col0 + cc;
          if (col < ldm) {                                          // columns >= M hold 0 and never win the column arg-max
            const int r_first = row0 + qq * 32;
            float cbest_v = 0.f;
            int cbest_r = -1;
            float cv[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) cv[i] = *reinterpret_cast<const float*>(sb + stg_off(qq * 32 + i, cc >> 2) + (cc & 3) * 4);
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (cv[i] > cbest_v) { cbest_v = cv[i]; cbest_r = r_first + i; }
            if (store_plain) {                                      // 32 consecutive columns of one row per warp instruction; rows
              float* crow = p.conf + ((long long)z * p.L.N + r_first) * ldm + col;     // [Nz, N) of a ragged frame are written as 0
#pragma unroll
              for (int i = 0; i < 32; ++i, crow += ldm)  // a stepped pointer: offsets i * M would be hoisted out of the chunk
                if (r_first + i < p.L.N) *crow = cv[i];     // loop as 32 loop-invariant values and spilled
            }
            if (cbest_r >= 0)
              atomicMax(p.colbest + (long long)z * p.L.M + col,
                        ((unsigned long long)__float_as_uint(cbest_v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)cbest_r));
          }
        }
        if (rbest_c >= 0)
          atomicMax(p.rowbest + (long long)z * p.L.N + row,
                    ((unsigned long long)__float_as_uint(rbest_v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)rbest_c));
      } else if (EPI == EPI_CONV || EPI == EPI_BIAS_PLANES) {
        // ---- out planes = [ReLU](acc + bias), 32 columns per chunk; rows that are no output are written as zero.
        // EPI_CONV: a convolution layer; the grid's border and padding rows are zero because the output is the next layer's
        // zero-bordered input.  EPI_BIAS_PLANES: a residual, if any, already sits in the accumulator (identity K-block); rows
        // past the segment's valid count are zero so that padding never accumulates state.
        bool row_ok;
        if (EPI == EPI_CONV) {
          const long long grow = (long long)out_row0 + r_in_tile;
          const int qpix = (int)(grow % p.cv_ppad);
          const int yy = qpix / p.cv_w2, xx = qpix - yy * p.cv_w2;
          row_ok = yy >= 1 && yy <= p.cv_h && xx >= 1 && xx <= p.cv_w;
        } else {
          row_ok = r_in_tile < n_valid;
        }
        const bool relu = EPI == EPI_CONV && p.relu;
        float peak = 0.f;              // EPI_CONV range guard: the largest |output| of this thread's row (see split_out_of_range)
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 32) {
          uint32_t v[32];
          ld32(c0, v);
          const int col0 = n_tile * BN + c0;
          store_planes32(c0, col0, out_row0, [&](int j) {
            const float2 bb = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col0) + j) : make_float2(0.f, 0.f);
            float2 sc = make_float2(fmaf(__uint_as_float(v[2 * j]), kPreInv, bb.x * kPre), fmaf(__uint_as_float(v[2 * j + 1]), kPreInv, bb.y * kPre));
            if (relu) sc = make_float2(fmaxf(sc.x, 0.f), fmaxf(sc.y, 0.f));
            if (EPI == EPI_CONV) peak = fmaxf(peak, fmaxf(fabsf(sc.x), fabsf(sc.y)));
            return row_ok ? sc : make_float2(0.f, 0.f);
          });
        }
        if (EPI == EPI_CONV && __any_sync(0xffffffffu, row_ok && split_out_of_range(peak)) && lane == 0 && p.range_flag) atomicOr(p.range_flag, 1);
      } else {
        // ---- planes out (row-major, 64 columns per chunk): EPI_QSCALE / EPI_L2NORM
        float inv_norm = 1.f;
        if (EPI == EPI_L2NORM) {                    // F.normalize: first pass over the accumulator for the row norm
          float ssp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
          for (int c0 = 0; c0 < BN; c0 += 32) {
            uint32_t v[32];
            ld32(c0, v);
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 bb = __ldg(reinterpret_cast<const float4*>(p.bias + c0) + j4);
              const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float x = fmaf(__uint_as_float(v[4 * j4 + e]), kProdInv, bv[e]);
                ssp[e] = fmaf(x, x, ssp[e]);
              }
            }
          }
          inv_norm = 1.f / fmaxf(sqrtf((ssp[0] + ssp[1]) + (ssp[2] + ssp[3])), 1e-12f);
          if (kStagePark) consumers_bar();          // both groups have read the whole row before either stages in place
        }
        int src = 0;
        float eps_m = 0.f;
        if (EPI == EPI_QSCALE) {
          src = p.L.src_seg(seg, p.cross);
          eps_m = 1e-6f / (float)max(p.L.seg_valid(src), 1);
        }
#pragma unroll kChunkUnroll
        for (int c0 = c_begin; c0 < c_end; c0 += 64) {
          uint32_t v0[32], v1[32];
          ld32(c0, v0);
          ld32(c0 + 32, v1);
          const int col0 = n_tile * BN + c0;
          float x[64];
          // warp-uniform parameter reads as 16-byte loads: 16 instead of 64 load instructions per chunk and thread
          const float4* bias4 = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
          for (int j4 = 0; j4 < 16; ++j4) {
            const float4 bb = __ldg(bias4 + j4);
            const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int j = 4 * j4 + e;
              x[j] = fmaf(__uint_as_float(j < 32 ? v0[j & 31] : v1[j & 31]), kProdInv, bv[e]);
            }
          }
          if (EPI == EPI_QSCALE) {
            // one 64-column chunk = one head (head-contiguous channels); the row's head dot product is thread-local
            const float4* km4 = reinterpret_cast<const float4*>(p.kmean + (long long)src * kD + col0);
            float dotp[4] = {0.f, 0.f, 0.f, 0.f};          // four independent chains instead of one 64-long dependent FFMA chain
#pragma unroll
            for (int j4 = 0; j4 < 16; ++j4) {
              const float4 kk = __ldg(km4 + j4);
              const float kv4[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int j = 4 * j4 + e;
                x[j] = elu1_fast(x[j]);
                dotp[e] = fmaf(x[j], kv4[e], dotp[e]);
              }
            }
            const float dot = (dotp[0] + dotp[1]) + (dotp[2] + dotp[3]);
            // a segment whose source has no valid rows (a frame without queries, in a cross layer) receives no message: Q' = 0.
            // q / eps_m would leave the fp16-split range and turn the message into inf x 0 = NaN
            const float zf = p.L.seg_valid(src) > 0 ? 1.f / (dot + eps_m) : 0.f;
#pragma unroll
            for (int j = 0; j < 64; ++j) x[j] *= zf;
          } else {  // EPI_L2NORM
#pragma unroll
            for (int j = 0; j < 64; ++j) x[j] *= inv_norm;
          }
          // two 32-column sub-chunks
#pragma unroll
          for (int sc = 0; sc < 2; ++sc)
            store_planes32(c0 + sc * 32, col0 + sc * 32, out_row0, [&](int j) { return make_float2(x[sc * 32 + 2 * j] * kPre, x[sc * 32 + 2 * j + 1] * kPre); });
        }
      }
      // the next tile's loads refill the ring: order this thread's reads of the parked tile before them (kStagePark: and the
      // stores staged in the boxes have read them)
      if (!PP) {                                // (PP: the next tile's epilogue waits on its own box in ld32)
        if (kStagePark && leader) tma_store_wait_read<0>();
        fence_async_smem();
        consumers_bar();
        if (threadIdx.x == 0) mbar_arrive(acc_free_bar);
      }
    }
    if (leader) tma_store_wait_all();
  }
  __syncthreads();
}

// ------------------------------------------------------------------ host: tensor maps
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(f);
  });
  return fn;
}

// 2D row-major tensor [rows, ld] (cols used: `cols`), box = box_cols x box_rows.  Swizzle follows the box row
// width (128 B -> SWIZZLE_128B, 64 B -> SWIZZLE_64B, anything else -> none).  Cached per (ptr, shape, box, dtype).
bool make_map(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows, bool f32) {
  const size_t esize = f32 ? 4 : 2;
  const size_t row_bytes = box_cols * esize;
  const CUtensorMapSwizzle swz = row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE);
  static std::map<std::tuple<const void*, long long, long long, long long, int, int, bool>, CUtensorMap> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  auto key = std::make_tuple(ptr, rows, cols, ld, box_cols, box_rows, f32);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return true; }
  EncodeFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  if (cache.size() > 4096) cache.clear();
  cache[key] = *out;
  return true;
}

// conf [B][N][M] fp32 as a 3-D tensor (box 32 x 128 x 1, SWIZZLE_128B): a 128-row tile that hangs over the end of a
// frame (rows >= N) or of a row (columns >= M) is clipped by the hardware.  Needs M % 4 == 0 (16-byte global strides)
// and a 16-byte aligned base.
bool make_map3(CUtensorMap* out, const float* ptr, int M, int N, int B) {
  EncodeFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[3] = {(cuuint64_t)M, (cuuint64_t)N, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)M * 4, (cuuint64_t)M * N * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)BM, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int g_conv_halo = 1;      // 0: nine row-shifted boxes per tile; 1: halo boxes (default)
int conv_halo_mode() { return g_conv_halo; }

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

template <int EPI, int ACV = ACV_NONE, bool HI = false, int BN_ = 256, bool PP = false>
cudaError_t launch_variant(int grid, cudaStream_t stream, const Maps& mp, const TcParams& tp) {
  auto* kern = gemm_tc_kernel<EPI, ACV, HI, BN_, PP>;
  if (cudaError_t e = ensure_smem_limit((const void*)kern, kSmemBytes)) return e;
  return launch_k(pdl_enabled(), kern, dim3(grid), dim3(kThreads), kSmemBytes, stream, mp, tp);
}

}  // namespace

cudaError_t ensure_smem_limit(const void* func, int bytes) {
  static std::map<std::pair<const void*, int>, int> done;   // (kernel, device) -> limit set
  static std::mutex mu;
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  std::lock_guard<std::mutex> lk(mu);
  int& set = done[{func, dev}];
  if (bytes <= set) return cudaSuccess;
  if (cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)) return e;
  set = bytes;
  return cudaSuccess;
}

void set_conv_halo_mode(int mode) { g_conv_halo = mode ? 1 : 0; }

bool make_tensor_map_2d(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows, bool f32) {
  return make_map(out, ptr, rows, cols, ld, box_cols, box_rows, f32);
}

int launch_gemm_tc(const GemmProblem& p, cudaStream_t stream) {
  const int bn = p.bn ? p.bn : BN;                 // column-tile width
  const bool bn_ok = p.epi == EPI_CONV ? bn == 64 || bn == 128 : p.epi == EPI_F32 ? bn == 128 || bn == BN : bn == BN;
  if (!bn_ok || (bn != BN && (p.K2 || p.a_conv || p.a_hi_only))) return -1;
  if (p.rows % (2 * BM) || p.n_out % bn || p.K1 % BK || p.K2 % BK || p.K1 <= 0 || p.batch <= 0) return -1;
  if ((p.epi == EPI_QSCALE || p.epi == EPI_L2NORM || p.epi == EPI_BIAS_PLANES) && p.n_out != BN) return -1;
  if (p.taps && (p.epi != EPI_CONV || p.taps > 9 || p.kb_per_tap <= 0 || p.taps * p.kb_per_tap * BK != p.K1 || p.K2 || p.batch != 1)) return -1;
  if (p.epi == EPI_CONV && (!p.bias || !p.out.hi || !p.out.lo || p.cv_ppad <= 0 || p.cv_w2 <= 0 || p.batch != 1)) return -1;
  if (p.a_hi_only && (p.a_conv || p.K2 || p.epi != EPI_QKV)) return -1;
  if (p.a_conv && (p.a_conv != ACV_NORM_RELU || p.batch != 1 || !p.a_raw || p.epi != EPI_BIAS_PLANES || p.b2_per_seg || !p.mu || !p.rstd)) return -1;
  const bool f32_out = p.epi == EPI_F32 || p.epi == EPI_F32_STATS;
  // the ping-pong schedule runs every 256-column problem of these epilogues as 128-column tiles (DESIGN.md 5.1)
  const bool pp = bn == BN && (f32_out || p.epi == EPI_SCORE_SUMS);
  const int tile_n = pp ? 128 : bn;                // column width of a tile
  // halo convolution: 3x3 taps in row-major order with unit horizontal steps, 64-column tiles (wider tiles have no room for two
  // halo stages in the ring)
  int halo = (p.epi == EPI_CONV && p.taps == 9 && bn == 64) ? conv_halo_mode() : 0;
  for (int t = 0; t < 9 && halo; ++t)
    if (p.tap_off[t] != (t / 3 - 1) * p.cv_w2 + (t % 3 - 1)) halo = 0;
  if (p.epi == EPI_QKV && (p.n_out != 2 * BN || p.batch != 1 || !p.out.hi || !p.bias)) return -1;
  if ((p.epi == EPI_QSCALE || p.epi == EPI_L2NORM) && !p.bias) return -1;
  const bool score = p.epi == EPI_SCORE_SUMS || p.epi == EPI_SCORE_CONF;
  int conf_tma = 0;
  const int conf_ld = p.conf_ld ? p.conf_ld : p.L.M;
  if (score && conf_ld < p.L.M) return -1;
  if (f32_out && (p.ldc % 4 || !p.c)) return -1;
  const long long a_rows = (long long)(p.batch - 1) * p.a_batch_rows + p.rows;
  const long long b1_rows = (long long)(p.batch - 1) * p.b_batch_rows + p.n_out;
  const long long b2_rows = p.b2_per_seg ? (long long)p.L.segs() * p.n_out : p.n_out;
  Maps mp;
  bool ok = make_map(&mp.b1h, p.b1.hi, b1_rows, p.K1, p.b1.ld, BK, tile_n, false) && make_map(&mp.b1l, p.b1.lo, b1_rows, p.K1, p.b1.ld, BK, tile_n, false);
  if (p.a_conv) { mp.a1h = mp.b1h; mp.a1l = mp.b1l; }     // every A1 tile comes in raw: the plane maps are never used
  else {
    const long long a_cols = p.taps ? (long long)p.kb_per_tap * BK : p.K1;      // convolution: A has C_in columns, the taps shift its rows
    const int a_box_rows = halo ? BM + 2 : BM;                                   // halo convolution: one box serves the three horizontal taps
    ok = ok && make_map(&mp.a1h, p.a1.hi, a_rows, a_cols, p.a1.ld, BK, a_box_rows, false) && make_map(&mp.a1l, p.a1.lo, a_rows, a_cols, p.a1.ld, BK, a_box_rows, false);
  }
  if (ok && p.a_conv) ok = make_map(&mp.a_raw, p.a_raw, a_rows, p.K1, p.a_raw_ld, 32, BM, true);
  else mp.a_raw = mp.b1h;
  if (ok && p.K2) {
    ok = make_map(&mp.b2h, p.b2.hi, b2_rows, p.K2, p.b2.ld, BK, tile_n, false) && make_map(&mp.b2l, p.b2.lo, b2_rows, p.K2, p.b2.ld, BK, tile_n, false) &&
         make_map(&mp.a2h, p.a2.hi, a_rows, p.K2, p.a2.ld, BK, BM, false) && make_map(&mp.a2l, p.a2.lo, a_rows, p.K2, p.a2.ld, BK, BM, false);
  } else if (ok) {
    mp.a2h = mp.a1h; mp.a2l = mp.a1l; mp.b2h = mp.b1h; mp.b2l = mp.b1l;
  }
  const long long out_rows = (long long)p.batch * p.rows;
  if (f32_out) {
    ok = ok && make_map(&mp.out_f32, p.c, out_rows, p.n_out, p.ldc, 32, BM, true);
    mp.out_hi = mp.out_f32; mp.out_lo = mp.out_f32;
  } else if (p.epi == EPI_QKV) {
    ok = ok && make_map(&mp.out_hi, p.out.hi, out_rows, 2 * BN, p.out.ld, 64, BM, false);
    mp.out_f32 = mp.out_hi;
    mp.out_lo = mp.out_hi;
  } else if (score) {
    mp.out_f32 = mp.b1h; mp.out_hi = mp.b1h; mp.out_lo = mp.b1h;
    if (p.epi == EPI_SCORE_CONF && p.conf && conf_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(p.conf) & 15) == 0)
      conf_tma = make_map3(&mp.out_f32, p.conf, conf_ld, p.L.N, p.batch) ? 1 : 0;
  } else {
    ok = ok && make_map(&mp.out_hi, p.out.hi, out_rows, p.n_out, p.out.ld, 32, BM, false) && make_map(&mp.out_lo, p.out.lo, out_rows, p.n_out, p.out.ld, 32, BM, false);
    mp.out_f32 = mp.out_hi;
  }
  if (!ok) return -2;
  TcParams tp{};
  tp.K1 = p.K1; tp.K2 = p.K2; tp.b2_per_seg = p.b2_per_seg; tp.n_out = p.n_out;
  // the zero-lo identity block exists for the residual GEMM mlp.3 (converted A), and the converter always comes with it
  if (p.b2_lo_zero && (p.epi != EPI_BIAS_PLANES || !p.K2 || !p.a_conv)) return -1;
  if (p.a_conv && !p.b2_lo_zero) return -1;
  tp.m_tiles = p.rows / BM; tp.n_tiles = p.n_out / tile_n; tp.batch = p.batch;
  tp.taps = p.taps; tp.kb_per_tap = p.kb_per_tap;
  for (int t = 0; t < 9; ++t) tp.tap_off[t] = p.tap_off[t];
  tp.cv_w2 = p.cv_w2; tp.cv_h = p.cv_h; tp.cv_w = p.cv_w; tp.cv_ppad = p.cv_ppad; tp.relu = p.relu; tp.range_flag = p.range_flag; tp.halo = halo;
  tp.a_batch_rows = p.a_batch_rows; tp.b_batch_rows = p.b_batch_rows; tp.c_batch_rows = p.rows;
  tp.seg_rows = (p.batch == 1 && p.L.R > 0 && p.L.rows() == p.rows) ? 1 : 0;
  tp.L = p.L; tp.bias = p.bias;
  tp.inv_scale = p.inv_scale; tp.rowsum_part = p.rowsum_part; tp.colsum_part = p.colsum_part; tp.inv_rowsum = p.inv_rowsum;
  tp.inv_colsum = p.inv_colsum; tp.conf = p.conf; tp.conf_tma = conf_tma; tp.conf_ld = conf_ld; tp.rowbest = p.rowbest; tp.colbest = p.colbest;
  tp.mu = p.mu; tp.rstd = p.rstd;
  tp.kmean = p.kmean; tp.cross = p.cross; tp.statpart = p.statpart;
  if ((p.epi == EPI_QSCALE || p.b2_per_seg || p.epi == EPI_QKV || p.epi == EPI_F32_STATS || p.a_conv) && !tp.seg_rows) return -1;
  const int total_units = tp.m_tiles * tp.n_tiles * tp.batch;
  int grid = total_units < num_sms() ? total_units : num_sms();
  if (p.max_ctas > 0 && grid > p.max_ctas) grid = p.max_ctas;      // test hook: the same tiles on fewer CTAs
  cudaError_t le;
  if (p.a_conv) {
    le = launch_variant<EPI_BIAS_PLANES, ACV_NORM_RELU>(grid, stream, mp, tp);
  } else {
    switch (p.epi) {
      case EPI_F32:
        le = bn == 128 ? launch_variant<EPI_F32, ACV_NONE, false, 128>(grid, stream, mp, tp)
                       : launch_variant<EPI_F32, ACV_NONE, false, 128, true>(grid, stream, mp, tp);
        break;
      case EPI_CONV:
        le = bn == 64 ? launch_variant<EPI_CONV, ACV_NONE, false, 64>(grid, stream, mp, tp) : launch_variant<EPI_CONV, ACV_NONE, false, 128>(grid, stream, mp, tp);
        break;
      case EPI_F32_STATS: le = launch_variant<EPI_F32_STATS, ACV_NONE, false, 128, true>(grid, stream, mp, tp); break;
      case EPI_QSCALE: le = launch_variant<EPI_QSCALE>(grid, stream, mp, tp); break;
      case EPI_L2NORM: le = launch_variant<EPI_L2NORM>(grid, stream, mp, tp); break;
      case EPI_SCORE_SUMS: le = launch_variant<EPI_SCORE_SUMS, ACV_NONE, false, 128, true>(grid, stream, mp, tp); break;
      case EPI_SCORE_CONF: le = launch_variant<EPI_SCORE_CONF>(grid, stream, mp, tp); break;
      case EPI_QKV: le = p.a_hi_only ? launch_variant<EPI_QKV, ACV_NONE, true>(grid, stream, mp, tp) : launch_variant<EPI_QKV>(grid, stream, mp, tp); break;
      case EPI_BIAS_PLANES: le = launch_variant<EPI_BIAS_PLANES>(grid, stream, mp, tp); break;
      default: return -1;
    }
  }
  if (le != cudaSuccess) return -2;
  return 0;
}

}  // namespace opb
