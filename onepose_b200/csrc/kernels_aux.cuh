// Bandwidth-bound helper kernels of the GATsSPG matcher (everything that is not a GEMM):
// layout changes, GATs aggregation, linear-attention state reduction, InstanceNorm statistics,
// dual-softmax bookkeeping, mutual-NN, and the adjacent producers (segmented means, leaf gathering).
// sm_90a; plain coalesced warp-per-row / block-per-tile kernels.  The kernels of the matcher's forward begin with
// griddep_sync() (programmatic dependent launch, see common.cuh).  split_planes, join_planes and the adjacent producers
// (exclusive_scan_i64, segmented_mean*, gather_*) do not: they are launched without PDL.
#pragma once
#include "block.cuh"
#include "common.cuh"
#include "gemm_tc.cuh"
#include "host_util.cuh"
#include "kv_state_tc.cuh"

namespace opb {

// ---------------------------------------------------------------------------------------
// Channel-first fp32 [batch][C=256][n_stride] -> point-major rows.  Row r of batch b lands at
// out row  b*out_batch_stride + row_offset + r.   (reference tensors are [B, D, n]:
// GATs_SuperGlue.py:184-186; the device works point-major so that a point is one 1 KB row.)
// MODE 0: fp16-split planes; rows [n_b, rows_out) are written as ZERO (n_b = nlen[b] for ragged batches, else n) so that
//         the padding of a segment never carries state from an earlier call.  MODE 1: fp32 rows, rows < n only.
// grid (ceil(rows_out/32), batch), block (32, 8)
// ---------------------------------------------------------------------------------------
template <int MODE>
__global__ void transpose_cf_to_rows(const float* __restrict__ in, int n, int n_stride, long long in_batch_stride, const int* __restrict__ nlen,
                                     int rows_out, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                                     float* __restrict__ out_f32, long long out_batch_stride_rows, int row_offset) {
  __shared__ float tile[kD][33];
  griddep_sync();
  const int p0 = blockIdx.x * 32;
  const float* src = in + (long long)blockIdx.y * in_batch_stride;
  const int nb = nlen ? min(max(nlen[blockIdx.y], 0), n) : n;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int c = ty; c < kD; c += 8) {
    int p = p0 + tx;
    tile[c][tx] = (p < nb) ? src[(long long)c * n_stride + p] : 0.f;
  }
  __syncthreads();
  const int tid = ty * 32 + tx;  // 256 threads = 256 channels
  const long long row_base = (long long)blockIdx.y * out_batch_stride_rows + row_offset + p0;
  const int p_end = MODE == 0 ? rows_out : nb;
  for (int p = 0; p < 32 && p0 + p < p_end; ++p) {
    float v = tile[tid][p];
    long long o = (row_base + p) * kD + tid;
    if (MODE == 0) {
      __half h, l;
      split_f32(v, h, l);
      out_hi[o] = h;
      out_lo[o] = l;
    } else {
      out_f32[o] = v;
    }
  }
}

// Per-chunk object table: which object each frame of the chunk matches against.  The host builds it for every chunk and
// hands it to assemble_layout BY VALUE (no host synchronisation, no staging buffer that a later call could overwrite while
// this one is in flight); assemble_layout also copies it into the workspace, where the later kernels of the chunk read it.
constexpr int kMaxChunkFrames = 64;
constexpr int kGatsFramesPerWarp = 16;   // leaf rows re-read once per 16 frames (8: 229 MB of leaf traffic per layer at B = 32, 16: 115 MB)
struct FrameObject {
  const __half* hi;       // the object's 3D rows [m_pad_obj, 256]: prologue state (hoisting) or raw db planes
  const __half* lo;
  const float* leaves;    // fp32 [M_b * L, 256] point-major
  const float* s2;        // [4][M_b * L] leaf logits of the 4 GATs layers
};
struct ChunkTable {
  FrameObject obj[kMaxChunkFrames];
  int mlen[kMaxChunkFrames];              // M_b: valid 3D rows of frame b (= Layout::mlen)
};
// GATs groups of a chunk for gats_aggregate_frames8, passed BY VALUE (read from the constant bank, no dependent global loads
// before the leaf rows): group g = frames [b_begin, b_end), a run of consecutive frames of one object, at most
// kGatsFramesPerWarp long.
struct GatsGroup {
  const float* leaves;    // the object's leaves [M * 8, 256]
  const float* s2;        // its leaf logits [4][M * 8]
  int b_begin, b_end, M, pad;
};
struct GatsGroups {
  GatsGroup g[kMaxChunkFrames];
  int n;
};

// Assemble the activation layout of a chunk: frame b's query segment from the compact query buffer xq [B*n_pad, 256] and its
// 3D-point segment from its object's rows tab.obj[b] (rows [M_b, m_pad) are written as zero).  Block (0, 0) also stores the
// table at tab_out.  One launch, 16-byte vectors.
// grid (blocks, B)
__global__ void assemble_layout(const __half* __restrict__ q_hi, const __half* __restrict__ q_lo, const __grid_constant__ ChunkTable tab,
                                ChunkTable* __restrict__ tab_out, __half* __restrict__ x_hi, __half* __restrict__ x_lo, Layout L) {
  griddep_sync();
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    const int* src = reinterpret_cast<const int*>(&tab);
    int* dst = reinterpret_cast<int*>(tab_out);
    for (int k = threadIdx.x; k < (int)(sizeof(ChunkTable) / sizeof(int)); k += blockDim.x) dst[k] = src[k];
  }
  const int b = blockIdx.y;
  const long long nq = q_hi ? (long long)L.n_pad * kD / 8 : 0;  // uint4 = 8 halves
  const long long nd = (long long)L.m_pad * kD / 8;
  const long long nvalid = (long long)tab.mlen[b] * kD / 8;
  const uint4* o_hi = reinterpret_cast<const uint4*>(tab.obj[b].hi);
  const uint4* o_lo = reinterpret_cast<const uint4*>(tab.obj[b].lo);
  const long long dst0 = (long long)b * L.R * kD / 8;
  const long long src_q0 = (long long)b * nq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nq + nd; i += (long long)gridDim.x * blockDim.x) {
    if (i < nq) {
      reinterpret_cast<uint4*>(x_hi)[dst0 + i] = reinterpret_cast<const uint4*>(q_hi)[src_q0 + i];
      reinterpret_cast<uint4*>(x_lo)[dst0 + i] = reinterpret_cast<const uint4*>(q_lo)[src_q0 + i];
    } else {
      const long long j = i - nq;
      const long long d = dst0 + (long long)L.n_pad * kD / 8 + j;
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      reinterpret_cast<uint4*>(x_hi)[d] = j < nvalid ? o_hi[j] : z;
      reinterpret_cast<uint4*>(x_lo)[d] = j < nvalid ? o_lo[j] : z;
    }
  }
}

// ---------------------------------------------------------------------------------------
// GATs: frame-invariant leaf logits  s2[layer][r] = leaf_row[r] . (W a[:256])_layer
// (reference GATs.py:40,78: wh_2d @ a[:out] == h_2d @ (W a[:out]) in exact arithmetic).
// warp per leaf row, all 4 GATs layers from one read.   wa2: [4][256]
// ---------------------------------------------------------------------------------------
__global__ void gats_leaf_logits(const float* __restrict__ leaves, long long n_rows,
                                 const float* __restrict__ wa2, float* __restrict__ s2) {
  griddep_sync();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  float w[4][8];
#pragma unroll
  for (int l = 0; l < 4; ++l)
#pragma unroll
    for (int j = 0; j < 8; ++j) w[l][j] = wa2[l * kD + (j >> 2) * 128 + lane * 4 + (j & 3)];
  for (long long r = warp; r < n_rows; r += n_warps) {
    const float4* row = reinterpret_cast<const float4*>(leaves + r * kD);
    float4 a = row[lane], b = row[32 + lane];
    float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(v[j], w[l][j], acc);
      acc = warp_sum(acc);
      if (lane == 0) s2[(long long)l * n_rows + r] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------
// GATs aggregation (reference GATs.py:35-88):
//   s3 = h3 . (W a[256:]);  e_self = LeakyReLU(2 s3);  e_j = LeakyReLU(s3 + s2_j)
//   att = softmax(e);  h' = att_self h3 + sum_j att_j leaf_j ;  out = ELU(h')
// include_self=0:  h' = sum_j att_j leaf_j / 2 + h3 (GATs.py:64-67); additional: h' += h3 (:61).
// with_linear_transform (GATs.py:56-57,64-65) multiplies the aggregated rows by W; aggregation and W commute
// (sum_j att_j (leaf_j W) = (sum_j att_j leaf_j) W), so `lin` = 1 writes the PRE-transform row
//   pre = att_self h3 + sum_j att_j leaf_j      (include_self)      |     sum_j att_j leaf_j / 2 + h3   (no self)
// to the compact buffer o_* [B*m_pad, 256] and the host finishes with one GEMM by W and gats_lin_finish.
// Writer shared by both aggregation kernels.
struct GatsOut {
  __half* hi;                 // lin = 0: the X planes (in place);  lin = 1: compact [B*m_pad, 256] planes
  __half* lo;
  int lin;
};
__device__ __forceinline__ void gats_write_row(const GatsOut& o, long long row, int lane, const float (&acc)[8], const float (&h3)[8],
                                               int include_self, int additional) {
  uint2 oh[2], ol[2];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float v = acc[j];
    if (!include_self) v = v * 0.5f + h3[j];
    else if (additional && !o.lin) v += h3[j];
    if (!o.lin) v = v > 0.f ? v : exp_fast(v) - 1.f;  // ELU (GATs.py:69-70); absolute error ~1e-7, the order of the fp16 split below
    __half hh, ll;
    split_f32(v, hh, ll);
    reinterpret_cast<__half*>(&oh[j >> 2])[j & 3] = hh;
    reinterpret_cast<__half*>(&ol[j >> 2])[j & 3] = ll;
  }
  uint2* qh = reinterpret_cast<uint2*>(o.hi + row * kD);
  uint2* ql = reinterpret_cast<uint2*>(o.lo + row * kD);
  qh[lane] = oh[0]; qh[32 + lane] = oh[1];
  ql[lane] = ol[0]; ql[32 + lane] = ol[1];
}
__device__ __forceinline__ void gats_read_h3(const __half* x_hi, const __half* x_lo, long long row, int lane, float (&h3)[8]) {
  // lane owns channels [lane*4, lane*4+4) and [128+lane*4, 128+lane*4+4)
  const uint2* ph = reinterpret_cast<const uint2*>(x_hi + row * kD);
  const uint2* pl = reinterpret_cast<const uint2*>(x_lo + row * kD);
#pragma unroll
  for (int half_i = 0; half_i < 2; ++half_i) {
    uint2 uh = ph[half_i * 32 + lane], ul = pl[half_i * 32 + lane];
    const __half* hh = reinterpret_cast<const __half*>(&uh);
    const __half* hl = reinterpret_cast<const __half*>(&ul);
#pragma unroll
    for (int j = 0; j < 4; ++j) h3[half_i * 4 + j] = join_f32(hh[j], hl[j]);
  }
}

// Generic leaf count: warp per (point, frame); frames of one point are adjacent warps so the leaf rows are served from
// L1/L2 after the first frame.  Frame b reads the leaves and the layer-`gi` leaf logits of its own object (tab->obj[b]).
__global__ void gats_aggregate(const __half* x_hi, const __half* x_lo, Layout L, const ChunkTable* __restrict__ tab, int n_leaf, int gi,
                               const float* __restrict__ wa3 /*[256]*/, int include_self, int additional,
                               float alpha, GatsOut out) {
  griddep_sync();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long total = (long long)L.M * L.B;
  if (warp >= total) return;
  const int b = (int)(warp % L.B);
  const int i = (int)(warp / L.B);
  const int Mb = tab->mlen[b];
  if (i >= Mb) return;
  const float* __restrict__ leaves = tab->obj[b].leaves;
  const float* __restrict__ s2 = tab->obj[b].s2 + (long long)gi * Mb * n_leaf;
  const long long row = (long long)b * L.R + L.n_pad + i;
  float h3[8];
  gats_read_h3(x_hi, x_lo, row, lane, h3);
  float s3 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) s3 = fmaf(h3[j], wa3[(j >> 2) * 128 + lane * 4 + (j & 3)], s3);
  s3 = warp_sum(s3);
  auto lrelu = [alpha](float v) { return v > 0.f ? v : alpha * v; };
  // logits of the leaves: lane j (< n_leaf) holds e_j
  float e = -INFINITY;
  if (lane < n_leaf) e = lrelu(s3 + s2[(long long)i * n_leaf + lane]);
  float e_self = include_self ? lrelu(2.f * s3) : -INFINITY;
  float mx = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  mx = fmaxf(mx, e_self);
  float p = (lane < n_leaf) ? exp_fast(e - mx) : 0.f;
  float p_self = include_self ? exp_fast(e_self - mx) : 0.f;
  float denom = warp_sum(p) + p_self;
  float inv = 1.f / denom;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = include_self ? (p_self * inv) * h3[j] : 0.f;
  // leaves in batches of 4 rows: 8 independent 16-byte loads per lane in flight before the first use
  for (int c0 = 0; c0 < n_leaf; c0 += 4) {
    float4 u[4], v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = min(c0 + k, n_leaf - 1);
      const float4* lr = reinterpret_cast<const float4*>(leaves + ((long long)i * n_leaf + c) * kD);
      u[k] = lr[lane];
      v[k] = lr[32 + lane];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = (c0 + k < n_leaf) ? __shfl_sync(0xffffffffu, p, (c0 + k) & 31) * inv : 0.f;
      acc[0] = fmaf(a, u[k].x, acc[0]); acc[1] = fmaf(a, u[k].y, acc[1]);
      acc[2] = fmaf(a, u[k].z, acc[2]); acc[3] = fmaf(a, u[k].w, acc[3]);
      acc[4] = fmaf(a, v[k].x, acc[4]); acc[5] = fmaf(a, v[k].y, acc[5]);
      acc[6] = fmaf(a, v[k].z, acc[6]); acc[7] = fmaf(a, v[k].w, acc[7]);
    }
  }
  gats_write_row(out, out.lin ? (long long)b * L.m_pad + i : row, lane, acc, h3, include_self, additional);
}

// Same layer, warp per (POINT, group of up to 16 consecutive frames of one object): the point's 8 leaf rows and leaf logits are
// read once into registers and reused for every frame of the group (the leaves are per-object constants; reference GATs.py:46
// reshapes the same tensor for every batch element).  Fast path for
// num_leaf == 8 (the released configuration, test_GATsSPG.yaml:5).
__global__ void __launch_bounds__(256, 2) gats_aggregate_frames8(const __half* x_hi, const __half* x_lo, Layout L,
                                                              const __grid_constant__ GatsGroups grp, int gi,
                                                              const float* __restrict__ wa3, int include_self, int additional, float alpha,
                                                              GatsOut out) {
  griddep_sync();
  const int lane = threadIdx.x & 31;
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_groups = grp.n;                         // frame groups: more warps in flight than points alone
  const int i = (int)(wid / n_groups), fg = (int)(wid % n_groups);
  const GatsGroup& G = grp.g[fg];
  if (i >= G.M) return;
  const int b_begin = G.b_begin, b_end = G.b_end;
  const float* __restrict__ leaves = G.leaves;
  const float* __restrict__ s2 = G.s2 + (long long)gi * G.M * 8;
  float4 lu[8], lv[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4* lr = reinterpret_cast<const float4*>(leaves + ((long long)i * 8 + c) * kD);
    lu[c] = lr[lane];
    lv[c] = lr[32 + lane];
  }
  const float s2l = lane < 8 ? s2[(long long)i * 8 + lane] : 0.f;
  float w3[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) w3[j] = wa3[(j >> 2) * 128 + lane * 4 + (j & 3)];
  auto lrelu = [alpha](float v) { return v > 0.f ? v : alpha * v; };
  // frames in batches of kGatsBatch: all their row loads are issued before the first is consumed (the kernel is bound by bytes
  // in flight: one frame at a time keeps ~2 KB per warp outstanding, far below what the HBM latency needs)
  constexpr int kGatsBatch = 4;
  for (int b0 = b_begin; b0 < b_end; b0 += kGatsBatch) {
    uint2 rh[kGatsBatch][2], rl[kGatsBatch][2];
#pragma unroll
    for (int k = 0; k < kGatsBatch; ++k) {
      const int b = min(b0 + k, b_end - 1);
      const long long row = (long long)b * L.R + L.n_pad + i;
      const uint2* ph = reinterpret_cast<const uint2*>(x_hi + row * kD);
      const uint2* pl = reinterpret_cast<const uint2*>(x_lo + row * kD);
      rh[k][0] = ph[lane]; rh[k][1] = ph[32 + lane];
      rl[k][0] = pl[lane]; rl[k][1] = pl[32 + lane];
    }
#pragma unroll
    for (int k = 0; k < kGatsBatch; ++k) {
      const int b = b0 + k;
      if (b >= b_end) break;
      const long long row = (long long)b * L.R + L.n_pad + i;
      float h3[8];
#pragma unroll
      for (int half_i = 0; half_i < 2; ++half_i) {
        const __half* hh = reinterpret_cast<const __half*>(&rh[k][half_i]);
        const __half* hl = reinterpret_cast<const __half*>(&rl[k][half_i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) h3[half_i * 4 + j] = join_f32(hh[j], hl[j]);
      }
      float s3 = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s3 = fmaf(h3[j], w3[j], s3);
      s3 = warp_sum(s3);
      float e = lane < 8 ? lrelu(s3 + s2l) : -INFINITY;
      const float e_self = include_self ? lrelu(2.f * s3) : -INFINITY;
      float mx = e;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));   // lanes 0..7 hold the leaf logits
      mx = fmaxf(__shfl_sync(0xffffffffu, mx, 0), e_self);
      const float p = lane < 8 ? exp_fast(e - mx) : 0.f;
      const float p_self = include_self ? exp_fast(e_self - mx) : 0.f;
      float ps = p;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
      const float inv = 1.f / (__shfl_sync(0xffffffffu, ps, 0) + p_self);
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = include_self ? (p_self * inv) * h3[j] : 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float a = __shfl_sync(0xffffffffu, p, c) * inv;
        acc[0] = fmaf(a, lu[c].x, acc[0]); acc[1] = fmaf(a, lu[c].y, acc[1]);
        acc[2] = fmaf(a, lu[c].z, acc[2]); acc[3] = fmaf(a, lu[c].w, acc[3]);
        acc[4] = fmaf(a, lv[c].x, acc[4]); acc[5] = fmaf(a, lv[c].y, acc[5]);
        acc[6] = fmaf(a, lv[c].z, acc[6]); acc[7] = fmaf(a, lv[c].w, acc[7]);
      }
      gats_write_row(out, out.lin ? (long long)b * L.m_pad + i : row, lane, acc, h3, include_self, additional);
    }
  }
}

// with_linear_transform, last step: x[3D row] = ELU(t[row] (+ x[3D row] if `additional` with include_self)) where t = pre . W
// (GATs.py:56-62, :64-70).  One thread = 8 channels of one row.  t: compact planes [B*m_pad, 256].
__global__ void gats_lin_finish(const __half* __restrict__ t_hi, const __half* __restrict__ t_lo, __half* __restrict__ x_hi,
                                __half* __restrict__ x_lo, Layout L, int add_h3) {
  griddep_sync();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over B*M*32
  if (idx >= (long long)L.B * L.M * 32) return;
  const int c8 = (int)(idx & 31);
  const long long pr = idx >> 5;
  const int b = (int)(pr / L.M), i = (int)(pr % L.M);
  if (i >= L.m_of(b)) return;                                              // pad rows of a smaller object stay zero
  const long long src = ((long long)b * L.m_pad + i) * kD + c8 * 8, dst = ((long long)b * L.R + L.n_pad + i) * kD + c8 * 8;
  const uint4 th = *reinterpret_cast<const uint4*>(t_hi + src), tlw = *reinterpret_cast<const uint4*>(t_lo + src);
  uint4 xh = *reinterpret_cast<const uint4*>(x_hi + dst), xl = *reinterpret_cast<const uint4*>(x_lo + dst);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float v = join_f32(reinterpret_cast<const __half*>(&th)[j], reinterpret_cast<const __half*>(&tlw)[j]);
    if (add_h3) v += join_f32(reinterpret_cast<const __half*>(&xh)[j], reinterpret_cast<const __half*>(&xl)[j]);
    v = v > 0.f ? v : exp_fast(v) - 1.f;
    __half h, l;
    split_f32(v, h, l);
    reinterpret_cast<__half*>(&xh)[j] = h;
    reinterpret_cast<__half*>(&xl)[j] = l;
  }
  *reinterpret_cast<uint4*>(x_hi + dst) = xh;
  *reinterpret_cast<uint4*>(x_lo + dst) = xl;
}

// ---------------------------------------------------------------------------------------
// Linear-attention state (reference GATs_SuperGlue.py:71-78), per segment s and head h:
//   Kmean[s][h][d]     = (1/m) sum_rows elu1(K[r,h,d])
//   KVmean[s][h][d][q] = (1/m) sum_rows elu1(K[r,h,d]) * V[r,h,q]
// Stage 1 (kv_state_tc.cu): one partial state per row group.  Stage 2, here: fixed-order sum over a segment's groups and the
// 1/m scale, written in the form the consumers want:
//   kmean [S][256]                     fp32, indexed by the segment itself (the q-projection epilogue picks the source segment)
//   bd    [S][256 (h*64+d)][256 (h*64+q)]  fp16-split planes, block-diagonal: bd[s] holds KVmean of the SOURCE segment of s
//         ('self': s, 'cross': the other side of the frame).  It is the B operand of the G-fold GEMM
//         G[s] = W0m . bd[s]^T  = the per-segment dynamic weight of mlp.0 (see api.cu); off-diagonal blocks stay zero.
// ---------------------------------------------------------------------------------------
constexpr int kKVPartial = kDh * kDh + kDh;  // 64x64 KV + 64 Ksum

// grid (S*H, 17), block 256
__global__ void kv_state_reduce(const float* __restrict__ partial, Layout L, KvGroups G, int cross,
                                float* __restrict__ kmean /*[S][256]*/, __half* __restrict__ bd_hi, __half* __restrict__ bd_lo) {
  griddep_sync();
  const int sh = blockIdx.x;
  const int seg = sh / kHeads, h = sh % kHeads;
  const int i = blockIdx.y * 256 + threadIdx.x;
  if (i >= kKVPartial) return;
  const bool is_kv = i < kDh * kDh;
  // KV blocks are written for the destination segment `seg` from its source; the K mean stays with its own segment
  const int from = is_kv ? L.src_seg(seg, cross) : seg;
  const int side = from & 1;
  const int group_rows = G.slabs * 256;
  const int g0 = (from >> 1) * (G.gq + G.gd) + (side ? G.gq : 0);
  const int valid = L.seg_valid(from);
  const int ng = (valid + group_rows - 1) / group_rows;
  float s = 0.f;
  for (int t = 0; t < ng; ++t) s += partial[((long long)(g0 + t) * kHeads + h) * kKVPartial + i];
  s = valid > 0 ? s * (1.f / (float)valid) : 0.f;            // empty segment (object prologue / query-only pass)
  if (is_kv) {
    const int d = i >> 6, q = i & 63;
    const long long o = ((long long)seg * kD + h * kDh + d) * kD + h * kDh + q;
    __half hh, ll;
    split_f32(s, hh, ll);
    bd_hi[o] = hh;
    bd_lo[o] = ll;
  } else {
    kmean[(long long)seg * kD + h * kDh + (i - kDh * kDh)] = s;
  }
}

// ---------------------------------------------------------------------------------------
// InstanceNorm1d(512) statistics over the valid rows of each segment
// (reference GATs_SuperGlue.py:126: no affine, biased variance, eps 1e-5).
// Stage 1: per 32-row quarter and channel: sum and sum of squared deviations from the quarter's mean (fp32) -- written by the
// mlp.0 GEMM epilogue (EPI_F32_STATS).
// Stage 2, here: per (segment, channel): fixed-order fp64 combine of the quarters -> mean, rstd.  The quarters' deviations
// are taken about a shift common to the whole segment, K = quarter 0's mean (law of total variance, the parallel form of
// Chan, Golub and LeVeque):  with u_t = s_t - n_t K,
//   M2 = sum_t M2_t + sum_t u_t^2 / n_t - (sum_t u_t)^2 / n,   mean = K + (sum_t u_t) / n
// -- plain sums, so the slices combine by addition and the loop has no division (n_t = 32 except in the last quarter).
// grid (S, 16), block (32 channels, kStatSlices slices): the slices keep enough independent loads in flight that the kernel is
// not a chain of dependent L2 round trips (8 slices: 17 us per launch at 224 quarters per segment)
// ---------------------------------------------------------------------------------------
constexpr int kStatSlices = 32;
__global__ void __launch_bounds__(32 * kStatSlices) in_stats_final(const float* __restrict__ part, Layout L, float* __restrict__ mu, float* __restrict__ rstd) {
  __shared__ double sh[kStatSlices][32][3];
  griddep_sync();
  const int seg = blockIdx.x;
  const int c = blockIdx.y * 32 + threadIdx.x;
  const int slice = threadIdx.y;
  const int q0 = L.seg_start(seg) / 32;
  const int valid = L.seg_valid(seg);
  const int nq = (valid + 31) / 32;
  const float2* p = reinterpret_cast<const float2*>(part) + (long long)q0 * 512 + c;
  const int n_last = valid - 32 * (nq - 1);                      // rows of the last quarter
  const double K = nq > 0 ? (double)p[0].x / (double)(nq > 1 ? 32 : n_last) : 0.0;
  const double inv_last = nq > 0 ? 1.0 / (double)n_last : 0.0;
  double u = 0.0, uu = 0.0, m2 = 0.0;
  for (int t = slice; t < nq; t += kStatSlices) {
    const float2 v = p[(long long)t * 512];
    const bool last = t == nq - 1;
    const double ut = fma(-(double)(last ? n_last : 32), K, (double)v.x);
    u += ut;
    uu = fma(ut * ut, last ? inv_last : 1.0 / 32.0, uu);
    m2 += (double)v.y;
  }
  sh[slice][threadIdx.x][0] = u;
  sh[slice][threadIdx.x][1] = uu;
  sh[slice][threadIdx.x][2] = m2;
  __syncthreads();
  if (slice == 0) {
    u = 0.0; uu = 0.0; m2 = 0.0;
#pragma unroll
    for (int k = 0; k < kStatSlices; ++k) { u += sh[k][threadIdx.x][0]; uu += sh[k][threadIdx.x][1]; m2 += sh[k][threadIdx.x][2]; }
    const double n = (double)(valid > 0 ? valid : 1);
    double var = (m2 + uu - u * u / n) / n;
    if (var < 0.0) var = 0.0;
    mu[seg * 512 + c] = (float)(K + u / n);
    rstd[seg * 512 + c] = (float)(1.0 / sqrt(var + 1e-5));
  }
}

// Range guard of the fp16-split operand format (|x| < 1023): an overflow anywhere in the GNN turns into inf/NaN and
// stays in the residual stream, so scanning the final X hi-plane once per chunk detects it (pad rows are zero by construction).
// Sets *flag = 1; mutual_match then reports "no match" for every point of the call instead of garbage.
__global__ void range_check(const __half* __restrict__ x_hi, long long n_vec /* elements / 8 */, int* __restrict__ flag) {
  griddep_sync();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vec) return;
  const uint4 u = reinterpret_cast<const uint4*>(x_hi)[i];
  const unsigned w[4] = {u.x, u.y, u.z, u.w};
  bool bad = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) bad |= ((w[k] & 0x7C00u) == 0x7C00u) || ((w[k] & 0x7C000000u) == 0x7C000000u);   // exponent all ones: inf / NaN
  if (bad) atomicOr(flag, 1);
}

// fp32 -> planes (debug / tests)
__global__ void split_planes(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) split_f32(x[i], hi[i], lo[i]);
}
// planes -> fp32: (hi + lo) / 64; lo = nullptr reads a single fp16 plane (the k,v projection's output) as hi / 64
__global__ void join_planes(const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = lo ? join_f32(hi[i], lo[i]) : __half2float(hi[i]) * kPreInv;
}

// ---------------------------------------------------------------------------------------
// Dual-softmax tail (reference GATs_SuperGlue.py:217-230).  With unit-norm operands and the fixed shift
//   e[n,m] = exp((cos[n,m] - 1) / scale)   in (exp(-2/scale), 1]
// softmax(scores,1)*softmax(scores,2) = e^2 / (colsum[m] * rowsum[n]); the two passes of the score GEMM (EPI_SCORE_SUMS,
// EPI_SCORE_CONF in gemm_tc.cu) never materialise the cos matrix.  Between them: fixed-order sums of the per-tile partials ->
// 1/rowsum, 1/colsum, and the arg-max accumulators of pass 2 are cleared.
// grid (ceil((n_pad + m_pad)/256), B), block 256
// ---------------------------------------------------------------------------------------
__global__ void score_sums_finalize(const float* __restrict__ rowsum_part, const float* __restrict__ colsum_part, Layout L, int n_parts,
                                    int q_groups, float* __restrict__ inv_rowsum, float* __restrict__ inv_colsum,
                                    unsigned long long* __restrict__ rowbest, unsigned long long* __restrict__ colbest) {
  griddep_sync();
  const int b = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int Nb = L.n_of(b);
  if (i < L.n_pad) {
    float s = 0.f;
    for (int t = 0; t < n_parts; ++t) s += rowsum_part[((long long)b * n_parts + t) * L.n_pad + i];
    inv_rowsum[b * L.n_pad + i] = i < Nb ? 1.f / s : 0.f;
    if (i < L.N) rowbest[(long long)b * L.N + i] = 0ull;
  } else if (i - L.n_pad < L.m_pad) {
    const int m = i - L.n_pad;
    const int Mb = L.m_of(b);
    const int qv = (Nb + 31) / 32;                      // quarters that hold valid query rows
    float s = 0.f;
    if (m < Mb)
      for (int t = 0; t < qv && t < q_groups; ++t) s += colsum_part[((long long)b * q_groups + t) * L.m_pad + m];
    inv_colsum[b * L.m_pad + m] = (m < Mb && qv > 0) ? 1.f / s : 0.f;
    if (m < Mb) colbest[(long long)b * L.M + m] = 0ull;
  }
}

// Mutual nearest neighbour + threshold (reference GATs_SuperGlue.py:220-230).  rowbest / colbest hold packed
// (conf bits << 32 | ~index): order-preserving for conf >= 0 with lowest-index-wins ties (torch.max returns the first maximum).
// A frame with no valid query rows (ragged batch) or a raised range flag yields -1 / 0 everywhere.  m1 / sc1 rows are
// m_out >= L.M wide; columns past the frame's own M_b are -1 / 0.
// One block per frame is plenty (N+M <= ~20k); grid (B), block 256.
__global__ void mutual_match(const unsigned long long* __restrict__ rowbest, const unsigned long long* __restrict__ colbest, Layout L,
                             float thr, const int* __restrict__ range_flag, int m_out, long long* __restrict__ m0, long long* __restrict__ m1,
                             float* __restrict__ sc0, float* __restrict__ sc1) {
  griddep_sync();
  const int b = blockIdx.x;
  const int N = L.N, M = L.m_of(b), Nb = L.n_of(b);
  const bool poisoned = *range_flag != 0 || Nb == 0;
  const unsigned long long* rb = rowbest + (long long)b * N;
  const unsigned long long* cb = colbest + (long long)b * L.M;
  auto idx_of = [](unsigned long long p) { return (int)(0xFFFFFFFFu - (unsigned)(p & 0xFFFFFFFFull)); };
  auto val_of = [](unsigned long long p) { return __uint_as_float((unsigned)(p >> 32)); };
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    long long mm = -1ll;
    float ms = 0.f;
    if (!poisoned && n < Nb) {
      const int i0 = idx_of(rb[n]);                       // -1: the row never saw a positive confidence (cannot happen for finite inputs)
      const bool mutual = i0 >= 0 && idx_of(cb[i0]) == n;
      ms = mutual ? val_of(rb[n]) : 0.f;
      if (mutual && ms > thr) mm = i0;
    }
    m0[(long long)b * N + n] = mm;
    sc0[(long long)b * N + n] = ms;
  }
  for (int m = threadIdx.x; m < m_out; m += blockDim.x) {
    long long mm = -1ll;
    float ms1 = 0.f;
    if (!poisoned && m < M) {
      const int i1 = idx_of(cb[m]);
      const int i0 = i1 >= 0 ? idx_of(rb[i1]) : -1;
      const bool mutual1 = i0 == m;
      // mscores0[i1], valid0[i1] recomputed (cheap) instead of read-after-write across threads
      const bool mutual0_i1 = i0 >= 0 && idx_of(cb[i0]) == i1;
      const float ms0_i1 = mutual0_i1 ? val_of(rb[i1]) : 0.f;
      const bool valid0_i1 = mutual0_i1 && ms0_i1 > thr;
      ms1 = mutual1 ? ms0_i1 : 0.f;
      if (mutual1 && valid0_i1) mm = i1;
    }
    m1[(long long)b * m_out + m] = mm;
    sc1[(long long)b * m_out + m] = ms1;
  }
}

// conf rows of a poisoned call / of frames without valid queries are not touched here: pass 2 writes every element of conf.
// ... up to the chunk's m_pad: when the conf rows are wider (a call whose largest object is in another chunk), this kernel
// zeroes columns [c0, ld) of every row.  Grid-stride, block 256
__global__ void conf_fill_tail(float* __restrict__ conf, long long rows, int ld, int c0) {
  griddep_sync();
  const int w = ld - c0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * w; i += (long long)gridDim.x * blockDim.x)
    conf[(i / w) * ld + c0 + i % w] = 0.f;
}

// ---------------------------------------------------------------------------------------
// Adjacent producers (offline feature files of an object, reference src/sfm/postprocess/feature_process.py:297-317 and
// src/utils/data_utils.py:143-205).
// ---------------------------------------------------------------------------------------
// Exclusive prefix sum of the track lengths: one block, each thread scans a contiguous chunk, then a block scan of the chunk sums.
__global__ void __launch_bounds__(1024) exclusive_scan_i64(const long long* __restrict__ in, long long* __restrict__ out, int n) {
  __shared__ long long sh[32];
  const int t = threadIdx.x;
  const int per = (n + 1023) / 1024;
  const int lo = min(t * per, n), hi = min(lo + per, n);
  long long acc = 0, total;
  for (int i = lo; i < hi; ++i) acc += in[i];
  long long run = block_scan(acc, SumS64(), 0ll, sh, &total);
  for (int i = lo; i < hi; ++i) { out[i] = run; run += in[i]; }
}

// numpy's pairwise sum of a contiguous run (numpy/core/src/umath/loops_utils.h: < 8 elements sequential; up to 128: eight
// interleaved accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) then the remainder; above: halves rounded down to
// a multiple of 8, recursively).  Restated here so that the GPU result is bit-identical.
__device__ inline double np_pairwise_sum(const double* a, long long n) {
  if (n < 8) {
    double res = 0.0;
    for (long long i = 0; i < n; ++i) res += a[i];
    return res;
  }
  if (n <= 128) {
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    long long i;
    for (i = 8; i < n - (n % 8); i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    }
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
  }
  long long n2 = n / 2;
  n2 -= n2 % 8;
  return np_pairwise_sum(a, n2) + np_pairwise_sum(a + n2, n - n2);
}

// mean_descriptors / mean_scores (feature_process.py:297-317): np.mean(x[start:end], axis=0) of each track's [len, D] fp64
// block, in numpy's summation order, which follows the caller's layout (numpy's reduction loop runs along the axis with the
// smaller stride):
//   channel_major == 0: x is [sum(len), D] row-major; numpy adds the rows in order, one running sum per channel;
//   channel_major != 0: x is [D, sum(len)], each channel's track contiguous; numpy sums it pairwise (D = 1 is this case).
// Both sums start from numpy's identity +0.0 (an all -0.0 track gives +0.0), then one division.  Thread per (track, channel).
__global__ void segmented_mean_f64(const double* __restrict__ x, const long long* __restrict__ seg_len, const long long* __restrict__ offsets,
                                   int M, int D, int channel_major, double* __restrict__ out) {
  const long long n_rows = offsets[M - 1] + seg_len[M - 1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)M * D; i += (long long)gridDim.x * blockDim.x) {
    const long long seg = i / D;
    const int c = (int)(i % D);
    const long long start = offsets[seg], len = seg_len[seg];
    double acc = 0.0;
    if (channel_major) {
      acc += np_pairwise_sum(x + c * n_rows + start, len);
    } else {
      for (long long r = 0; r < len; ++r) acc += x[(start + r) * D + c];
    }
    out[i] = acc / (double)len;
  }
}

// build_features3d_leaves / pad_features3d_random (data_utils.py:143-205): column gather from the channel-first descriptor
// matrix [dim, n_src] extended by the all-ones dustbin column (index n_src), then truncation / all-ones padding to n_out
// columns; scores likewise with a zero dustbin / zero padding.  `idx` [n_idx] int64 holds, per output column, the source column
// (values in [0, n_src]); output columns >= n_idx are padding.  idx == nullptr: identity (pad_features3d_random).
// grid (ceil(n_out/256), dim), block 256: coalesced along the column axis.
__global__ void gather_columns_f32(const float* __restrict__ src, int dim, long long n_src, const long long* __restrict__ idx, long long n_idx,
                                   float* __restrict__ dst, long long n_out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (j >= n_out || c >= dim) return;
  float v = 1.f;                                           // padding / dustbin descriptor = all ones
  if (j < n_idx) {
    const long long s = idx ? idx[j] : j;
    if (s >= 0 && s < n_src) v = src[(long long)c * n_src + s];
  }
  dst[(long long)c * n_out + j] = v;
}
__global__ void gather_scores_f32(const float* __restrict__ src, long long n_src, const long long* __restrict__ idx, long long n_idx,
                                  float* __restrict__ dst, long long n_out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  float v = 0.f;                                           // padding / dustbin score = 0
  if (j < n_idx) {
    const long long s = idx ? idx[j] : j;
    if (s >= 0 && s < n_src) v = src[s];
  }
  dst[j] = v;
}

}  // namespace opb
