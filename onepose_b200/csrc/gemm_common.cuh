// GEMM problem description shared by the wgmma core (product) and the SIMT fp32 core (cross-check of the
// tensor-core arithmetic; reachable through opb_debug_gemm only).  Both consume the SAME fp16-split operands, so
// the SIMT result is an fp32 reference for the tensor-core result on identical inputs.
#pragma once
#include "common.cuh"

namespace opb {

// C[batch][rows, n_out] = A[rows, K1+K2] . B[n_out, K1+K2]^T  (+ bias[n_out])
//   reduction columns [0,K1)      : a1[:, 0:K1]  with b1[n, 0:K1]
//   reduction columns [K1,K1+K2)  : a2[:, 0:K2]  with b2[(seg*n_out + n), 0:K2]   (b2_per_seg)
//                                                 or b2[n, 0:K2]
// where seg = L.seg_of_row(row) -- per-frame/side dynamic weights (the G fold).
// Batched form: batch z uses A rows offset z*a_batch_rows, B rows offset z*b_batch_rows, output rows offset z*rows
// (score GEMM: B operand = activations of the same frame; G fold: A = shared weight (a_batch_rows = 0), B = per-segment state).
// Epilogue of the wgmma core (what happens to the accumulator tile before it leaves the SM):
enum GemmEpilogue {
  EPI_F32 = 0,        // c[rows, ldc] fp32 = acc (+bias)
  EPI_F32_STATS = 1,  // EPI_F32 + InstanceNorm partials (sum, sum of squared deviations from the mean, per 32-row quarter and column) -> statpart
  EPI_QSCALE = 2,     // Q' = elu1(acc+bias) / (elu1(.) . Kmean_src + 1e-6/m_src) per head -> out planes   (n_out = 256)
  EPI_L2NORM = 5,     // F.normalize(acc + bias) over the 256 columns -> out planes                          (n_out = 256)
  // dual-softmax tail on the batched score GEMM (one batch = one frame; rows = queries, columns = 3D points):
  EPI_SCORE_SUMS = 6, // e = exp((cos-1)/scale): per-half-tile row sums and per-32-row column sums -> rowsum_part / colsum_part
  EPI_SCORE_CONF = 7, // conf = e^2 / (rowsum*colsum) -> conf [B,N,M] (optional) + packed row / column arg-max (atomicMax)
  EPI_QKV = 9,        // k,v projection (n_out = 512): out.hi[rows, 512] = fp16(64 * [elu1(K) | V]), pad rows zero -- the
                      // single-pass operands of kv_state_h
  EPI_BIAS_PLANES = 10,  // out planes = acc + bias (bias may be null), rows past the segment's valid count written as zero.
                      // The residual GEMM of a layer uses it with the residual INSIDE the reduction:
                      // x_new = [hn | x] . [W1 | I]^T + b  (K2 = 256 identity block; x_hi*64 + x_lo*64 is exact in the fp32
                      // accumulator), so the epilogue has no global loads -- every chunk of an epilogue ends in a proxy fence that
                      // waits for the thread's outstanding loads, which made a load-x-in-the-epilogue form latency-bound
  EPI_CONV = 11,      // 3x3 / 1x1 convolution over a zero-bordered pixel grid (superpoint.cu): out planes = [ReLU](acc + bias) on the
                      // interior pixels, zero on the border / padding rows (so the output is again a valid zero-bordered grid)
};

struct GemmProblem {
  CPlanes a1, a2, b1, b2;
  int K1, K2;
  int b2_per_seg;
  int b2_lo_zero;        // the lo plane of b2 is identically zero (identity K-block): its A_hi.B_lo pass is skipped (bit-identical)
  int a_hi_only;         // use only the hi plane of A (A_lo neither loaded nor multiplied): for a product whose OUTPUT is rounded to one
                         // fp16 plane anyway (k,v projection: the dropped term is below the output rounding, zero-mean per row, and the
                         // consumer averages over the segment's rows)
  int rows, n_out;       // per batch; rows % 256 == 0 (segments are 256-row aligned), n_out % bn == 0
  int bn;                // column-tile width of the wgmma core, 0 = 256: EPI_CONV 64 / 128, EPI_F32 128 / 256, any other epilogue 256
  // Implicit-GEMM convolution over a row-major pixel grid (A = activations [pixels, C_in], one row per pixel of a grid with a zero
  // border): reduction block `tap` (= kb / kb_per_tap) reads the A rows shifted by tap_off[tap] pixels and the B columns
  // [tap*C_in, (tap+1)*C_in) -- the 9 taps of a 3x3 kernel are 9 row-shifted TMA loads of the same matrix, never an im2col buffer.
  int taps;              // 0: plain GEMM
  int kb_per_tap;        // C_in / 64
  int tap_off[9];
  // EPI_CONV: pixel-grid geometry (row r is pixel q = r % cv_ppad of its image; y = q / cv_w2, x = q % cv_w2; interior:
  // 1 <= y <= cv_h, 1 <= x <= cv_w) and the activation
  int cv_w2, cv_h, cv_w, cv_ppad, relu;
  int* range_flag;       // EPI_CONV: set to 1 when an output leaves the split operand range (split_out_of_range), or nullptr
  int batch;
  long long a_batch_rows, b_batch_rows, c_batch_elems;
  Layout L;
  const float* bias;     // [n_out] or nullptr
  float* c;              // fp32 [rows, ldc]
  int ldc;
  // ---- wgmma core only ----
  int epi;               // GemmEpilogue
  Planes out;            // planes output [rows, out.ld] (EPI_QSCALE / EPI_L2NORM / EPI_BIAS_PLANES; EPI_QKV: out.hi only)
  const float* kmean;    // EPI_QSCALE: [S][256]
  int cross;             // EPI_QSCALE: source segment selection
  float* statpart;       // EPI_F32_STATS: [rows/32][n_out][2]
  // A-operand conversion inside the wgmma core (gemm_tc.cu ACV_NORM_RELU): A1 = ReLU((a_raw - mu_seg) * rstd_seg)  (K1 columns);
  // a_raw is fp32 [rows, a_raw_ld]
  int a_conv;
  const float* a_raw;
  int a_raw_ld;
  const float* mu;                  // [S][512]
  const float* rstd;
  // EPI_SCORE_*: L gives N, M, n_pad, m_pad
  float inv_scale;
  float* rowsum_part;               // [B][2*n_out/256][n_pad]
  float* colsum_part;               // [B][rows/32][m_pad]
  const float* inv_rowsum;          // [B][n_pad]
  const float* inv_colsum;          // [B][m_pad]
  float* conf;                      // [B][N][conf_ld] or nullptr; columns past frame b's L.m_of(b) are written as 0
  int conf_ld;                      // columns of a conf row, >= L.M (0: L.M)
  unsigned long long* rowbest;      // [B][N]
  unsigned long long* colbest;      // [B][M]
  int max_ctas;                     // test hook (opb_debug_gemm): grid = min(units, SMs, max_ctas); 0 = min(units, SMs)
};

int launch_gemm_simt(const GemmProblem& p, cudaStream_t stream);

}  // namespace opb
