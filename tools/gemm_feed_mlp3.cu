// Launcher of the mlp.3-shaped wgmma GEMM for tools/gemm_feed.py: the converter variant (ACV_NORM_RELU) with the identity
// K-block, on caller-supplied buffers and with any K1.  Host code only; gemm_feed.py compiles it into a temporary directory
// and links it against the library build it measures (opb::launch_gemm_tc is an exported C++ symbol of that build).
//   x <- [ReLU((hid - mu_seg) * rstd_seg) | x] . [W1 | I]^T + b     hid fp32 [rows, K1], W1 planes [256, K1], x / I planes ld 256
// Layout: `frames` frames of n_pad + m_pad rows, every row valid.  mu / rstd are indexed [seg * 512 + column] as in the
// matcher, so for K1 > 512 they need (segments + K1 / 512) * 512 entries.
#include "gemm_tc.cuh"

extern "C" int feed_mlp3(const float* hid, int K1, const void* w1_hi, const void* w1_lo, const void* x_hi, const void* x_lo, void* out_hi,
                         void* out_lo, const void* eye_hi, const void* eye_lo, const float* bias, const float* mu, const float* rstd,
                         int frames, int n_pad, int m_pad, int identity_diag, void* stream) {
  using namespace opb;
  GemmProblem p{};
  p.L.B = frames; p.L.N = n_pad; p.L.M = m_pad; p.L.n_pad = n_pad; p.L.m_pad = m_pad; p.L.R = n_pad + m_pad;
  p.batch = 1; p.rows = p.L.rows();
  p.K1 = K1; p.b1 = CPlanes{(const __half*)w1_hi, (const __half*)w1_lo, K1}; p.n_out = kD; p.bias = bias;
  p.epi = EPI_BIAS_PLANES; p.out = Planes{(__half*)out_hi, (__half*)out_lo, kD};
  p.a2 = CPlanes{(const __half*)x_hi, (const __half*)x_lo, kD}; p.K2 = kD;
  p.b2 = CPlanes{(const __half*)eye_hi, (const __half*)eye_lo, kD}; p.b2_lo_zero = 1; p.b2_identity = identity_diag;
  p.a_conv = 1; p.a_raw = hid; p.a_raw_ld = K1; p.mu = mu; p.rstd = rstd;
  return launch_gemm_tc(p, (cudaStream_t)stream);
}
