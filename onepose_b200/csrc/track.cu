// The reference tracker's flow-only state machine on the GPU, one thread per track in fp64: what BATracker runs around
// flow_track in the live demo's order (inference_demo.py:253-299, track_interval = 5) with track(..., flow_track_only=True).
//   update_kf            ba_tracker.py:128-145   the 10 cm / 10 deg gate against the last reported pose      opb_track_gate
//   add_kf               :147-235                pose_pred onto the history at a track's first frame         opb_track_gate
//   track                :727-802                the flow / motion / pose_pred choice, the init override     opb_track_select
//   motion_prediction    :275-293                constant-velocity extrapolation of the last three poses     opb_track_select
//   cm_degree_5_metric   :105-111                translation (cm) and rotation (deg) distance of two poses
//
// The distances and cy of mat2euler are pnp.pose_errors' arithmetic -- index order, every operation rounded on its own
// (__dadd_rn and friends, so that nothing is contracted into a fused multiply-add) -- so that a threshold decision on equal
// inputs comes out as the model's (tests/track_reference.py).  The motion pose's translation is exact in the same way; its
// rotation goes through CUDA's atan2 / sin / cos, which are not glibc's, and matches the model to a tolerance (DESIGN §5.10).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kTrackInterval = 5;          // inference_demo.py:144
constexpr double kUpdateCm = 10.0, kUpdateDeg = 10.0;   // update_kf (:133)
constexpr double kMotionCm = 10.0, kMotionDeg = 10.0, kMotionPx = 10.0;   // track (:742)
constexpr int kMotionCount = 3;            // use_motion_cnt < 3 (:742)
constexpr double kFlowCm = 20.0, kFlowDeg = 20.0;        // track (:745)
constexpr int kHistory = 3;                // motion_prediction reads pose_list[-3:]
constexpr int kThreads = 128;
constexpr double kRad2Deg = 57.29577951308232;           // 180 / pi, as numpy's and torch's rad2deg
constexpr double kEps4 = 4.0 * 2.220446049250313e-16;    // transforms3d's _EPS4: 4 * eps(f64)

// cm_degree_5_metric(a, b) = pnp.pose_errors: |t_a - t_b| * 100 and the angle of R_a R_b^T from its clamped trace.
__device__ void cm_degree(const double* a, const double* b, double& cm, double& deg) {
  double s = 0.0;
  for (int r = 0; r < 3; ++r) {
    const double d = __dsub_rn(a[4 * r + 3], b[4 * r + 3]);
    s = r ? __dadd_rn(s, __dmul_rn(d, d)) : __dmul_rn(d, d);
  }
  cm = __dmul_rn(sqrt(s), 100.0);
  double tr = 0.0;
  for (int r = 0; r < 3; ++r) {
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(a[4 * r], b[4 * r]), __dmul_rn(a[4 * r + 1], b[4 * r + 1])), __dmul_rn(a[4 * r + 2], b[4 * r + 2]));
    tr = r ? __dadd_rn(tr, d) : d;
  }
  tr = tr <= 3.0 ? tr : 3.0;                 // a NaN trace becomes 3, as `trace if trace <= 3 else 3`
  deg = __dmul_rn(acos(__ddiv_rn(__dsub_rn(tr, 1.0), 2.0)), kRad2Deg);
}

// transforms3d.euler.mat2euler(M, 'sxyz') of the rotation block of a row-major 4x4.
__device__ void mat2euler(const double* M, double e[3]) {
  const double cy = sqrt(__dadd_rn(__dmul_rn(M[0], M[0]), __dmul_rn(M[4], M[4])));
  if (cy > kEps4) {
    e[0] = atan2(M[9], M[10]);
    e[1] = atan2(-M[8], cy);
    e[2] = atan2(M[4], M[0]);
  } else {
    e[0] = atan2(-M[6], M[5]);
    e[1] = atan2(-M[8], cy);
    e[2] = 0.0;
  }
}

// transforms3d.euler.euler2mat(ai, aj, ak, 'sxyz') into the rotation block of a row-major 4x4.
__device__ void euler2mat(const double a[3], double* M) {
  double si, ci, sj, cj, sk, ck;
  sincos(a[0], &si, &ci);
  sincos(a[1], &sj, &cj);
  sincos(a[2], &sk, &ck);
  const double cc = __dmul_rn(ci, ck), cs = __dmul_rn(ci, sk), sc = __dmul_rn(si, ck), ss = __dmul_rn(si, sk);
  M[0] = __dmul_rn(cj, ck);
  M[1] = __dsub_rn(__dmul_rn(sj, sc), cs);
  M[2] = __dadd_rn(__dmul_rn(sj, cc), ss);
  M[4] = __dmul_rn(cj, sk);
  M[5] = __dadd_rn(__dmul_rn(sj, ss), cc);
  M[6] = __dsub_rn(__dmul_rn(sj, cs), sc);
  M[8] = -sj;
  M[9] = __dmul_rn(cj, si);
  M[10] = __dmul_rn(cj, ci);
}

// motion_prediction() from the history h0, h1, ht (oldest first), with the reference's slip: rot_t is mat2euler of h1.
__device__ void motion_prediction(const double* h0, const double* h1, const double* ht, double* out) {
  double r0[3], r1[3], a[3];
  mat2euler(h0, r0);
  mat2euler(h1, r1);
  for (int i = 0; i < 3; ++i) {
    const double speed = __ddiv_rn(__dadd_rn(__dsub_rn(r1[i], r0[i]), __dsub_rn(r1[i], r1[i])), 2.0);
    a[i] = __dadd_rn(r1[i], speed);
  }
  euler2mat(a, out);
  for (int r = 0; r < 3; ++r) {
    const double speed = __ddiv_rn(__dadd_rn(__dsub_rn(h1[4 * r + 3], h0[4 * r + 3]), __dsub_rn(ht[4 * r + 3], h1[4 * r + 3])), 2.0);
    out[4 * r + 3] = __dadd_rn(ht[4 * r + 3], speed);
  }
  out[12] = out[13] = out[14] = 0.0;
  out[15] = 1.0;
}

__device__ __forceinline__ void copy16(double* dst, const double* src) {
  for (int i = 0; i < 16; ++i) dst[i] = src[i];
}

// A track is at its first frame (the demo's id == 0) when its counter is 0 -- a fresh or reset track -- or its history is empty.
__device__ __forceinline__ bool first_frame(int64_t frame, int len) { return frame <= 0 || len <= 0; }

// pose_list.append(p) on the history: oldest first, the oldest dropped past kHistory.
__device__ void push(double* h, int32_t& len, const double* p) {
  int n = min(max(len, 0), kHistory);
  if (n == kHistory) {
    for (int k = 0; k + 1 < kHistory; ++k) copy16(h + 16 * k, h + 16 * (k + 1));
    n = kHistory - 1;
  }
  copy16(h + 16 * n, p);
  len = n + 1;
}

__global__ void __launch_bounds__(kThreads) gate_kernel(const double* __restrict__ pose_pred, int B, const int64_t* __restrict__ frame,
                                                       double* __restrict__ hist, int32_t* __restrict__ hist_len, int32_t* __restrict__ gate) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* pp = pose_pred + 16 * (size_t)b;
  double* h = hist + 48 * (size_t)b;
  int32_t len = hist_len[b];
  const int64_t f = frame[b];
  if (first_frame(f, len)) {             // update_kf accepts (no keyframe yet), then add_kf pushes pose_pred
    len = 0;
    push(h, len, pp);
    hist_len[b] = len;
    gate[b] = OPB_TRACK_GATE_ADD;
  } else if (f % kTrackInterval == 0) {
    double cm, deg;
    cm_degree(pp, h + 16 * (min(len, kHistory) - 1), cm, deg);
    gate[b] = (cm > kUpdateCm || deg > kUpdateDeg) ? OPB_TRACK_GATE_REJECT : OPB_TRACK_GATE_ACCEPT;
  } else {
    gate[b] = OPB_TRACK_GATE_NONE;
  }
}

__global__ void __launch_bounds__(kThreads) select_kernel(const double* __restrict__ pose_pred, const double* __restrict__ pose_flow,
                                                         const double* __restrict__ kpt_dist, int B, int64_t* __restrict__ frame,
                                                         double* __restrict__ hist, int32_t* __restrict__ hist_len, int32_t* __restrict__ init_cnt,
                                                         int32_t* __restrict__ use_motion_cnt, double* __restrict__ pose_out,
                                                         int32_t* __restrict__ branch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* pp = pose_pred + 16 * (size_t)b;
  double* out = pose_out + 16 * (size_t)b;
  double* h = hist + 48 * (size_t)b;
  int32_t len = min(hist_len[b], kHistory);
  const int64_t f = frame[b];
  frame[b] = f + 1;
  if (first_frame(f, len)) {            // the demo reports pose_pred and does not call track()
    copy16(out, pp);
    branch[b] = OPB_TRACK_KEYFRAME;
    return;
  }
  const double* pf = pose_flow + 16 * (size_t)b;
  double cm, deg;
  cm_degree(h + 16 * (len - 1), pf, cm, deg);
  const double kd = kpt_dist[b];
  int32_t umc = use_motion_cnt[b];
  bool flow;
  if (((cm > kMotionCm || deg > kMotionDeg) && umc < kMotionCount) || kd > kMotionPx) {
    flow = false;
  } else {
    flow = cm < kFlowCm && deg < kFlowDeg;
  }
  int32_t code;
  if (flow) {
    umc = 0;
    copy16(out, pf);
    code = OPB_TRACK_FLOW;
  } else {
    umc += 1;
    if (len < kHistory) {
      copy16(out, pp);
      code = OPB_TRACK_PRED;
    } else {
      motion_prediction(h, h + 16, h + 32, out);
      code = OPB_TRACK_MOTION;
    }
  }
  use_motion_cnt[b] = umc;
  const int32_t ic = init_cnt[b];
  if (ic > 0) {                          // the first frames report the matcher pose ('pose_gt' = pose_pred in the demo)
    init_cnt[b] = ic - 1;
    copy16(out, pp);
    code = OPB_TRACK_INIT;
  }
  push(h, len, out);
  hist_len[b] = len;
  branch[b] = code;
}

}  // namespace
}  // namespace opb

extern "C" int opb_track_gate(const double* pose_pred, int32_t B, const int64_t* frame, double* hist, int32_t* hist_len, int32_t* gate, void* stream) {
  REQUIRE(__func__, pose_pred && frame && hist && hist_len && gate && B > 0);
  LAUNCH_NH(__func__, opb::gate_kernel, (unsigned)((B + opb::kThreads - 1) / opb::kThreads), opb::kThreads, 0, (cudaStream_t)stream, pose_pred, B,
            frame, hist, hist_len, gate);
  return OPB_OK;
}

extern "C" int opb_track_select(const double* pose_pred, const double* pose_flow, const double* kpt_dist, int32_t B, int64_t* frame, double* hist,
                                int32_t* hist_len, int32_t* init_cnt, int32_t* use_motion_cnt, double* pose_out, int32_t* branch, void* stream) {
  REQUIRE(__func__, pose_pred && pose_flow && kpt_dist && frame && hist && hist_len && init_cnt && use_motion_cnt && pose_out && branch && B > 0);
  LAUNCH_NH(__func__, opb::select_kernel, (unsigned)((B + opb::kThreads - 1) / opb::kThreads), opb::kThreads, 0, (cudaStream_t)stream, pose_pred,
            pose_flow, kpt_dist, B, frame, hist, hist_len, init_cnt, use_motion_cnt, pose_out, branch);
  return OPB_OK;
}
