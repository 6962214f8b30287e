// Pose-guided crop on the GPU: the step between one frame's pose and the next frame's extractor input in the reference's live
// loop (inference_demo.py:193-247).  Replaces, for B frames and without leaving the device,
//   previous_pose_detect   local_feature_2D_detector.py:232-259   reproj -> min / max -> astype(int32)        opb_boxes_from_poses
//   crop_img_by_bbox       :160-186   get_K_crop_resize x 2, get_image_crop_resize x 2, then / 255           opb_crop_resize
//                          the same where crop b reads frame frame_index[b] (several boxes per frame)   opb_crop_resize_indexed
//   parse_scanned_data.py   :151-159   the same two warps on colour frames, kept in uint8                    opb_crop_resize_colour
//   get_image_crop_resize / get_K_crop_resize   data_utils.py:233-272   one cv2.warpAffine, T @ K             opb_warp_crop_u8
//
// The pixels are OpenCV's, bit for bit.  cv2.warpAffine(INTER_LINEAR) on 8-bit data with a constant border is integer
// arithmetic once the 2x3 matrix is inverted (DESIGN, "The crop"), and get_affine_transform's matrix is three float32 point
// pairs through cv2.getAffineTransform's fp64 LU solve; both are restated here operation by operation with __dmul_rn /
// __dadd_rn / __ddiv_rn so that nothing is contracted into a fused multiply-add.  The model is tests/crop_reference.py.
//
// Two launches per call, both on the caller's stream: one thread per frame builds the transforms (and K_crop, status), then
// one thread per output pixel warps.  crop_img_by_bbox's two chained warps are evaluated per output pixel: a stage-2 pixel
// reads 4 stage-1 pixels, each of which is warp_pixel() on the frame rounded to uint8 -- 16 reads of the frame, no
// intermediate image (stage 1 has the box's size, which differs per frame and can exceed the frame).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kMaxCoord = 1 << 20;   // |box coordinate| bound: beyond it cv2's 22.10 fixed-point coordinates overflow int32
constexpr int kMaxSide = 32767;      // box / image side bound: cv2 addresses pixels by int16
constexpr int kWarpThreads = 256;

// fp64 / fp32 operations that stay separate roundings
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

__device__ __forceinline__ bool box_ok(const int32_t* box) {
  const int64_t w = (int64_t)box[2] - box[0], h = (int64_t)box[3] - box[1];
  bool ok = w > 0 && w <= kMaxSide && h > 0 && h <= kMaxSide;
  for (int i = 0; i < 4; ++i) ok = ok && box[i] >= -kMaxCoord && box[i] <= kMaxCoord;
  return ok;
}

// OpenCV's LUImpl (core/src/matrix_decomp.cpp) for a 6x6 system with one right-hand side: the pivot is the first entry of
// largest magnitude, d = -1 / pivot, row_j += (a_ji * d) * row_i, then back substitution.  b becomes the solution.
__device__ bool lu_solve6(double (*a)[6], double* b) {
  for (int i = 0; i < 6; ++i) {
    int k = i;
    for (int j = i + 1; j < 6; ++j)
      if (fabs(a[j][i]) > fabs(a[k][i])) k = j;
    if (fabs(a[k][i]) < 2.220446049250313e-16 * 100) return false;
    if (k != i) {
      for (int j = i; j < 6; ++j) { const double t = a[i][j]; a[i][j] = a[k][j]; a[k][j] = t; }
      const double t = b[i]; b[i] = b[k]; b[k] = t;
    }
    const double d = __ddiv_rn(-1.0, a[i][i]);
    for (int j = i + 1; j < 6; ++j) {
      const double alpha = mul(a[j][i], d);
      for (int c = i + 1; c < 6; ++c) a[j][c] = add(a[j][c], mul(alpha, a[i][c]));
      b[j] = add(b[j], mul(alpha, b[i]));
    }
  }
  for (int i = 5; i >= 0; --i) {
    double s = b[i];
    for (int c = i + 1; c < 6; ++c) s = sub(s, mul(a[i][c], b[c]));
    b[i] = __ddiv_rn(s, a[i][i]);
  }
  return true;
}

// get_affine_transform(center, [src_w, .], rot = 0, [dst_w, dst_h]) (data_utils.py:24-57) -> T[6], row-major 2x3.  The three
// point pairs are float32 as there: the centre, the point src_w / 2 (dst_w / 2) above it, and get_3rd_point of the two.  Only
// the width enters: both axes scale by dst_w / src_w.
__device__ void affine_transform(double cx, double cy, int src_w, int dst_w, int dst_h, double* T) {
  float s[3][2], d[3][2];
  s[0][0] = (float)cx;
  s[0][1] = (float)cy;
  s[1][0] = (float)add(cx, 0.0);
  s[1][1] = (float)add(cy, mul((double)src_w, -0.5));
  d[0][0] = (float)mul((double)dst_w, 0.5);
  d[0][1] = (float)mul((double)dst_h, 0.5);
  d[1][0] = __fadd_rn(d[0][0], 0.f);
  d[1][1] = __fadd_rn(d[0][1], (float)mul((double)dst_w, -0.5));
  float (*pts[2])[2] = {s, d};
  for (int p = 0; p < 2; ++p) {
    float (*q)[2] = pts[p];
    const float dx = __fsub_rn(q[0][0], q[1][0]), dy = __fsub_rn(q[0][1], q[1][1]);
    q[2][0] = __fadd_rn(q[1][0], -dy);
    q[2][1] = __fadd_rn(q[1][1], dx);
  }
  double a[6][6], b[6];
  for (int i = 0; i < 3; ++i) {                 // cv2.getAffineTransform's system: rows (x y 1 0 0 0), (0 0 0 x y 1)
    for (int c = 0; c < 6; ++c) a[2 * i][c] = a[2 * i + 1][c] = 0.0;
    a[2 * i][0] = a[2 * i + 1][3] = s[i][0];
    a[2 * i][1] = a[2 * i + 1][4] = s[i][1];
    a[2 * i][2] = a[2 * i + 1][5] = 1.0;
    b[2 * i] = d[i][0];
    b[2 * i + 1] = d[i][1];
  }
  const bool ok = lu_solve6(a, b);              // cv2.solve leaves zeros for a singular system
  for (int c = 0; c < 6; ++c) T[c] = ok ? b[c] : 0.0;
}

// [T; 0 0 1] @ K for row-major 3x3 K, products summed in index order
__device__ void apply_to_K(const double* T, const double* K, double* out) {
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) out[r * 3 + c] = add(add(mul(T[r * 3], K[c]), mul(T[r * 3 + 1], K[3 + c])), mul(T[r * 3 + 2], K[6 + c]));
  for (int c = 0; c < 3; ++c) out[6 + c] = K[6 + c];
}

// Crop b of crop_transforms_kernel below; frame_ok false rejects it as a rejected box does.
__device__ __forceinline__ void crop_transforms(int b, bool frame_ok, const int32_t* __restrict__ box, const double* __restrict__ K, int stages,
                                                int out_h, int out_w, double* __restrict__ trans, double* __restrict__ K_crop,
                                                int32_t* __restrict__ status) {
  const int32_t* bx = box + (size_t)b * 4;
  double* T = trans + (size_t)b * stages * 6;
  const bool ok = frame_ok && box_ok(bx);
  if (status) status[b] = ok ? 1 : 0;
  double Kc[9];
  if (K)
    for (int i = 0; i < 9; ++i) Kc[i] = K[(size_t)b * 9 + i];
  if (!ok) {
    for (int i = 0; i < stages * 6; ++i) T[i] = 0.0;
  } else {
    const int w = bx[2] - bx[0], h = bx[3] - bx[1];
    const double cx = __ddiv_rn((double)(bx[0] + bx[2]), 2.0), cy = __ddiv_rn((double)(bx[1] + bx[3]), 2.0);
    for (int s = 0; s < stages; ++s) {
      if (s == 0) affine_transform(cx, cy, w, stages == 2 ? w : out_w, stages == 2 ? h : out_h, T);
      else affine_transform(__ddiv_rn((double)w, 2.0), __ddiv_rn((double)h, 2.0), w, out_w, out_h, T + 6);
      if (K) {
        double Kn[9];
        apply_to_K(T + s * 6, Kc, Kn);
        for (int i = 0; i < 9; ++i) Kc[i] = Kn[i];
      }
    }
  }
  if (K)
    for (int i = 0; i < 9; ++i) K_crop[(size_t)b * 9 + i] = Kc[i];
}

// One thread per frame: the transform(s) of the box, K_crop and status.  stages = 2 is crop_img_by_bbox (box -> its own size
// -> [out_h, out_w]), stages = 1 is one get_image_crop_resize (box -> [out_h, out_w]).  trans [B][stages][6].  A rejected box
// gives zero transforms, K_crop = K and status 0.  K / K_crop / status may be null.
__global__ void crop_transforms_kernel(const int32_t* __restrict__ box, const double* __restrict__ K, int B, int stages, int out_h, int out_w,
                                       double* __restrict__ trans, double* __restrict__ K_crop, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  crop_transforms(b, true, box, K, stages, out_h, out_w, trans, K_crop, status);
}

// frame_index[b] names the frame of crop b among n_frames
__device__ __forceinline__ bool frame_in_range(const int32_t* __restrict__ frame_index, int b, int n_frames) {
  const int32_t f = frame_index[b];
  return f >= 0 && f < n_frames;
}

// crop_transforms_kernel for crop_img_by_bbox (stages = 2) where crop b reads frame frame_index[b]: an index outside
// [0, n_frames) is rejected as a rejected box is.
__global__ void crop_transforms_indexed_kernel(const int32_t* __restrict__ box, const int32_t* __restrict__ frame_index, int n_frames,
                                               const double* __restrict__ K, int B, int out_size, double* __restrict__ trans,
                                               double* __restrict__ K_crop, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  crop_transforms(b, frame_in_range(frame_index, b, n_frames), box, K, 2, out_size, out_size, trans, K_crop, status);
}

// warpAffine's inversion of the forward matrix T (imgproc/src/imgwarp.cpp): m maps an output pixel to its source position
__device__ void invert_transform(const double* T, double* m) {
  double D = sub(mul(T[0], T[4]), mul(T[1], T[3]));
  D = D != 0.0 ? __ddiv_rn(1.0, D) : 0.0;
  m[0] = mul(T[4], D);
  m[4] = mul(T[0], D);
  m[1] = mul(T[1], -D);
  m[3] = mul(T[3], -D);
  m[2] = sub(mul(-m[0], T[2]), mul(m[1], T[5]));
  m[5] = sub(mul(-m[3], T[2]), mul(m[4], T[5]));
}

// The C channel values of one pixel, in memory order.
template <int C>
struct Px {
  int v[C];
};

// One pixel of cv2.warpAffine(src, T, INTER_LINEAR), border constant 0, for 8-bit data of C channels; m = invert_transform(T),
// src(x, y) gives the Px<C> at a position inside [0, sw) x [0, sh) and is called for those only.  Source coordinates in 1/1024
// (rint = round half to even), reduced to 1/32; the four weights are cv2's int16 table entries rint(w * 32768) of the float32
// products (1 - fx/32 | fx/32) * (1 - fy/32 | fy/32): those products are exact, so an entry is 32 * (32 - fx | fx) * (32 - fy |
// fy) and sums to 32768 as it stands -- but for fx = fy = 0, where 32768 saturates to 32767 and cv2's fix-up puts the 1 on a
// neighbour, which cannot change the rounded pixel (|p1 - p0| < 16384).  tests/test_crop_reference_cpu.py checks both
// statements.  cv2 warps a multi-channel image with the same positions and weights for every channel, so channel c is the grey
// warp of plane c (tests/test_scan_reference_cpu.py checks it against cv2).
template <int C, class Src>
__device__ __forceinline__ Px<C> warp_pixel(const double* m, int x, int y, int sw, int sh, Src src) {
  const long long ad = __double2ll_rn(mul(mul(m[0], (double)x), 1024.0)), bd = __double2ll_rn(mul(mul(m[3], (double)x), 1024.0));
  const long long X0 = __double2ll_rn(mul(add(mul(m[1], (double)y), m[2]), 1024.0)) + 16;
  const long long Y0 = __double2ll_rn(mul(add(mul(m[4], (double)y), m[5]), 1024.0)) + 16;
  const long long X = (X0 + ad) >> 5, Y = (Y0 + bd) >> 5;
  const int sx = (int)min(max(X >> 5, -32768LL), 32767LL), sy = (int)min(max(Y >> 5, -32768LL), 32767LL);   // saturate_cast<short>
  const int fx = (int)(X & 31), fy = (int)(Y & 31);
  const bool x0 = sx >= 0 && sx < sw, x1 = sx + 1 >= 0 && sx + 1 < sw, y0 = sy >= 0 && sy < sh, y1 = sy + 1 >= 0 && sy + 1 < sh;
  Px<C> acc{};
  auto tap = [&](int w, int u, int v) {
    const Px<C> p = src(u, v);
    for (int c = 0; c < C; ++c) acc.v[c] += w * p.v[c];
  };
  if (y0 && x0) tap((32 - fx) * (32 - fy), sx, sy);
  if (y0 && x1) tap(fx * (32 - fy), sx + 1, sy);
  if (y1 && x0) tap((32 - fx) * fy, sx, sy + 1);
  if (y1 && x1) tap(fx * fy, sx + 1, sy + 1);
  for (int c = 0; c < C; ++c) acc.v[c] = (acc.v[c] * 32 + (1 << 14)) >> 15;
  return acc;
}

// Output pixels of crop b = blockIdx.y from frame f (read only when frame_ok), C channels a pixel; see crop_warp_kernel below.
// out_u8 is [B][out_h][out_w][C]; out_f32 (C = 1 only) [B][out_h][out_w].
template <int C>
__device__ __forceinline__ void crop_warp(int f, bool frame_ok, const uint8_t* __restrict__ frames, long long frame_pitch, long long row_pitch,
                                          int H, int W, const int32_t* __restrict__ box, const double* __restrict__ trans, int stages, int out_h,
                                          int out_w, uint8_t* __restrict__ out_u8, float* __restrict__ out_f32) {
  __shared__ double m[2][6];
  __shared__ int ok;
  const int b = blockIdx.y;
  const int32_t* bx = box + (size_t)b * 4;
  if (threadIdx.x == 0) ok = frame_ok && box_ok(bx);
  if ((int)threadIdx.x < stages) invert_transform(trans + ((size_t)b * stages + threadIdx.x) * 6, m[threadIdx.x]);
  __syncthreads();
  const long long idx = (long long)blockIdx.x * kWarpThreads + threadIdx.x;
  if (idx >= (long long)out_h * out_w) return;
  const int x = (int)(idx % out_w), y = (int)(idx / out_w);
  const uint8_t* frame = frames + (size_t)f * frame_pitch;
  auto pixel = [&](int u, int v) {
    const uint8_t* q = frame + (size_t)v * row_pitch + (size_t)u * C;
    Px<C> p;
    for (int c = 0; c < C; ++c) p.v[c] = (int)__ldg(q + c);
    return p;
  };
  Px<C> val{};
  if (ok) {
    if (stages == 1) {
      val = warp_pixel<C>(m[0], x, y, W, H, pixel);
    } else {
      const double* m1 = m[0];
      val = warp_pixel<C>(m[1], x, y, bx[2] - bx[0], bx[3] - bx[1], [&](int u, int v) { return warp_pixel<C>(m1, u, v, W, H, pixel); });
    }
  }
  const size_t o = (size_t)b * out_h * out_w + (size_t)idx;
  if (out_u8)
    for (int c = 0; c < C; ++c) out_u8[o * C + c] = (uint8_t)val.v[c];
  else out_f32[o] = __fdiv_rn((float)val.v[0], 255.f);
}

// One thread per output pixel of frame blockIdx.y.  stages as in crop_transforms_kernel, whose trans this reads.  The result
// goes to out_u8 as it is, or to out_f32 as numpy's float32 `/ 255`; a rejected box gives zeros.
__global__ void __launch_bounds__(kWarpThreads) crop_warp_kernel(const uint8_t* __restrict__ frames, long long frame_pitch, long long row_pitch, int H,
                                                                 int W, const int32_t* __restrict__ box, const double* __restrict__ trans, int stages,
                                                                 int out_h, int out_w, uint8_t* __restrict__ out_u8, float* __restrict__ out_f32) {
  crop_warp<1>(blockIdx.y, true, frames, frame_pitch, row_pitch, H, W, box, trans, stages, out_h, out_w, out_u8, out_f32);
}

// crop_warp_kernel for crop_img_by_bbox into fp32 where crop blockIdx.y reads frame frame_index[blockIdx.y] of n_frames; an
// index outside that range gives zeros.
__global__ void __launch_bounds__(kWarpThreads) crop_warp_indexed_kernel(const uint8_t* __restrict__ frames, long long frame_pitch,
                                                                         long long row_pitch, int n_frames, int H, int W,
                                                                         const int32_t* __restrict__ frame_index, const int32_t* __restrict__ box,
                                                                         const double* __restrict__ trans, int out_size, float* __restrict__ out) {
  const int b = blockIdx.y;
  const bool in = frame_in_range(frame_index, b, n_frames);
  crop_warp<1>(in ? frame_index[b] : 0, in, frames, frame_pitch, row_pitch, H, W, box, trans, 2, out_size, out_size, nullptr, out);
}

// crop_img_by_bbox's two warps into uint8 for frames of C channels: crop blockIdx.y reads frame frame_index[blockIdx.y] of
// n_frames (an index outside that range gives zeros), or frame blockIdx.y when frame_index is null.
template <int C>
__global__ void __launch_bounds__(kWarpThreads) crop_warp_colour_kernel(const uint8_t* __restrict__ frames, long long frame_pitch, long long row_pitch,
                                                                        int n_frames, int H, int W, const int32_t* __restrict__ frame_index,
                                                                        const int32_t* __restrict__ box, const double* __restrict__ trans, int out_size,
                                                                        uint8_t* __restrict__ out) {
  const int b = blockIdx.y;
  const bool in = !frame_index || frame_in_range(frame_index, b, n_frames);
  crop_warp<C>(frame_index ? (in ? frame_index[b] : 0) : b, in, frames, frame_pitch, row_pitch, H, W, box, trans, 2, out_size, out_size, out, nullptr);
}

// One thread per frame: vis_utils.reproj (:209-236) of n points, (K_homo @ pose_homo) @ X then the division by the third row, and
// previous_pose_detect's box (:247-249): min / max, then C truncation.  Products are summed in index order.
__global__ void boxes_from_poses_kernel(const double* __restrict__ K, const double* __restrict__ pose, const double* __restrict__ pts, int B, int n,
                                        double* __restrict__ proj, int32_t* __restrict__ box) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* Kb = K + (size_t)b * 9;
  const double* Pb = pose + (size_t)b * 12;
  double P[3][4];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) P[r][c] = add(add(mul(Kb[r * 3], Pb[c]), mul(Kb[r * 3 + 1], Pb[4 + c])), mul(Kb[r * 3 + 2], Pb[8 + c]));
  double lo[2] = {INFINITY, INFINITY}, hi[2] = {-INFINITY, -INFINITY};
  bool finite = true;
  for (int i = 0; i < n; ++i) {
    const double* X = pts + ((size_t)b * n + i) * 3;
    double p[3];
    for (int r = 0; r < 3; ++r) p[r] = add(add(add(mul(P[r][0], X[0]), mul(P[r][1], X[1])), mul(P[r][2], X[2])), P[r][3]);
    for (int a = 0; a < 2; ++a) {
      const double v = __ddiv_rn(p[a], p[2]);
      if (proj) proj[((size_t)b * n + i) * 2 + a] = v;
      finite = finite && isfinite(v);
      lo[a] = fmin(lo[a], v);
      hi[a] = fmax(hi[a], v);
    }
  }
  const double e[4] = {lo[0], lo[1], hi[0], hi[1]};
  for (int a = 0; a < 4; ++a) finite = finite && e[a] > -2147483649.0 && e[a] < 2147483648.0;   // what astype(int32) defines
  for (int a = 0; a < 4; ++a) box[(size_t)b * 4 + a] = finite ? (int32_t)e[a] : 0;
}

int launch_crop(const char* fn, const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* box,
                const double* K, int stages, int32_t out_h, int32_t out_w, uint8_t* out_u8, float* out_f32, double* trans, double* K_crop,
                int32_t* status, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH_NH(fn, crop_transforms_kernel, (unsigned)((B + 127) / 128), 128, 0, st, box, K, B, stages, out_h, out_w, trans, K_crop, status);
  if (frames) {
    const long long blocks = ((long long)out_h * out_w + kWarpThreads - 1) / kWarpThreads;
    LAUNCH_NH(fn, crop_warp_kernel, dim3((unsigned)blocks, (unsigned)B), kWarpThreads, 0, st, frames, frame_pitch, row_pitch, H, W, box, trans, stages,
              out_h, out_w, out_u8, out_f32);
  }
  return OPB_OK;
}

int check_frames(const char* fn, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W) {
  REQUIRE(fn, B > 0 && B <= 65535 && H > 0 && H <= kMaxSide && W > 0 && W <= kMaxSide && row_pitch >= W && frame_pitch >= 0);
  return OPB_OK;
}

}  // namespace
}  // namespace opb

extern "C" int opb_boxes_from_poses(const double* K, const double* pose, const double* corners, int32_t B, int32_t n_corners, double* proj,
                                    int32_t* box, void* stream) {
  REQUIRE(__func__, K && pose && corners && box && B > 0 && n_corners > 0);
  LAUNCH_NH(__func__, opb::boxes_from_poses_kernel, (unsigned)((B + 127) / 128), 128, 0, (cudaStream_t)stream, K, pose, corners, B, n_corners, proj,
            box);
  return OPB_OK;
}

extern "C" int opb_crop_resize(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* box,
                               const double* K, int32_t crop_size, float* image, double* K_crop, double* trans, int32_t* status, void* stream) {
  REQUIRE(__func__, frames && box && K && image && K_crop && trans && status);
  if (int rc = opb::check_frames(__func__, frame_pitch, row_pitch, B, H, W)) return rc;
  REQUIRE(__func__, crop_size > 0 && crop_size % 8 == 0 && crop_size <= opb::kMaxSide);
  return opb::launch_crop(__func__, frames, frame_pitch, row_pitch, B, H, W, box, K, 2, crop_size, crop_size, nullptr, image, trans, K_crop, status,
                          stream);
}

extern "C" int opb_crop_resize_indexed(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t n_frames, int32_t H, int32_t W,
                                       const int32_t* frame_index, int32_t B, const int32_t* box, const double* K, int32_t crop_size, float* image,
                                       double* K_crop, double* trans, int32_t* status, void* stream) {
  REQUIRE(__func__, frames && frame_index && box && K && image && K_crop && trans && status);
  if (int rc = opb::check_frames(__func__, frame_pitch, row_pitch, B, H, W)) return rc;
  REQUIRE(__func__, n_frames > 0 && crop_size > 0 && crop_size % 8 == 0 && crop_size <= opb::kMaxSide);
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH_NH(__func__, opb::crop_transforms_indexed_kernel, (unsigned)((B + 127) / 128), 128, 0, st, box, frame_index, n_frames, K, B, crop_size,
            trans, K_crop, status);
  const long long blocks = ((long long)crop_size * crop_size + opb::kWarpThreads - 1) / opb::kWarpThreads;
  LAUNCH_NH(__func__, opb::crop_warp_indexed_kernel, dim3((unsigned)blocks, (unsigned)B), opb::kWarpThreads, 0, st, frames, frame_pitch, row_pitch,
            n_frames, H, W, frame_index, box, trans, crop_size, image);
  return OPB_OK;
}

extern "C" int opb_warp_crop_u8(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* box,
                                const double* K, int32_t out_h, int32_t out_w, uint8_t* out, double* trans, double* K_crop, void* stream) {
  REQUIRE(__func__, box && trans && (frames != nullptr) == (out != nullptr) && (K != nullptr) == (K_crop != nullptr));
  REQUIRE(__func__, B > 0 && B <= 65535 && out_h > 0 && out_h <= opb::kMaxSide && out_w > 0 && out_w <= opb::kMaxSide);
  if (frames)
    if (int rc = opb::check_frames(__func__, frame_pitch, row_pitch, B, H, W)) return rc;
  return opb::launch_crop(__func__, frames, frame_pitch, row_pitch, B, H, W, box, K, 1, out_h, out_w, out, nullptr, trans, K_crop, nullptr, stream);
}

extern "C" int opb_crop_resize_colour(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t n_frames, int32_t H, int32_t W, int32_t C,
                                      const int32_t* frame_index, int32_t B, const int32_t* box, const double* K, int32_t crop_size, uint8_t* image,
                                      double* K_crop, double* trans, int32_t* status, void* stream) {
  REQUIRE(__func__, frames && box && K && image && K_crop && trans && status);
  REQUIRE(__func__, C == 3 || C == 4);
  if (int rc = opb::check_frames(__func__, frame_pitch, row_pitch, B, H, W)) return rc;
  REQUIRE(__func__, row_pitch >= (int64_t)W * C);
  REQUIRE(__func__, n_frames > 0 && (frame_index != nullptr || n_frames == B));
  REQUIRE(__func__, crop_size > 0 && crop_size % 8 == 0 && crop_size <= opb::kMaxSide);
  cudaStream_t st = (cudaStream_t)stream;
  if (frame_index)
    LAUNCH_NH(__func__, opb::crop_transforms_indexed_kernel, (unsigned)((B + 127) / 128), 128, 0, st, box, frame_index, n_frames, K, B, crop_size,
              trans, K_crop, status);
  else
    LAUNCH_NH(__func__, opb::crop_transforms_kernel, (unsigned)((B + 127) / 128), 128, 0, st, box, K, B, 2, crop_size, crop_size, trans, K_crop, status);
  const dim3 grid((unsigned)(((long long)crop_size * crop_size + opb::kWarpThreads - 1) / opb::kWarpThreads), (unsigned)B);
  if (C == 3)
    LAUNCH_NH(__func__, opb::crop_warp_colour_kernel<3>, grid, opb::kWarpThreads, 0, st, frames, frame_pitch, row_pitch, n_frames, H, W, frame_index, box,
              trans, crop_size, image);
  else
    LAUNCH_NH(__func__, opb::crop_warp_colour_kernel<4>, grid, opb::kWarpThreads, 0, st, frames, frame_pitch, row_pitch, n_frames, H, W, frame_index, box,
              trans, crop_size, image);
  return OPB_OK;
}
