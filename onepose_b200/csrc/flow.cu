// Pyramidal Lucas-Kanade on the GPU: cv2.calcOpticalFlowPyrLK for B image pairs, and the per-track steps around it that the
// reference tracker's flow_track (src/tracker/ba_tracker.py:295-356) runs on the host.
//   kpt_flow_track   :113-126   cv2.calcOpticalFlowPyrLK(winSize 15, maxLevel 2, (EPS|COUNT, 10, 0.03))   opb_calc_optical_flow_pyr_lk
//                               np.where(status == 1), mkpts2d[valid], mkpts3d[valid]                       opb_flow_compact
//   flow_track       :326-327   mean |project(kpt3ds, K_crop, pose_init) - mkpts2d|                        opb_flow_reprojection
//
// The points, status and err are OpenCV's bit for bit (OpenCV 4.13 on x86; the model is tests/lk_reference.py and DESIGN
// §5.9 lists what was probed).  The window arithmetic is integer up to the fp32 sums of the structure tensor and the mismatch
// vector; those are added in the order of OpenCV's SIMD loops, and every fp32 / fp64 operation after them is a separate
// rounding (__fadd_rn and friends) so that nothing is contracted into a fused multiply-add.
//
// Launches, all on the caller's stream: one per pyramid level (the Scharr derivatives of prev at that level and pyrDown of
// both images to the next), then one thread per point for the tracking, coarsest level first.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "block.cuh"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kMaxLevel = 4;
constexpr int kMaxWin = 31;
constexpr int kMaxSideLk = 32767;
constexpr int kPyrThreads = 256;
constexpr int kTrackThreads = 128;
constexpr int kCompactThreads = 1024;
constexpr int kWBits = 14;

// Level sizes of a pyramid whose level 0 is h x w: each level ceil-halves the one above.
__host__ __device__ inline int level_dim(int d, int l) {
  for (int i = 0; i < l; ++i) d = (d + 1) / 2;
  return d;
}

// The last level cv2.buildOpticalFlowPyramid builds: after level l it stops when the next level has a side <= the window's.
__host__ __device__ inline int last_level(int h, int w, int win_w, int win_h, int max_level) {
  for (int l = 0; l < max_level; ++l) {
    w = (w + 1) / 2;
    h = (h + 1) / 2;
    if (w <= win_w || h <= win_h) return l;
  }
  return max_level;
}

__host__ __device__ inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// Workspace layout (include/onepose_b200.h): per pair a slot of pair_bytes; inside it, per level l = 0..max_level of the
// H x W pyramid, the prev derivatives int16 [h_l, w_l, 2], then for l >= 1 the prev and next images uint8 [h_l, w_l], each
// 16-byte aligned.  A pair smaller than H x W uses the top-left corner of each level with the pitch w_l.
struct PyrLayout {
  size_t der[kMaxLevel + 1], prev[kMaxLevel + 1], next[kMaxLevel + 1];
  size_t pair_bytes;
};

__host__ __device__ inline PyrLayout make_layout(int H, int W, int max_level) {
  PyrLayout L{};
  size_t o = 0;
  for (int l = 0; l <= max_level; ++l) {
    const size_t px = (size_t)level_dim(H, l) * level_dim(W, l);
    L.der[l] = o;
    o = align16(o + px * 4);
    if (l > 0) {
      L.prev[l] = o;
      o = align16(o + px);
      L.next[l] = o;
      o = align16(o + px);
    }
  }
  L.pair_bytes = o;
  return L;
}

struct Params {
  const uint8_t* prev;
  const uint8_t* next;
  long long prev_frame_pitch, prev_row_pitch, next_frame_pitch, next_row_pitch;
  const int32_t* sizes;   // [B, 2] = (h, w) per pair, or null: every pair is H x W
  int B, H, W, win_w, win_h, max_level;
  uint8_t* ws;
  PyrLayout L;
};

// Pair b's image size; an entry of sizes outside [1, H] x [1, W] is clamped into it, so that no read leaves the caller's images
// and no write leaves the pair's workspace slot.
__device__ inline void pair_size(const Params& p, int b, int& h, int& w) {
  h = p.sizes ? min(max(p.sizes[2 * b], 1), p.H) : p.H;
  w = p.sizes ? min(max(p.sizes[2 * b + 1], 1), p.W) : p.W;
}

// An image level: level 0 is the caller's image, the others live in the workspace with pitch w_l.
struct Plane {
  const uint8_t* p;
  long long pitch;
  int h, w;
};

__device__ inline Plane image_level(const Params& p, int b, bool nxt, int l) {
  int h, w;
  pair_size(p, b, h, w);
  if (l == 0)
    return nxt ? Plane{p.next + b * p.next_frame_pitch, p.next_row_pitch, h, w} : Plane{p.prev + b * p.prev_frame_pitch, p.prev_row_pitch, h, w};
  const uint8_t* base = p.ws + (size_t)b * p.L.pair_bytes + (nxt ? p.L.next[l] : p.L.prev[l]);
  return Plane{base, level_dim(p.W, l), level_dim(h, l), level_dim(w, l)};
}

__device__ inline short2* deriv_level(const Params& p, int b, int l) {
  return reinterpret_cast<short2*>(p.ws + (size_t)b * p.L.pair_bytes + p.L.der[l]);
}

// cv::borderInterpolate(i, n, BORDER_REFLECT_101)
__device__ __forceinline__ int reflect101(int i, int n) {
  if ((unsigned)i < (unsigned)n) return i;
  if (n == 1) return 0;
  do {
    i = i < 0 ? -i : 2 * n - 2 - i;
  } while ((unsigned)i >= (unsigned)n);
  return i;
}

__device__ __forceinline__ int px(const Plane& P, int y, int x) { return P.p[(long long)reflect101(y, P.h) * P.pitch + reflect101(x, P.w)]; }

// Level l of pair b = blockIdx.y: task blockIdx.z = 0 writes the Scharr derivatives of prev_l, tasks 1 and 2 pyrDown prev_l / next_l into level l + 1.
// One thread per output pixel.
__global__ void __launch_bounds__(kPyrThreads) pyramid_kernel(Params p, int l) {
  const int b = blockIdx.y, task = blockIdx.z;
  int h0, w0;
  pair_size(p, b, h0, w0);
  const int top = last_level(h0, w0, p.win_w, p.win_h, p.max_level);
  if (l > top || (task > 0 && l == top)) return;
  const Plane src = image_level(p, b, task == 2, l);
  const int oh = task ? (src.h + 1) / 2 : src.h, ow = task ? (src.w + 1) / 2 : src.w;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)oh * ow) return;
  const int y = (int)(i / ow), x = (int)(i % ow);
  if (task == 0) {
    // calcScharrDeriv: vertical [3 10 3] and [-1 0 1] first, then horizontal [-1 0 1] and [3 10 3]
    int t0[3], t1[3];
    for (int k = 0; k < 3; ++k) {
      const int xx = x + k - 1;
      const int a = px(src, y - 1, xx), c = px(src, y, xx), d = px(src, y + 1, xx);
      t0[k] = (a + d) * 3 + c * 10;
      t1[k] = d - a;
    }
    deriv_level(p, b, l)[(size_t)y * level_dim(p.W, l) + x] = make_short2((short)(t0[2] - t0[0]), (short)((t1[2] + t1[0]) * 3 + t1[1] * 10));
    return;
  }
  // pyrDown: [1 4 6 4 1]^2, (sum + 128) >> 8
  const int k5[5] = {1, 4, 6, 4, 1};
  int s = 0;
  for (int dy = 0; dy < 5; ++dy) {
    int r = 0;
    for (int dx = 0; dx < 5; ++dx) r += k5[dx] * px(src, 2 * y + dy - 2, 2 * x + dx - 2);
    s += k5[dy] * r;
  }
  const Plane dst = image_level(p, b, task == 2, l + 1);
  const_cast<uint8_t*>(dst.p)[(size_t)y * dst.pitch + x] = (uint8_t)((s + 128) >> 8);
}

// cvFloor; a non-finite or huge coordinate maps far outside every image (cv2's conversion gives INT_MIN there).
__device__ __forceinline__ int cv_floor(float v) { return fabsf(v) < 1e9f ? (int)floorf(v) : -(1 << 30); }

struct Weights {
  int w00, w01, w10, w11;
};

// cvRound of the fp32 bilinear products at fraction (a, b); the fourth weight makes up 1 << 14.
__device__ __forceinline__ Weights weights(float a, float b) {
  const float s = (float)(1 << kWBits);
  Weights w;
  w.w00 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), __fsub_rn(1.f, b)), s));
  w.w01 = __float2int_rn(__fmul_rn(__fmul_rn(a, __fsub_rn(1.f, b)), s));
  w.w10 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), b), s));
  w.w11 = (1 << kWBits) - w.w00 - w.w01 - w.w10;
  return w;
}

__device__ __forceinline__ int descale(int v, int n) { return (v + (1 << (n - 1))) >> n; }

// The image window at (y, x) from the integer corner (iy, ix), in 1/32 grey levels.
__device__ __forceinline__ int win_px(const Plane& P, int iy, int ix, int y, int x, const Weights& w) {
  const int yy = iy + y, xx = ix + x;
  return descale(px(P, yy, xx) * w.w00 + px(P, yy, xx + 1) * w.w01 + px(P, yy + 1, xx) * w.w10 + px(P, yy + 1, xx + 1) * w.w11, kWBits - 5);
}

// The derivative window at (y, x), zero outside the level.
__device__ __forceinline__ short2 der_at(const short2* d, int pitch, int h, int w, int y, int x) {
  return (unsigned)y < (unsigned)h && (unsigned)x < (unsigned)w ? d[(size_t)y * pitch + x] : make_short2(0, 0);
}

__device__ __forceinline__ void win_der(const short2* d, int pitch, int h, int w, int iy, int ix, int y, int x, const Weights& wt, int& gx, int& gy) {
  const int yy = iy + y, xx = ix + x;
  const short2 a = der_at(d, pitch, h, w, yy, xx), b = der_at(d, pitch, h, w, yy, xx + 1);
  const short2 c = der_at(d, pitch, h, w, yy + 1, xx), e = der_at(d, pitch, h, w, yy + 1, xx + 1);
  gx = descale(a.x * wt.w00 + b.x * wt.w01 + c.x * wt.w10 + e.x * wt.w11, kWBits);
  gy = descale(a.y * wt.w00 + b.y * wt.w01 + c.y * wt.w10 + e.y * wt.w11, kWBits);
}

__device__ __forceinline__ bool outside(int ix, int iy, int w, int h, int win_w, int win_h) {
  return ix < -win_w || ix >= w || iy < -win_h || iy >= h;
}

// One thread per point: LKTrackerInvoker over the levels of its pair, coarsest first.
__global__ void __launch_bounds__(kTrackThreads) track_kernel(Params p, const float* __restrict__ pts, const int32_t* __restrict__ offsets, int total,
                                                              int max_count, double eps2, float min_eig, float* __restrict__ next_pts,
                                                              uint8_t* __restrict__ status, float* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int lo = 0, hi = p.B;                        // the pair that owns row i: offsets[b] <= i < offsets[b + 1]
  while (hi - lo > 1) {
    const int mid = (lo + hi) / 2;
    if (offsets[mid] <= i) lo = mid;
    else hi = mid;
  }
  const int b = lo;
  int h0, w0;
  pair_size(p, b, h0, w0);
  const int top = last_level(h0, w0, p.win_w, p.win_h, p.max_level);
  const int ww = p.win_w, wh = p.win_h;
  const float hx = (float)(ww - 1) * 0.5f, hy = (float)(wh - 1) * 0.5f;
  const int xv = ww / 8 * 8;                   // columns OpenCV's SIMD loops cover; the rest of a row goes one by one
  const float px0 = pts[2 * (size_t)i], py0 = pts[2 * (size_t)i + 1];
  bool st = true;
  float e_out = 0.f;
  float nx = 0.f, ny = 0.f;                    // nextPts[i]
  for (int l = top; l >= 0; --l) {
    const Plane I = image_level(p, b, false, l), J = image_level(p, b, true, l);
    const short2* dI = deriv_level(p, b, l);
    const int dpitch = level_dim(p.W, l);
    const float sc = (float)(1.0 / (1 << l));
    float prx = __fmul_rn(px0, sc), pry = __fmul_rn(py0, sc);
    if (l == top) {
      nx = prx;
      ny = pry;
    } else {
      nx = __fmul_rn(nx, 2.f);
      ny = __fmul_rn(ny, 2.f);
    }
    prx = __fsub_rn(prx, hx);
    pry = __fsub_rn(pry, hy);
    const int ipx = cv_floor(prx), ipy = cv_floor(pry);
    if (outside(ipx, ipy, I.w, I.h, ww, wh)) {
      if (l == 0) {
        st = false;
        e_out = 0.f;
      }
      continue;
    }
    const Weights wp = weights(__fsub_rn(prx, (float)ipx), __fsub_rn(pry, (float)ipy));
    // structure tensor: columns x < xv into lane x % 4, the rest into the scalar sum, lanes added last
    float a11[4] = {0.f, 0.f, 0.f, 0.f}, a12[4] = {0.f, 0.f, 0.f, 0.f}, a22[4] = {0.f, 0.f, 0.f, 0.f};
    float t11 = 0.f, t12 = 0.f, t22 = 0.f;
    for (int y = 0; y < wh; ++y) {
      for (int x0 = 0; x0 < xv; x0 += 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          int gx, gy;
          win_der(dI, dpitch, I.h, I.w, ipy, ipx, y, x0 + k, wp, gx, gy);
          a11[k] = __fadd_rn(a11[k], (float)(gx * gx));     // the products are exact in fp32: |g| <= 4080
          a12[k] = __fadd_rn(a12[k], (float)(gx * gy));
          a22[k] = __fadd_rn(a22[k], (float)(gy * gy));
        }
      }
      for (int x = xv; x < ww; ++x) {
        int gx, gy;
        win_der(dI, dpitch, I.h, I.w, ipy, ipx, y, x, wp, gx, gy);
        t11 = __fadd_rn(t11, (float)(gx * gx));
        t12 = __fadd_rn(t12, (float)(gx * gy));
        t22 = __fadd_rn(t22, (float)(gy * gy));
      }
    }
    const float kScale = 1.f / (1 << 20);
    const float A11 = __fmul_rn(__fadd_rn(t11, __fadd_rn(__fadd_rn(a11[0], a11[2]), __fadd_rn(a11[1], a11[3]))), kScale);
    const float A12 = __fmul_rn(__fadd_rn(t12, __fadd_rn(__fadd_rn(a12[0], a12[2]), __fadd_rn(a12[1], a12[3]))), kScale);
    const float A22 = __fmul_rn(__fadd_rn(t22, __fadd_rn(__fadd_rn(a22[0], a22[2]), __fadd_rn(a22[1], a22[3]))), kScale);
    float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
    const float dd = __fsub_rn(A11, A22);
    const float eig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(__fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12)))),
                                (float)(2 * ww * wh));
    if (eig < min_eig || D < 1.1920929e-07f) {
      if (l == 0) st = false;
      continue;
    }
    D = __fdiv_rn(1.f, D);
    float qx = __fsub_rn(nx, hx), qy = __fsub_rn(ny, hy);
    float pdx = 0.f, pdy = 0.f;
    for (int j = 0; j < max_count; ++j) {
      const int inx = cv_floor(qx), iny = cv_floor(qy);
      if (outside(inx, iny, J.w, J.h, ww, wh)) {
        if (l == 0) st = false;
        break;
      }
      const Weights wn = weights(__fsub_rn(qx, (float)inx), __fsub_rn(qy, (float)iny));
      // mismatch: per row, blocks of 8 columns whose products k and k + 4 are added as integers into lane k
      float b1l[4] = {0.f, 0.f, 0.f, 0.f}, b2l[4] = {0.f, 0.f, 0.f, 0.f};
      float b1t = 0.f, b2t = 0.f;
      for (int y = 0; y < wh; ++y) {
        for (int x0 = 0; x0 < xv; x0 += 8) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            int s1 = 0, s2 = 0;
#pragma unroll
            for (int h = 0; h < 8; h += 4) {
              const int x = x0 + k + h;
              int gx, gy;
              win_der(dI, dpitch, I.h, I.w, ipy, ipx, y, x, wp, gx, gy);
              const int diff = win_px(J, iny, inx, y, x, wn) - win_px(I, ipy, ipx, y, x, wp);
              s1 += diff * gx;
              s2 += diff * gy;
            }
            b1l[k] = __fadd_rn(b1l[k], (float)s1);
            b2l[k] = __fadd_rn(b2l[k], (float)s2);
          }
        }
        for (int x = xv; x < ww; ++x) {
          int gx, gy;
          win_der(dI, dpitch, I.h, I.w, ipy, ipx, y, x, wp, gx, gy);
          const int diff = win_px(J, iny, inx, y, x, wn) - win_px(I, ipy, ipx, y, x, wp);
          b1t = __fadd_rn(b1t, (float)(diff * gx));
          b2t = __fadd_rn(b2t, (float)(diff * gy));
        }
      }
      const float b1 = __fmul_rn(__fadd_rn(b1t, __fadd_rn(__fadd_rn(b1l[0], b1l[2]), __fadd_rn(b1l[1], b1l[3]))), kScale);
      const float b2 = __fmul_rn(__fadd_rn(b2t, __fadd_rn(__fadd_rn(b2l[0], b2l[2]), __fadd_rn(b2l[1], b2l[3]))), kScale);
      const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, b2), __fmul_rn(A22, b1)), D);
      const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, b1), __fmul_rn(A11, b2)), D);
      qx = __fadd_rn(qx, dx);
      qy = __fadd_rn(qy, dy);
      nx = __fadd_rn(qx, hx);
      ny = __fadd_rn(qy, hy);
      if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= eps2) break;
      if (j > 0 && fabs((double)__fadd_rn(dx, pdx)) < 0.01 && fabs((double)__fadd_rn(dy, pdy)) < 0.01) {   // oscillation: half a step back
        nx = __fsub_rn(nx, __fmul_rn(dx, 0.5f));
        ny = __fsub_rn(ny, __fmul_rn(dy, 0.5f));
        break;
      }
      pdx = dx;
      pdy = dy;
    }
    if (l == 0 && st) {                          // err: mean |J - I| over the window at the final position, in grey levels
      const float ex = __fsub_rn(nx, hx), ey = __fsub_rn(ny, hy);
      const int iex = cv_floor(ex), iey = cv_floor(ey);
      if (outside(iex, iey, J.w, J.h, ww, wh)) {
        st = false;
        break;
      }
      const Weights we = weights(__fsub_rn(ex, (float)iex), __fsub_rn(ey, (float)iey));
      int sum = 0;                                 // below 2^24, so cv2's fp32 sum of the same integers is exact
      for (int y = 0; y < wh; ++y)
        for (int x = 0; x < ww; ++x) sum += abs(win_px(J, iey, iex, y, x, we) - win_px(I, ipy, ipx, y, x, wp));
      e_out = __fdiv_rn((float)sum, (float)(32 * ww * wh));
    }
  }
  next_pts[2 * (size_t)i] = nx;
  next_pts[2 * (size_t)i + 1] = ny;
  status[i] = st ? 1 : 0;
  err[i] = st ? e_out : 0.f;
}

// One block: for each track b in order, the rows r < counts[b] of [b * cap, (b + 1) * cap) with status 1, in index order, are
// appended to the outputs (as fp64), offsets[b] .. offsets[b + 1] marking track b's range, and copied to the front of track
// b's rows of pad2d / pad3d (as fp32, the rest of its rows zero).
__global__ void __launch_bounds__(kCompactThreads) compact_kernel(const uint8_t* __restrict__ status, const float* __restrict__ pts2d,
                                                                  const float* __restrict__ pts3d, const int32_t* __restrict__ counts, int B, int cap,
                                                                  double* __restrict__ out2d, double* __restrict__ out3d, int32_t* __restrict__ offsets,
                                                                  int32_t* __restrict__ n_tracked, float* __restrict__ pad2d, float* __restrict__ pad3d) {
  __shared__ int sh[kCompactThreads / 32];
  const int t = threadIdx.x;
  int base = 0;
  for (int b = 0; b < B; ++b) {
    const int n = min(max(counts[b], 0), cap);
    const int start = base;
    if (t == 0) offsets[b] = start;
    for (int c = 0; c < n; c += kCompactThreads) {
      const int r = c + t;
      const size_t row = (size_t)b * cap + r;
      const bool keep = r < n && status[row] == 1;
      int total;
      const int rank = base - start + block_rank(keep, sh, &total);
      if (keep) {
        const size_t o = (size_t)start + rank, q = (size_t)b * cap + rank;
        for (int k = 0; k < 2; ++k) {
          out2d[2 * o + k] = pts2d[2 * row + k];
          pad2d[2 * q + k] = pts2d[2 * row + k];
        }
        for (int k = 0; k < 3; ++k) {
          out3d[3 * o + k] = pts3d[3 * row + k];
          pad3d[3 * q + k] = pts3d[3 * row + k];
        }
      }
      base += total;
    }
    const int kept = base - start;
    for (int r = kept + t; r < cap; r += kCompactThreads) {
      const size_t q = (size_t)b * cap + r;
      for (int k = 0; k < 2; ++k) pad2d[2 * q + k] = 0.f;
      for (int k = 0; k < 3; ++k) pad3d[3 * q + k] = 0.f;
    }
    if (t == 0) n_tracked[b] = kept;
  }
  if (t == 0) offsets[B] = base;
}

// One thread per track: tracking_utils.project(pts3d, K, pose) -- X R^T + t, then K, then x / z -- and the mean distance to
// pts2d, in fp64 (NaN for a track without points, as np.mean of nothing).
__global__ void reprojection_kernel(const double* __restrict__ K, const double* __restrict__ pose, const double* __restrict__ pts2d,
                                    const double* __restrict__ pts3d, const int32_t* __restrict__ offsets, int B, double* __restrict__ dist) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* k = K + 9 * (size_t)b;
  const double* P = pose + 12 * (size_t)b;
  double s = 0.0;
  const int lo = offsets[b], hi = offsets[b + 1];
  for (int i = lo; i < hi; ++i) {
    const double* X = pts3d + 3 * (size_t)i;
    double c[3], q[3];
    for (int r = 0; r < 3; ++r) c[r] = X[0] * P[4 * r] + X[1] * P[4 * r + 1] + X[2] * P[4 * r + 2] + P[4 * r + 3];
    for (int r = 0; r < 3; ++r) q[r] = c[0] * k[3 * r] + c[1] * k[3 * r + 1] + c[2] * k[3 * r + 2];
    const double dx = q[0] / q[2] - pts2d[2 * (size_t)i], dy = q[1] / q[2] - pts2d[2 * (size_t)i + 1];
    s += sqrt(dx * dx + dy * dy);
  }
  dist[b] = s / (double)(hi - lo);
}

}  // namespace
}  // namespace opb

extern "C" int opb_optical_flow_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t max_level, int64_t* bytes) {
  REQUIRE(__func__, bytes && B > 0 && H > 0 && H <= opb::kMaxSideLk && W > 0 && W <= opb::kMaxSideLk && max_level >= 0 &&
                        max_level <= opb::kMaxLevel);
  *bytes = (int64_t)B * (int64_t)opb::make_layout(H, W, max_level).pair_bytes;
  return OPB_OK;
}

extern "C" int opb_calc_optical_flow_pyr_lk(const uint8_t* prev, int64_t prev_frame_pitch, int64_t prev_row_pitch, const uint8_t* next,
                                            int64_t next_frame_pitch, int64_t next_row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* sizes,
                                            const float* pts, const int32_t* offsets, int32_t total, int32_t win_w, int32_t win_h, int32_t max_level,
                                            int32_t criteria_type, int32_t max_count, double epsilon, double min_eig_threshold, int32_t flags,
                                            void* workspace, int64_t workspace_bytes, float* next_pts, uint8_t* status, float* err, void* stream) {
  using namespace opb;
  REQUIRE(__func__, prev && next && offsets && workspace && (total == 0 || (pts && next_pts && status && err)));
  REQUIRE(__func__, ((uintptr_t)workspace & 15) == 0);   // the derivative planes are read and written as short2
  REQUIRE(__func__, B > 0 && B <= 65535 && H > 0 && H <= kMaxSideLk && W > 0 && W <= kMaxSideLk && total >= 0);
  REQUIRE(__func__, prev_row_pitch >= W && next_row_pitch >= W && prev_frame_pitch >= 0 && next_frame_pitch >= 0);
  REQUIRE(__func__, win_w >= 3 && win_w <= kMaxWin && win_w % 2 == 1 && win_h >= 3 && win_h <= kMaxWin && win_h % 2 == 1);
  REQUIRE(__func__, max_level >= 0 && max_level <= kMaxLevel);
  REQUIRE(__func__, (criteria_type & ~3) == 0 && criteria_type != 0);
  REQUIRE(__func__, !(criteria_type & 1) || (max_count >= 1 && max_count <= 100));
  REQUIRE(__func__, !(criteria_type & 2) || epsilon >= 0.0);
  REQUIRE(__func__, min_eig_threshold >= 0.0);
  REQUIRE(__func__, flags == 0);   // OPTFLOW_USE_INITIAL_FLOW and OPTFLOW_LK_GET_MIN_EIGENVALS are not supported
  const PyrLayout L = make_layout(H, W, max_level);
  REQUIRE(__func__, workspace_bytes >= (int64_t)B * (int64_t)L.pair_bytes);
  // calcOpticalFlowPyrLK's criteria: COUNT absent -> 30 steps, EPS absent -> 0.01; eps at most 10, compared squared
  const int count = (criteria_type & 1) ? max_count : 30;
  const double eps = (criteria_type & 2) ? fmin(epsilon, 10.0) : 0.01;
  Params p{prev, next, prev_frame_pitch, prev_row_pitch, next_frame_pitch, next_row_pitch, sizes, B, H, W, win_w, win_h, max_level,
           (uint8_t*)workspace, L};
  cudaStream_t st = (cudaStream_t)stream;
  for (int l = 0; l <= max_level; ++l) {
    const long long npx = (long long)level_dim(H, l) * level_dim(W, l);
    LAUNCH_NH(__func__, pyramid_kernel, dim3((unsigned)((npx + kPyrThreads - 1) / kPyrThreads), (unsigned)B, 3), kPyrThreads, 0, st, p, l);
  }
  if (total > 0)
    LAUNCH_NH(__func__, track_kernel, (unsigned)((total + kTrackThreads - 1) / kTrackThreads), kTrackThreads, 0, st, p, pts, offsets, total, count,
              eps * eps, (float)min_eig_threshold, next_pts, status, err);
  return OPB_OK;
}

extern "C" int opb_flow_compact(const uint8_t* status, const float* pts2d, const float* pts3d, const int32_t* counts, int32_t B, int32_t cap,
                                double* out2d, double* out3d, int32_t* offsets, int32_t* n_tracked, float* pad2d, float* pad3d, void* stream) {
  REQUIRE(__func__, counts && offsets && n_tracked && B > 0 && cap >= 0 && (int64_t)B * cap <= (int64_t)INT32_MAX);
  REQUIRE(__func__, cap == 0 || (status && pts2d && pts3d && out2d && out3d && pad2d && pad3d));
  LAUNCH_NH(__func__, opb::compact_kernel, 1, opb::kCompactThreads, 0, (cudaStream_t)stream, status, pts2d, pts3d, counts, B, cap, out2d, out3d,
            offsets, n_tracked, pad2d, pad3d);
  return OPB_OK;
}

extern "C" int opb_flow_reprojection(const double* K, const double* pose, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B,
                                     double* dist, void* stream) {
  REQUIRE(__func__, K && pose && offsets && dist && B > 0);
  LAUNCH_NH(__func__, opb::reprojection_kernel, (unsigned)((B + 127) / 128), 128, 0, (cudaStream_t)stream, K, pose, pts2d, pts3d, offsets, B, dist);
  return OPB_OK;
}
