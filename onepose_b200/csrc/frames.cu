// Colour camera frames to the reference's grey frames on the GPU.  The reference reads every frame it works on as
// cv2.imread(path, cv2.IMREAD_GRAYSCALE) of a colour PNG (src/datasets/normalized_dataset.py:25-26, data_utils.py:275-276,
// local_feature_2D_detector.py:12, :155, :173); opb_grey_frames gives those pixels from the colour pixels in memory, for F frames
// in one launch, and optionally the `image / 255.` that NormalizedDataset applies next.
//
// OpenCV 4.13's grey of a colour 8-bit PNG is (9797 R + 19234 G + 3737 B) >> 15: integer weights that sum to 2^15, truncated.
// It is not cv2.cvtColor(COLOR_BGR2GRAY), which rounds 14-bit weights and differs by one level on half of the colours.  The
// model and the probes that settled each constant are tests/grey_reference.py and DESIGN 5.11.
//
// One thread per group of 4 pixels of a row.  Where the group's bytes start at a multiple of 4 (the pitches and base pointers
// allow it: every group of a frame then does), they are read as 3 (BGR, RGB) or 4 (BGRA, RGBA) 32-bit words and the grey as one
// word; otherwise, and at a row's last partial group, byte by byte.  The fp32 output goes as one float4 where it is 16-byte
// aligned.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "grey.cuh"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kMaxSide = 32767;      // the crop's bounds (crop.cu): the frames this feeds
constexpr int kMaxFrames = 65535;
constexpr int kThreads = 256;
constexpr int kGroup = 4;            // pixels per thread

// Frame blockIdx.y; thread -> (row, group of kGroup pixels).  C channels per pixel, red first (RGB / RGBA) or third (BGR / BGRA).
template <int C>
__global__ void __launch_bounds__(kThreads) grey_frames_kernel(const uint8_t* __restrict__ frames, long long frame_pitch, long long row_pitch,
                                                               int H, int W, bool red_first, uint8_t* __restrict__ grey,
                                                               long long grey_frame_pitch, long long grey_row_pitch, float* __restrict__ image) {
  const int groups = (W + kGroup - 1) / kGroup;
  const long long idx = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (long long)H * groups) return;
  const int y = (int)(idx / groups), x0 = (int)(idx - (long long)y * groups) * kGroup;
  const int f = blockIdx.y;
  const uint8_t* src = frames + (size_t)f * frame_pitch + (size_t)y * row_pitch + (size_t)x0 * C;
  uint8_t* dst = grey + (size_t)f * grey_frame_pitch + (size_t)y * grey_row_pitch + x0;
  const int n = min(kGroup, W - x0);
  uint32_t g[kGroup];
  if (n == kGroup && ((uintptr_t)src & 3) == 0) {
    uint32_t w[C];                                       // the group's 4 * C bytes, little-endian: byte k of the group is byte k & 3 of w[k >> 2]
#pragma unroll
    for (int i = 0; i < C; ++i) w[i] = __ldg(reinterpret_cast<const uint32_t*>(src) + i);
#pragma unroll
    for (int p = 0; p < kGroup; ++p) {
      uint32_t c[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) c[k] = (w[(p * C + k) >> 2] >> (8 * ((p * C + k) & 3))) & 255u;
      g[p] = grey_of(c[0], c[1], c[2], red_first);
    }
  } else {
#pragma unroll
    for (int p = 0; p < kGroup; ++p)
      g[p] = p < n ? grey_of(__ldg(src + p * C), __ldg(src + p * C + 1), __ldg(src + p * C + 2), red_first) : 0u;
  }
  if (n == kGroup && ((uintptr_t)dst & 3) == 0) {
    *reinterpret_cast<uint32_t*>(dst) = g[0] | g[1] << 8 | g[2] << 16 | g[3] << 24;
  } else {
    for (int p = 0; p < n; ++p) dst[p] = (uint8_t)g[p];
  }
  if (image) {                                           // [F, 1, H, W] dense; numpy's float32 `/ 255.`, a true division
    float v[kGroup];
#pragma unroll
    for (int p = 0; p < kGroup; ++p) v[p] = __fdiv_rn((float)g[p], 255.f);
    float* out = image + ((size_t)f * H + y) * W + x0;
    if (n == kGroup && ((uintptr_t)out & 15) == 0) {
      *reinterpret_cast<float4*>(out) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
      for (int p = 0; p < n; ++p) out[p] = v[p];
    }
  }
}

}  // namespace
}  // namespace opb

extern "C" int opb_grey_frames(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t F, int32_t H, int32_t W, int32_t order,
                               uint8_t* grey, int64_t grey_frame_pitch, int64_t grey_row_pitch, float* image, void* stream) {
  REQUIRE(__func__, frames && grey);
  REQUIRE(__func__, F > 0 && F <= opb::kMaxFrames && H > 0 && H <= opb::kMaxSide && W > 0 && W <= opb::kMaxSide);
  REQUIRE(__func__, order >= OPB_ORDER_BGR && order <= OPB_ORDER_RGBA);
  const int C = order == OPB_ORDER_BGRA || order == OPB_ORDER_RGBA ? 4 : 3;
  REQUIRE(__func__, row_pitch >= (int64_t)W * C);
  REQUIRE(__func__, frame_pitch == 0 || frame_pitch >= (int64_t)H * row_pitch);
  REQUIRE(__func__, grey_row_pitch >= W && grey_frame_pitch >= (int64_t)H * grey_row_pitch);
  const bool red_first = order == OPB_ORDER_RGB || order == OPB_ORDER_RGBA;
  const long long blocks = ((long long)H * ((W + opb::kGroup - 1) / opb::kGroup) + opb::kThreads - 1) / opb::kThreads;
  const dim3 grid((unsigned)blocks, (unsigned)F);
  cudaStream_t st = (cudaStream_t)stream;
  if (C == 3)
    LAUNCH_NH(__func__, opb::grey_frames_kernel<3>, grid, opb::kThreads, 0, st, frames, frame_pitch, row_pitch, H, W, red_first, grey,
              grey_frame_pitch, grey_row_pitch, image);
  else
    LAUNCH_NH(__func__, opb::grey_frames_kernel<4>, grid, opb::kThreads, 0, st, frames, frame_pitch, row_pitch, H, W, red_first, grey,
              grey_frame_pitch, grey_row_pitch, image);
  return OPB_OK;
}
