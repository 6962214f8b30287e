// OpenCV 4.13's IMREAD_GRAYSCALE of a colour 8-bit PNG, shared by the frame conversion (frames.cu) and the PNG reader
// (png_decode.cu): (9797 R + 19234 G + 3737 B) >> 15, integer weights that sum to 2^15, truncated.  The model and the probes that
// settled each constant are tests/grey_reference.py and DESIGN 5.11.
#pragma once
#include <stdint.h>

namespace opb {

__device__ __forceinline__ uint32_t grey_of(uint32_t c0, uint32_t c1, uint32_t c2, bool red_first) {
  const uint32_t r = red_first ? c0 : c2, b = red_first ? c2 : c0;
  return (9797u * r + 19234u * c1 + 3737u * b) >> 15;
}

}  // namespace opb
