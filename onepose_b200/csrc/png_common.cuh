// Pieces the PNG writer (png.cu) and reader (png_decode.cu) share: zlib's CRC-32 with crc32_combine (multmodp / x2nmodp) and a
// warp's CRC of one chunk, and Adler-32 from its two sums.  Both also use the block-wide scans of block.cuh.
#pragma once
#include <stdint.h>

#include "block.cuh"

namespace opb {
namespace {

// ---- CRC-32 (zlib's crc32 and crc32_combine: multmodp / x2nmodp) ----

constexpr uint32_t kPoly = 0xedb88320u;
__device__ uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}
__device__ uint32_t x2nmodp(const uint32_t* x2n, int64_t n, unsigned k) {
  uint32_t p = 1u << 31;
  while (n) {
    if (n & 1) p = multmodp(x2n[k & 31], p);
    n >>= 1;
    ++k;
  }
  return p;
}
__device__ uint32_t crc_bytes(const uint32_t* table, uint32_t crc, const uint8_t* p, int64_t n) {
  crc = ~crc;
  for (int64_t i = 0; i < n; ++i) crc = table[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
  return ~crc;
}
__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

// The CRC table and x^(2^n) mod p for n < 32, filled by one warp.
__device__ inline void crc_tables(uint32_t* table, uint32_t* x2n, int lane) {
  for (int i = lane; i < 256; i += 32) {
    uint32_t v = (uint32_t)i;
    for (int b = 0; b < 8; ++b) v = v & 1 ? (v >> 1) ^ kPoly : v >> 1;
    table[i] = v;
  }
  if (lane == 0) {
    uint32_t p = 1u << 30;                 // x^1
    x2n[0] = p;
    for (int n = 1; n < 32; ++n) x2n[n] = p = multmodp(p, p);
  }
  __syncwarp();
}

// CRC-32 of p[0 .. total) by one warp: lane l takes bytes [l * seg, (l + 1) * seg), lane 0 joins them in order by
// crc32_combine and returns the CRC (other lanes return garbage).  part holds 32 values.
__device__ inline uint32_t warp_crc(const uint32_t* table, const uint32_t* x2n, uint32_t* part, const uint8_t* p, int64_t total, int lane) {
  const int64_t seg = (total + 31) / 32;
  const int64_t b0 = min(total, lane * seg), b1 = min(total, b0 + seg);
  __syncwarp();
  part[lane] = crc_bytes(table, 0, p + b0, b1 - b0);
  __syncwarp();
  uint32_t crc = part[0];
  if (lane == 0)
    for (int l = 1; l < 32; ++l) {
      const int64_t n = min(total, (l + 1) * seg) - min(total, l * seg);
      if (n > 0) crc = multmodp(x2nmodp(x2n, n, 3), crc) ^ part[l];
    }
  __syncwarp();
  return crc;
}

// Adler-32 of n bytes from s1 = the sum of the bytes and s2 = the sum of (n - i) * byte i.
__host__ __device__ inline uint32_t adler_of_sums(unsigned long long s1, unsigned long long s2, int64_t n) {
  const unsigned long long A = (1 + s1) % 65521, B = ((unsigned long long)n % 65521 + s2 % 65521) % 65521;
  return (uint32_t)((B << 16) | A);
}

}  // namespace
}  // namespace opb
