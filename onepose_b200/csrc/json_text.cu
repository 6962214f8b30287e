// The text of the reference's per-image 2D annotation files on the GPU: save_2d_anno_for_each_image (feature_process.py:233-262)
// json.dump-s {"keypoints2d", "descriptors2d", "scores2d", "assign_matrix", "num_matches"} with json's default separators, every
// fp32 feature widened to a Python float by .tolist().
//   float_repr     float.__repr__ of the widened double: the shortest decimal that reads back as that double, the nearest one
//                  when several are shortest and the even last digit on a tie; fixed notation for decimal exponents -4 .. 15
//                  (".0" on integral values), otherwise d.ddde+XX; json's NaN / Infinity / -Infinity
//   int_repr       int.__repr__
// The digits come from Burger and Dybvig's free-format algorithm in exact 256-bit integer arithmetic: every fp32 value, widened,
// is m * 2^e with m < 2^24 and -172 <= e <= 104, so the scaled value, its neighbours' midpoints and the power of ten all fit.
// The same code runs on the host (opb_json_float_repr_host), so the rules are checked against Python without a GPU.
//
// An image's text is a run of items: item j is the glue before number j (brackets, separators and keys) and the number; the
// last item, num_matches, also closes the object.  opb_anno2d_text_lengths sizes every item and scans them per image, and
// opb_anno2d_text_write writes each item at its offset: two passes over the same item function.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string.h>

#include <cub/block/block_scan.cuh>

#include "../../include/onepose_b200.h"
#include "host_util.cuh"

namespace opb {
namespace {

#define HD __host__ __device__ __forceinline__

constexpr int kReprMax = 24;        // the longest float repr, "-1.2345678901234567e-45", and its NUL-free padding
constexpr int kItemMax = 64;        // the longest item: glue, a number and the closing brace
constexpr int kScanThreads = 1024;

HD uint64_t mul_hi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// 256-bit unsigned integers, little-endian 64-bit limbs.  No operation overflows for the values float_digits forms.
struct U256 {
  uint64_t w[4];
};
HD U256 u_from(uint64_t v) { return U256{{v, 0, 0, 0}}; }
HD void u_mul(U256& a, uint64_t m) {
  uint64_t carry = 0;
  for (int i = 0; i < 4; ++i) {
    const uint64_t lo = a.w[i] * m, hi = mul_hi(a.w[i], m);
    a.w[i] = lo + carry;
    carry = hi + (a.w[i] < lo);
  }
}
HD void u_shl(U256& a, int s) {        // 0 <= s < 256
  const int q = s >> 6, r = s & 63;
  for (int i = 3; i >= 0; --i) {
    uint64_t v = i - q >= 0 ? a.w[i - q] << r : 0;
    if (r && i - q - 1 >= 0) v |= a.w[i - q - 1] >> (64 - r);
    a.w[i] = v;
  }
}
HD int u_cmp(const U256& a, const U256& b) {
  for (int i = 3; i >= 0; --i)
    if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
  return 0;
}
HD U256 u_add(const U256& a, const U256& b) {
  U256 c;
  uint64_t carry = 0;
  for (int i = 0; i < 4; ++i) {
    const uint64_t s = a.w[i] + b.w[i];
    c.w[i] = s + carry;
    carry = (s < a.w[i]) | (c.w[i] < s);
  }
  return c;
}
HD void u_sub(U256& a, const U256& b) {        // a >= b
  uint64_t borrow = 0;
  for (int i = 0; i < 4; ++i) {
    const uint64_t d = a.w[i] - b.w[i];
    const uint64_t nb = (a.w[i] < b.w[i]) | (d < borrow);
    a.w[i] = d - borrow;
    borrow = nb;
  }
}
HD void u_pow10(U256& a, int k) {      // a *= 10^k, k >= 0
  for (; k >= 19; k -= 19) u_mul(a, 10000000000000000000ull);
  uint64_t p = 1;
  for (; k > 0; --k) p *= 10;
  u_mul(a, p);
}

// The shortest digits of |x| widened to a double (x finite, nonzero): x = 0.d1 d2 .. dn * 10^k.  Returns n (<= 17).
// Burger and Dybvig's free format with both ends of the rounding interval included: a widened fp32 value has an even double
// significand, so round-half-even reads either end back as x.
HD int float_digits(float x, char* dig, int* k_out) {
  uint32_t b;
  memcpy(&b, &x, 4);
  b &= 0x7fffffffu;
  uint32_t m = b & 0x7fffffu;
  int e = (int)(b >> 23);
  if (e == 0) e = -149;                 // subnormal: m * 2^-149
  else {
    m |= 0x800000u;
    e -= 150;
  }
  while (m < 0x800000u) {               // m in [2^23, 2^24): the double's significand is m * 2^29
    m <<= 1;
    --e;
  }
  // In units of 2^(e - 31): x = m * 2^31, the gap to the midpoint above is 2 (half the double's ulp 2^(e - 29)), and 1 below a
  // power of two, where the double below is half as far.
  U256 r = u_from((uint64_t)m << 31), mp = u_from(2), mm = u_from(m == 0x800000u ? 1 : 2), s = u_from(1);
  const int se = e - 31;
  if (se >= 0) {
    u_shl(r, se);
    u_shl(mp, se);
    u_shl(mm, se);
  } else {
    u_shl(s, -se);
  }
  // floor((e + 23) log10 2) <= floor(log10 x); the loop below raises k to the first power of ten above the interval
  int k = ((e + 23) * 78913) >> 18;
  if (k >= 0) u_pow10(s, k);
  else {
    u_pow10(r, -k);
    u_pow10(mp, -k);
    u_pow10(mm, -k);
  }
  while (u_cmp(u_add(r, mp), s) >= 0) {
    u_mul(s, 10);
    ++k;
  }
  int n = 0;
  for (;;) {
    u_mul(r, 10);
    u_mul(mp, 10);
    u_mul(mm, 10);
    int d = 0;
    while (u_cmp(r, s) >= 0) {
      u_sub(r, s);
      ++d;
    }
    const bool low = u_cmp(r, mm) <= 0;
    const bool high = u_cmp(u_add(r, mp), s) >= 0;
    if (!low && !high) {
      dig[n++] = (char)('0' + d);
      continue;
    }
    if (low && high) {
      U256 r2 = r;
      u_shl(r2, 1);
      const int c = u_cmp(r2, s);
      if (c > 0 || (c == 0 && (d & 1))) ++d;
    } else if (high) {
      ++d;
    }
    dig[n++] = (char)('0' + d);
    break;
  }
  *k_out = k;
  return n;
}

HD int put(char* out, const char* s) {
  int n = 0;
  for (; s[n]; ++n) out[n] = s[n];
  return n;
}

// float.__repr__ of (double)x as json.dump writes it; returns the length (<= 23).
HD int float_repr(float x, char* out) {
  uint32_t b;
  memcpy(&b, &x, 4);
  const bool neg = b >> 31;
  const uint32_t a = b & 0x7fffffffu;
  if (a > 0x7f800000u) return put(out, "NaN");
  if (a == 0x7f800000u) return put(out, neg ? "-Infinity" : "Infinity");
  if (a == 0) return put(out, neg ? "-0.0" : "0.0");
  int len = 0;
  if (neg) out[len++] = '-';
  char dig[20];
  int k;
  const int n = float_digits(x, dig, &k);
  const int e10 = k - 1;                // decimal exponent of the first digit
  if (e10 >= -4 && e10 < 16) {
    if (e10 >= 0) {
      for (int i = 0; i <= e10; ++i) out[len++] = i < n ? dig[i] : '0';
      out[len++] = '.';
      if (n <= e10 + 1) out[len++] = '0';
      for (int i = e10 + 1; i < n; ++i) out[len++] = dig[i];
    } else {
      out[len++] = '0';
      out[len++] = '.';
      for (int i = 0; i < -e10 - 1; ++i) out[len++] = '0';
      for (int i = 0; i < n; ++i) out[len++] = dig[i];
    }
  } else {
    out[len++] = dig[0];
    if (n > 1) {
      out[len++] = '.';
      for (int i = 1; i < n; ++i) out[len++] = dig[i];
    }
    out[len++] = 'e';
    out[len++] = e10 < 0 ? '-' : '+';
    const int ae = e10 < 0 ? -e10 : e10;   // <= 45: two digits
    out[len++] = (char)('0' + ae / 10);
    out[len++] = (char)('0' + ae % 10);
  }
  return len;
}

// int.__repr__; returns the length (<= 20).
HD int int_repr(int64_t v, char* out) {
  char t[20];
  uint64_t u = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
  int n = 0;
  do {
    t[n++] = (char)('0' + u % 10);
    u /= 10;
  } while (u);
  int len = 0;
  if (v < 0) out[len++] = '-';
  while (n) out[len++] = t[--n];
  return len;
}

// The per-image inputs of a chunk: image c of the chunk is row img[c] of the features, with n[c] features and k[c] pairs at
// columns pair_off[c] .. of the pairs [2, pair_stride].
struct Anno2dImages {
  const int64_t* desc;                  // [Fc, 4]: feature row, n, k, pair offset
  const int64_t* item_off;              // [Fc + 1]: the first item of each image in the chunk's item arrays
  int D, cap;
  const float* keypoints;               // [F, cap, 2]
  const float* descriptors;             // [F, D, cap]
  const float* scores;                  // [F, cap]
  const int64_t* pairs;                 // [2, pair_stride]
  int64_t pair_stride;
};

// Item j of chunk image c: its glue and number, written to buf; returns the length (<= kItemMax).
__device__ int anno2d_item(const Anno2dImages& a, int c, int64_t j, char* buf) {
  const int64_t f = a.desc[c * 4], n = a.desc[c * 4 + 1], k = a.desc[c * 4 + 2], po = a.desc[c * 4 + 3];
  int len;
  if (j < 2 * n) {
    len = put(buf, j == 0 ? "{\"keypoints2d\": [[" : (j & 1) ? ", " : "], [");
    return len + float_repr(a.keypoints[(f * a.cap + (j >> 1)) * 2 + (j & 1)], buf + len);
  }
  j -= 2 * n;
  if (j < (int64_t)a.D * n) {
    const int64_t d = j / n, i = j % n;
    len = put(buf, j == 0 ? "]], \"descriptors2d\": [[" : i == 0 ? "], [" : ", ");
    return len + float_repr(a.descriptors[(f * a.D + d) * a.cap + i], buf + len);
  }
  j -= (int64_t)a.D * n;
  if (j < n) {
    len = put(buf, j == 0 ? "]], \"scores2d\": [[" : "], [");
    return len + float_repr(a.scores[f * a.cap + j], buf + len);
  }
  j -= n;
  if (j < 2 * k) {
    const int64_t row = j / k, i = j % k;
    len = put(buf, j == 0 ? "]], \"assign_matrix\": [[" : i == 0 ? "], [" : ", ");
    return len + int_repr(a.pairs[row * a.pair_stride + po + i], buf + len);
  }
  len = put(buf, "]], \"num_matches\": ");
  len += int_repr(k, buf + len);
  buf[len++] = '}';
  return len;
}

// blockIdx.y = chunk image, threads stride over its items: each item's length
__global__ void anno2d_lengths_kernel(Anno2dImages a, int32_t* __restrict__ pos) {
  const int c = blockIdx.y;
  const int64_t first = a.item_off[c], items = a.item_off[c + 1] - first;
  char buf[kItemMax];
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < items; j += (int64_t)gridDim.x * blockDim.x)
    pos[first + j] = anno2d_item(a, c, j, buf);
}

// One block per chunk image: its lengths become in-image offsets in place (an exclusive scan), and its length goes to len[c].
__global__ void __launch_bounds__(kScanThreads) anno2d_scan_kernel(const int64_t* __restrict__ item_off, int32_t* __restrict__ pos,
                                                                   int64_t* __restrict__ len) {
  using Scan = cub::BlockScan<int32_t, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int c = blockIdx.x;
  const int64_t first = item_off[c], items = item_off[c + 1] - first;
  int32_t base = 0;                     // an image's text is below 2^31 bytes (the entry bounds its items)
  for (int64_t t0 = 0; t0 < items; t0 += kScanThreads) {
    const int64_t j = t0 + threadIdx.x;
    const int32_t v = j < items ? pos[first + j] : 0;
    int32_t x, total;
    Scan(tmp).ExclusiveSum(v, x, total);
    if (j < items) pos[first + j] = base + x;
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) len[c] = base;
}

// offsets[0 .. Fc]: the exclusive sum of the image lengths (Fc is small: one thread)
__global__ void anno2d_offsets_kernel(const int64_t* __restrict__ len, int Fc, int64_t* __restrict__ offsets) {
  int64_t s = 0;
  for (int c = 0; c < Fc; ++c) {
    offsets[c] = s;
    s += len[c];
  }
  offsets[Fc] = s;
}

__global__ void anno2d_write_kernel(Anno2dImages a, const int32_t* __restrict__ pos, const int64_t* __restrict__ offsets,
                                    char* __restrict__ out) {
  const int c = blockIdx.y;
  const int64_t first = a.item_off[c], items = a.item_off[c + 1] - first;
  char buf[kItemMax];
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < items; j += (int64_t)gridDim.x * blockDim.x) {
    const int len = anno2d_item(a, c, j, buf);
    char* dst = out + offsets[c] + pos[first + j];
    for (int i = 0; i < len; ++i) dst[i] = buf[i];
  }
}

__global__ void float_repr_kernel(const float* __restrict__ x, int64_t n, char* __restrict__ out, int32_t* __restrict__ len) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  char buf[kReprMax];
  const int l = float_repr(x[i], buf);
  for (int t = 0; t < kReprMax; ++t) out[i * kReprMax + t] = t < l ? buf[t] : 0;
  len[i] = l;
}

// Grid of the item kernels: enough blocks for the largest image, at most 4096 per image.
dim3 item_grid(int64_t max_items, int Fc) {
  return dim3((unsigned)std::min<int64_t>((max_items + 255) / 256, 4096), (unsigned)Fc);
}

int check_images(const char* fn, const int64_t* desc, const int64_t* item_off, int32_t Fc, int64_t max_items, int32_t D, int32_t cap,
                 const float* keypoints, const float* descriptors, const float* scores, const int64_t* pairs, int64_t pair_stride,
                 void* workspace, int64_t workspace_bytes) {
  REQUIRE(fn, desc && item_off && keypoints && descriptors && scores && pairs && workspace);
  REQUIRE(fn, Fc > 0 && Fc <= 65535 && D > 0 && cap > 0 && pair_stride > 0);
  REQUIRE(fn, max_items > 0 && max_items <= OPB_ANNO2D_MAX_IMAGE_ITEMS);
  REQUIRE(fn, workspace_bytes >= 0);
  return OPB_OK;
}

}  // namespace
}  // namespace opb

extern "C" int opb_json_float_repr(const float* x, int64_t n, char* out, int32_t* len, void* stream) {
  REQUIRE(__func__, n >= 0 && (n == 0 || (x && out && len)));
  if (n > 0)
    LAUNCH_NH(__func__, opb::float_repr_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, x, n, out, len);
  return OPB_OK;
}

extern "C" int opb_json_float_repr_host(const float* x, int64_t n, char* out, int32_t* len) {
  REQUIRE(__func__, n >= 0 && (n == 0 || (x && out && len)));
  for (int64_t i = 0; i < n; ++i) {
    char buf[opb::kReprMax];
    const int l = opb::float_repr(x[i], buf);
    for (int t = 0; t < opb::kReprMax; ++t) out[i * opb::kReprMax + t] = t < l ? buf[t] : 0;
    len[i] = l;
  }
  return OPB_OK;
}

extern "C" int opb_anno2d_text_workspace_bytes(int32_t Fc, int64_t items, int64_t* bytes) {
  REQUIRE(__func__, bytes && Fc > 0 && items > 0);
  *bytes = (int64_t)(((size_t)items * 4 + 255) / 256 * 256 + (size_t)Fc * 8);
  return OPB_OK;
}

extern "C" int opb_anno2d_text_lengths(const int64_t* images, const int64_t* item_off, int32_t Fc, int64_t items, int64_t max_items,
                                       int32_t D, int32_t cap, const float* keypoints, const float* descriptors, const float* scores,
                                       const int64_t* pairs, int64_t pair_stride, void* workspace, int64_t workspace_bytes,
                                       int64_t* offsets, void* stream) {
  if (int rc = opb::check_images(__func__, images, item_off, Fc, max_items, D, cap, keypoints, descriptors, scores, pairs, pair_stride,
                                 workspace, workspace_bytes))
    return rc;
  REQUIRE(__func__, offsets && items > 0 && items >= max_items);
  const size_t pos_bytes = ((size_t)items * 4 + 255) / 256 * 256;
  REQUIRE(__func__, workspace_bytes >= (int64_t)(pos_bytes + (size_t)Fc * 8));
  int32_t* pos = (int32_t*)workspace;
  int64_t* len = (int64_t*)((char*)workspace + pos_bytes);
  const opb::Anno2dImages a{images, item_off, D, cap, keypoints, descriptors, scores, pairs, pair_stride};
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH_NH(__func__, opb::anno2d_lengths_kernel, opb::item_grid(max_items, Fc), 256, 0, st, a, pos);
  LAUNCH_NH(__func__, opb::anno2d_scan_kernel, (unsigned)Fc, opb::kScanThreads, 0, st, item_off, pos, len);
  LAUNCH_NH(__func__, opb::anno2d_offsets_kernel, 1, 1, 0, st, (const int64_t*)len, (int)Fc, offsets);
  return OPB_OK;
}

extern "C" int opb_anno2d_text_write(const int64_t* images, const int64_t* item_off, int32_t Fc, int64_t max_items, int32_t D, int32_t cap,
                                     const float* keypoints, const float* descriptors, const float* scores, const int64_t* pairs,
                                     int64_t pair_stride, const void* workspace, const int64_t* offsets, char* out, void* stream) {
  if (int rc = opb::check_images(__func__, images, item_off, Fc, max_items, D, cap, keypoints, descriptors, scores, pairs, pair_stride,
                                 (void*)workspace, 0))
    return rc;
  REQUIRE(__func__, offsets && out);
  const opb::Anno2dImages a{images, item_off, D, cap, keypoints, descriptors, scores, pairs, pair_stride};
  LAUNCH_NH(__func__, opb::anno2d_write_kernel, opb::item_grid(max_items, Fc), 256, 0, (cudaStream_t)stream, a, (const int32_t*)workspace,
            offsets, out);
  return OPB_OK;
}
