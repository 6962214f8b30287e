// PNG files of 8-bit frames as cv2.imencode('.png', frame) (OpenCV 4.13, libpng, zlib 1.3) writes them, byte for byte, for F frames
// of one shape in one call (parse_scanned_data.py:173, :177, :264-273).  The rules -- SUB rows (NONE at width 1), deflate level 1
// with Z_RLE at memLevel 8, libpng's window and header choice, IDAT chunks of 8192 bytes -- and the decomposition are DESIGN §5.15;
// the model and the numpy emulation of these kernels are tests/png_reference.py.
//
//   png_filter_kernel   tiles of 4096 filtered bytes: filter byte, SUB difference and channel swap read straight from the frames,
//                       Adler-32's two sums, and each tile's first and last run head
//   png_carry_kernel    per frame: the last run head before each tile and the first after it (max / min scans over tiles)
//   png_tokens_kernel   tiles again: deflate_rle's greedy distance-1 tokens from each byte's run, counted, then (second launch)
//                       written at their index after a scan of the tile counts (png_scan_kernel), with each block's first byte
//   png_tree_kernel     one CTA per deflate block of 16383 symbols: histograms, then one thread for zlib's build_tree (heap with
//                       the depth tie-break, gen_bitlen's repair, gen_codes), scan_tree / send_tree and the stored / fixed /
//                       dynamic choice; the dynamic header goes to the block's record as a bit string
//   png_offsets_kernel  per frame: each block's bit offset (stored blocks byte-aligned), the stream length and the file size
//   png_pack_kernel     one CTA per block: token bit offsets by a block scan, bits OR-ed into the zeroed stream
//   png_frame_kernel    one warp per IDAT chunk: the chunk's bytes and its CRC-32 (per-lane CRCs joined by crc32_combine);
//                       signature, IHDR and IEND by the first and last chunk's warps
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "host_util.cuh"
#include "png_common.cuh"

namespace opb {
namespace {

constexpr int kTile = 4096;                 // filtered bytes per tile
constexpr int kTileThreads = 256;
constexpr int kPerThread = kTile / kTileThreads;
constexpr int kBlockSymbols = 16383;        // zlib's sym_end at memLevel 8
constexpr int kChunk = 8192;                // libpng's IDAT size (PNG_ZBUF_SIZE)
constexpr int kHdrBytes = 640;              // the longest dynamic header: 14 + 57 + 316 * 14 bits
constexpr int kScanThreads = 1024;
constexpr int kPackThreads = 256;
constexpr int64_t kMaxFiltered = 1ll << 28;  // Adler-32's second sum stays in 64 bits

enum { kStored = 0, kFixed = 1, kDynamic = 2 };

struct Block {                               // one deflate block's record
  int32_t type, stored_len, start, hdr_bits;
  int64_t bits;                              // fixed / dynamic: the block's bits with its 3 type bits
  int64_t off;                               // bit offset in the zlib stream
  uint16_t lcode[286];
  uint8_t llen[286];
  uint16_t dcode0;
  uint8_t dlen0, pad_;
  uint8_t hdr[kHdrBytes];
};

struct Frame {                               // per frame
  unsigned long long s1, s2;                 // Adler-32: sum of bytes, sum of (n - i) * byte
  int32_t tokens;
  int32_t pad_;
  int64_t zlen;                              // zlib stream bytes; -1: does not fit its slot
};

__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct PngLayout {
  int64_t n, nt, nb, zcap;                   // filtered bytes, tiles, block records and stream capacity per frame
  size_t filt, tok, tile, blk, frame, zbuf, total;   // byte offsets in the workspace
};

// zlib 1.3's deflateBound for this stream (level 1, memLevel 8, the window below).
__host__ __device__ inline int64_t window_bits(int64_t n) {
  int wb = 15;
  if (n <= 16384) {
    int64_t half = 1 << 14;
    while (n + 262 <= half) half >>= 1, --wb;
  }
  return wb < 9 ? 9 : wb;
}
__host__ __device__ inline int64_t deflate_bound(int64_t n) {
  if (window_bits(n) == 15) return n + (n >> 12) + (n >> 14) + (n >> 25) + 13;
  return n + (n >> 3) + (n >> 8) + (n >> 9) + 4 + 6;
}
__host__ __device__ inline int64_t png_bound(int64_t n) {
  const int64_t z = deflate_bound(n);
  return z + 12 * ((z + kChunk - 1) / kChunk) + 45;
}

PngLayout layout(int F, int64_t n) {
  PngLayout L;
  L.n = n;
  L.nt = (n + kTile - 1) / kTile;
  L.nb = n / kBlockSymbols + 1;
  L.zcap = (int64_t)align256((size_t)deflate_bound(n) + 8);
  size_t o = 0;
  L.filt = o; o += align256((size_t)F * align256((size_t)n));
  L.tok = o; o += align256((size_t)F * n * 2);
  L.tile = o; o += align256((size_t)F * L.nt * 4) * 4;
  L.blk = o; o += align256((size_t)F * L.nb * sizeof(Block));
  L.frame = o; o += align256((size_t)F * sizeof(Frame));
  L.zbuf = o; o += (size_t)F * L.zcap;
  L.total = o;
  return L;
}

struct Args {
  const uint8_t* frames;
  int64_t frame_pitch, row_pitch;
  int H, W, C;
  int64_t n, row;                            // filtered bytes per frame and per row (1 + W C)
  int64_t nt, nb, zcap, fstride;             // fstride: filtered bytes' stride per frame
  uint8_t* filt;
  uint16_t* tok;
  int32_t *tile_first, *tile_last, *tile_count, *tile_off;   // tile_first / tile_last become the carries
  Block* blk;
  Frame* fr;
  uint8_t* zbuf;
};

// ---- filtering ----

__device__ __forceinline__ uint8_t filtered_byte(const Args& a, const uint8_t* src, int64_t i) {
  const int64_t y = i / a.row, j = i - y * a.row;
  if (j == 0) return a.W > 1 ? 1 : 0;
  const int b = (int)(j - 1), x = b / a.C, ch = b - x * a.C;
  const int sc = (a.C >= 3 && ch < 3) ? 2 - ch : ch;          // BGR(A) is stored as RGB(A)
  const uint8_t* p = src + y * a.row_pitch + (int64_t)x * a.C + sc;
  return a.W > 1 && x > 0 ? (uint8_t)(p[0] - p[-a.C]) : p[0];
}

__global__ void __launch_bounds__(kTileThreads) png_filter_kernel(Args a) {
  __shared__ unsigned long long sh64[32];
  __shared__ int32_t sh32[32];
  const int f = blockIdx.y;
  const int64_t t = blockIdx.x, base = t * kTile;
  const uint8_t* src = a.frames + f * a.frame_pitch;
  uint8_t* out = a.filt + f * a.fstride;
  unsigned long long s1 = 0, s2 = 0;
  int32_t first = (int32_t)a.n, last = -1;
  for (int k = 0; k < kPerThread; ++k) {
    const int64_t i = base + k * kTileThreads + threadIdx.x;
    if (i >= a.n) break;
    const uint8_t v = filtered_byte(a, src, i);
    out[i] = v;
    s1 += v;
    s2 += (unsigned long long)(a.n - i) * v;
    if (i == 0 || filtered_byte(a, src, i - 1) != v) {
      first = min(first, (int32_t)i);
      last = max(last, (int32_t)i);
    }
  }
  s1 = block_reduce(s1, Sum64(), sh64);
  s2 = block_reduce(s2, Sum64(), sh64);
  first = block_reduce(first, Min(), sh32);
  last = block_reduce(last, Max(), sh32);
  if (threadIdx.x == 0) {
    atomicAdd(&a.fr[f].s1, s1);
    atomicAdd(&a.fr[f].s2, s2);
    a.tile_first[f * a.nt + t] = first;
    a.tile_last[f * a.nt + t] = last;
  }
}

// Per frame: tile_last[t] becomes the last run head before tile t (exclusive max scan), tile_first[t] the first after it
// (exclusive min scan from the end, n when none).
__global__ void __launch_bounds__(kScanThreads) png_carry_kernel(Args a) {
  __shared__ int32_t sh[32];
  const int f = blockIdx.x;
  int32_t* last = a.tile_last + f * a.nt;
  int32_t* first = a.tile_first + f * a.nt;
  int32_t carry = -1, tot;
  for (int64_t c = 0; c < a.nt; c += kScanThreads) {
    const int64_t t = c + threadIdx.x;
    const int32_t exc = block_scan(t < a.nt ? last[t] : -1, Max(), -1, sh, &tot);
    if (t < a.nt) last[t] = max(carry, exc);
    carry = max(carry, tot);
  }
  carry = (int32_t)a.n;
  for (int64_t c = ((a.nt - 1) / kScanThreads) * kScanThreads; c >= 0; c -= kScanThreads) {
    const int64_t t = c + threadIdx.x;
    const int32_t exc = block_scan(t < a.nt ? first[t] : (int32_t)a.n, Min(), (int32_t)a.n, sh, &tot, true);
    if (t < a.nt) first[t] = min(carry, exc);
    carry = min(carry, tot);
  }
}

// deflate_rle's token starting at byte i of a run [s, e): 0 when i starts none, else its length (1: literal).  The run's first
// byte is a literal; the e - s - 1 repeats are matches of 258 while 258 remain, then one match of the rest if it is 3 or more,
// else literals.
__device__ __forceinline__ int token_at(int32_t i, int32_t s, int32_t e) {
  const int32_t k = i - s;
  if (k == 0) return 1;
  const int32_t r = e - s - 1, q = r / 258, m = r - q * 258, j = k - 1, c = j / 258, t = j - c * 258;
  if (c < q) return t == 0 ? 258 : 0;
  if (m >= 3) return t == 0 ? m : 0;
  return 1;
}

// Tiles of the filtered stream, kPerThread consecutive bytes per thread.  emit = false: each tile's token count; emit = true:
// the tokens at their index (tile_off + the in-tile scan) and each block's first byte.
template <bool emit>
__global__ void __launch_bounds__(kTileThreads) png_tokens_kernel(Args a) {
  __shared__ int32_t sh[32];
  const int f = blockIdx.y;
  const int64_t t = blockIdx.x, base = t * kTile;
  const uint8_t* s = a.filt + f * a.fstride;
  const int64_t p0 = base + (int64_t)threadIdx.x * kPerThread;
  const int64_t left = a.n - p0;
  const int cnt = left <= 0 ? 0 : left < kPerThread ? (int)left : kPerThread;
  uint8_t b[kPerThread + 1];
  for (int k = 0; k < kPerThread + 1; ++k) b[k] = (k < cnt + 1 && p0 + k < a.n) ? s[p0 + k] : 0;
  const uint8_t before = p0 > 0 && p0 < a.n ? s[p0 - 1] : 0;
  int32_t my_last = -1, my_next = (int32_t)a.n;             // last head in my bytes; first head after my first byte
  for (int k = 0; k < cnt; ++k)
    if (p0 + k == 0 || b[k] != (k ? b[k - 1] : before)) my_last = (int32_t)(p0 + k);
  for (int k = cnt - 1; k >= 0; --k)
    if (p0 + k + 1 < a.n && b[k + 1] != b[k]) my_next = (int32_t)(p0 + k + 1);
  int32_t tot;
  const int32_t run_in = max(a.tile_last[f * a.nt + t], block_scan(my_last, Max(), -1, sh, &tot));
  const int32_t run_out = min(a.tile_first[f * a.nt + t], block_scan(my_next, Min(), (int32_t)a.n, sh, &tot, true));
  // each byte's run [start, end) and token
  int32_t start = run_in, n_tok = 0;
  int32_t ends[kPerThread];
  {
    int32_t e = run_out;
    for (int k = cnt - 1; k >= 0; --k) {
      if (p0 + k + 1 < a.n && b[k + 1] != b[k]) e = (int32_t)(p0 + k + 1);
      ends[k] = e;
    }
  }
  int lens[kPerThread];
  for (int k = 0; k < cnt; ++k) {
    const int32_t i = (int32_t)(p0 + k);
    if (i == 0 || b[k] != (k ? b[k - 1] : before)) start = i;
    lens[k] = token_at(i, start, ends[k]);
    n_tok += lens[k] != 0;
  }
  const int32_t exc = block_scan(n_tok, Sum32(), 0, sh, &tot);
  if (!emit) {
    if (threadIdx.x == 0) a.tile_count[f * a.nt + t] = tot;
    return;
  }
  int32_t idx = a.tile_off[f * a.nt + t] + exc;
  uint16_t* tok = a.tok + (int64_t)f * a.n;
  Block* blk = a.blk + (int64_t)f * a.nb;
  for (int k = 0; k < cnt; ++k) {
    if (!lens[k]) continue;
    tok[idx] = lens[k] >= 3 ? (uint16_t)(256 + lens[k] - 3) : b[k];
    if (idx % kBlockSymbols == 0) blk[idx / kBlockSymbols].start = (int32_t)(p0 + k);
    ++idx;
  }
}

__global__ void __launch_bounds__(kScanThreads) png_scan_kernel(Args a) {
  __shared__ int32_t sh[32];
  const int f = blockIdx.x;
  const int32_t* cnt = a.tile_count + f * a.nt;
  int32_t* off = a.tile_off + f * a.nt;
  int32_t carry = 0;
  for (int64_t c = 0; c < a.nt; c += kScanThreads) {
    const int64_t t = c + threadIdx.x;
    const int32_t v = t < a.nt ? cnt[t] : 0;
    int32_t tot;
    const int32_t exc = block_scan(v, Sum32(), 0, sh, &tot);
    if (t < a.nt) off[t] = carry + exc;
    carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) a.fr[f].tokens = carry;
}

// ---- zlib's trees (trees.c), one thread ----

__constant__ uint8_t kExtraL[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t kExtraD[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kExtraBl[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ uint8_t kBlOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ uint8_t kBaseLength[29] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 255};

__device__ __forceinline__ int length_code(int lc) {      // zlib's _length_code of length - 3
  if (lc == 255) return 28;
  int c = 0;
  while (c < 27 && kBaseLength[c + 1] <= lc) ++c;
  return c;
}
__device__ __forceinline__ int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }

constexpr int kHeap = 2 * 286 + 1;

struct TreeSmem {
  uint32_t freq[kHeap];
  uint16_t dad[kHeap], heap[kHeap];
  uint8_t depth[kHeap], len[kHeap];
  uint16_t bl_count[16];
  uint32_t lfreq[286];
  uint8_t llen[288], dlen[31], bllen[19];
  uint16_t lcode[288];
  uint32_t blfreq[19];
  uint16_t blcode[19];
  int32_t matches;
};

__device__ void pqdownheap(TreeSmem& S, int heap_len, int k) {
  const int v = S.heap[k];
  int j = k << 1;
  while (j <= heap_len) {
    if (j < heap_len && (S.freq[S.heap[j + 1]] < S.freq[S.heap[j]] ||
                         (S.freq[S.heap[j + 1]] == S.freq[S.heap[j]] && S.depth[S.heap[j + 1]] <= S.depth[S.heap[j]])))
      ++j;
    if (S.freq[v] < S.freq[S.heap[j]] || (S.freq[v] == S.freq[S.heap[j]] && S.depth[v] <= S.depth[S.heap[j]])) break;
    S.heap[k] = S.heap[j];
    k = j;
    j <<= 1;
  }
  S.heap[k] = (uint16_t)v;
}

// build_tree + gen_bitlen over freq[0 .. elems) (in S.freq): lengths into out_len, returns max_code; adds to opt / stat.
// kind 0: literal/length (static lengths, extra from 257), 1: distance (static 5, extra from 0), 2: bit lengths (no static).
__device__ int build_tree(TreeSmem& S, int elems, int kind, uint8_t* out_len, int64_t& opt, int64_t& stat) {
  const int max_length = kind == 2 ? 7 : 15;
  int heap_len = 0, heap_max = kHeap, max_code = -1;
  for (int n = 0; n < elems; ++n) {
    S.depth[n] = 0;
    if (S.freq[n]) S.heap[++heap_len] = (uint16_t)(max_code = n);
  }
  while (heap_len < 2) {
    const int node = max_code < 2 ? ++max_code : 0;
    S.heap[++heap_len] = (uint16_t)node;
    S.freq[node] = 1;
    S.depth[node] = 0;
    opt -= 1;
    if (kind == 0) stat -= static_llen(node);
    if (kind == 1) stat -= 5;
  }
  for (int n = heap_len / 2; n >= 1; --n) pqdownheap(S, heap_len, n);
  int node = elems;
  do {
    const int n = S.heap[1];
    S.heap[1] = S.heap[heap_len--];
    pqdownheap(S, heap_len, 1);
    const int m = S.heap[1];
    S.heap[--heap_max] = (uint16_t)n;
    S.heap[--heap_max] = (uint16_t)m;
    S.freq[node] = S.freq[n] + S.freq[m];
    S.depth[node] = (uint8_t)((S.depth[n] >= S.depth[m] ? S.depth[n] : S.depth[m]) + 1);
    S.dad[n] = S.dad[m] = (uint16_t)node;
    S.heap[1] = (uint16_t)node++;
    pqdownheap(S, heap_len, 1);
  } while (heap_len >= 2);
  S.heap[--heap_max] = S.heap[1];
  // gen_bitlen
  for (int b = 0; b < 16; ++b) S.bl_count[b] = 0;
  S.len[S.heap[heap_max]] = 0;
  int overflow = 0, h;
  for (h = heap_max + 1; h < kHeap; ++h) {
    const int n = S.heap[h];
    int bits = S.len[S.dad[n]] + 1;
    if (bits > max_length) bits = max_length, ++overflow;
    S.len[n] = (uint8_t)bits;
    if (n > max_code) continue;
    S.bl_count[bits]++;
    int xbits = 0;
    if (kind == 0 && n >= 257) xbits = kExtraL[n - 257];
    if (kind == 1) xbits = kExtraD[n];
    if (kind == 2) xbits = kExtraBl[n];
    opt += (int64_t)S.freq[n] * (bits + xbits);
    if (kind == 0) stat += (int64_t)S.freq[n] * (static_llen(n) + xbits);
    if (kind == 1) stat += (int64_t)S.freq[n] * (5 + xbits);
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (S.bl_count[bits] == 0) --bits;
      S.bl_count[bits]--;
      S.bl_count[bits + 1] += 2;
      S.bl_count[max_length]--;
      overflow -= 2;
    } while (overflow > 0);
    h = kHeap;
    for (int bits = max_length; bits != 0; --bits) {
      int n = S.bl_count[bits];
      while (n != 0) {
        const int m = S.heap[--h];
        if (m > max_code) continue;
        if (S.len[m] != bits) {
          opt += ((int64_t)bits - S.len[m]) * S.freq[m];
          S.len[m] = (uint8_t)bits;
        }
        --n;
      }
    }
  }
  for (int n = 0; n < elems; ++n) out_len[n] = (n <= max_code && S.freq[n]) ? S.len[n] : 0;
  return max_code;
}

// gen_codes: canonical codes of lens[0 .. n), bit-reversed for LSB-first output.
__device__ void gen_codes(const uint8_t* lens, int n, uint16_t* codes) {
  uint16_t count[16] = {0}, next[16];
  for (int i = 0; i < n; ++i) count[lens[i]]++;
  count[0] = 0;
  unsigned code = 0;
  for (int b = 1; b < 16; ++b) next[b] = (uint16_t)(code = (code + count[b - 1]) << 1);
  for (int i = 0; i < n; ++i)
    if (lens[i]) codes[i] = (uint16_t)(__brev(next[lens[i]]++) >> (32 - lens[i]));
}

// scan_tree (send = false: bit-length frequencies) and send_tree (send = true: items into the bit writer) of lens[0 .. max_code].
struct BitWriter {
  uint8_t* out;
  int bits;
  unsigned long long acc;
  int nacc;
  __device__ void put(unsigned v, int n) {
    acc |= (unsigned long long)v << nacc;
    nacc += n;
    bits += n;
    while (nacc >= 8) *out++ = (uint8_t)acc, acc >>= 8, nacc -= 8;
  }
  __device__ void flush() {
    if (nacc) *out++ = (uint8_t)acc;
  }
};

template <bool send>
__device__ void tree_runs(TreeSmem& S, const uint8_t* lens, int max_code, BitWriter* w) {
  int prevlen = -1, nextlen = lens[0], count = 0, max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  auto item = [&](int sym, int xv, int xb) {
    if (send) {
      w->put(S.blcode[sym], S.bllen[sym]);
      if (xb) w->put((unsigned)xv, xb);
    } else {
      S.blfreq[sym]++;
    }
  };
  for (int n = 0; n <= max_code; ++n) {
    const int curlen = nextlen;
    nextlen = n + 1 <= max_code ? lens[n + 1] : 0xffff;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      for (; count; --count) item(curlen, 0, 0);
    } else if (curlen != 0) {
      if (curlen != prevlen) item(curlen, 0, 0), --count;
      item(16, count - 3, 2);
    } else if (count <= 10) {
      item(17, count - 3, 3);
    } else {
      item(18, count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

// One CTA per block record; blocks past the frame's count return.  _tr_flush_block's choice: stored when stored_len + 4 <=
// min(opt, static) bytes (always in zlib's window: DESIGN §5.15), else fixed when static <= opt, else dynamic.
__global__ void __launch_bounds__(256) png_tree_kernel(Args a) {
  __shared__ TreeSmem S;
  const int f = blockIdx.y, k = blockIdx.x;
  const int32_t T = a.fr[f].tokens;
  const int nblocks = T / kBlockSymbols + 1;
  if (k >= nblocks) return;
  Block& B = a.blk[(int64_t)f * a.nb + k];
  const int32_t t0 = k * kBlockSymbols, t1 = min(T, t0 + kBlockSymbols);
  const uint16_t* tok = a.tok + (int64_t)f * a.n;
  for (int i = threadIdx.x; i < 286; i += blockDim.x) S.lfreq[i] = 0;
  if (threadIdx.x == 0) S.matches = 0;
  __syncthreads();
  int my_matches = 0;
  for (int32_t i = t0 + threadIdx.x; i < t1; i += blockDim.x) {
    const int v = tok[i];
    if (v < 256) atomicAdd(&S.lfreq[v], 1u);
    else atomicAdd(&S.lfreq[257 + length_code(v - 256)], 1u), ++my_matches;
  }
  atomicAdd(&S.matches, my_matches);
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int32_t start = t1 > t0 ? B.start : (int32_t)a.n;
  const int32_t end = t1 < T ? a.blk[(int64_t)f * a.nb + k + 1].start : (int32_t)a.n;
  int64_t opt = 0, stat = 0, dopt = 0;
  S.lfreq[256] = 1;
  for (int i = 0; i < 286; ++i) S.freq[i] = S.lfreq[i];
  const int lmax = build_tree(S, 286, 0, S.llen, opt, stat);
  for (int i = 0; i < 30; ++i) S.freq[i] = 0;
  S.freq[0] = (uint32_t)S.matches;
  const int dmax = build_tree(S, 30, 1, S.dlen, opt, stat);
  for (int i = 0; i < 19; ++i) S.blfreq[i] = 0;
  tree_runs<false>(S, S.llen, lmax, nullptr);
  tree_runs<false>(S, S.dlen, dmax, nullptr);
  for (int i = 0; i < 19; ++i) S.freq[i] = S.blfreq[i];
  int64_t unused = 0;
  build_tree(S, 19, 2, S.bllen, dopt, unused);
  int max_blindex = 18;
  while (max_blindex >= 3 && S.bllen[kBlOrder[max_blindex]] == 0) --max_blindex;
  opt += dopt + 3 * (max_blindex + 1) + 5 + 5 + 4;
  int64_t opt_lenb = (opt + 3 + 7) >> 3;
  const int64_t static_lenb = (stat + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
  B.stored_len = end - start;
  B.hdr_bits = 0;
  if ((int64_t)(end - start) + 4 <= opt_lenb) {
    B.type = kStored;
    B.bits = 0;
    return;
  }
  uint16_t dcode[30];
  if (static_lenb == opt_lenb) {
    B.type = kFixed;
    B.bits = 3 + stat;
    for (int i = 0; i < 288; ++i) S.llen[i] = (uint8_t)static_llen(i);    // codes 286, 287 shift the 9-bit codes
    for (int i = 0; i < 30; ++i) S.dlen[i] = 5;
  } else {
    B.type = kDynamic;
    B.bits = 3 + opt;
    gen_codes(S.bllen, 19, S.blcode);
    BitWriter w{B.hdr, 0, 0ull, 0};
    w.put((unsigned)(lmax + 1 - 257), 5);
    w.put((unsigned)dmax, 5);
    w.put((unsigned)(max_blindex + 1 - 4), 4);
    for (int r = 0; r <= max_blindex; ++r) w.put(S.bllen[kBlOrder[r]], 3);
    tree_runs<true>(S, S.llen, lmax, &w);
    tree_runs<true>(S, S.dlen, dmax, &w);
    w.flush();
    B.hdr_bits = w.bits;
  }
  gen_codes(S.llen, B.type == kFixed ? 288 : 286, S.lcode);
  for (int i = 0; i < 286; ++i) B.lcode[i] = S.lcode[i];
  gen_codes(S.dlen, 30, dcode);
  for (int i = 0; i < 286; ++i) B.llen[i] = S.llen[i];
  B.dcode0 = dcode[0];
  B.dlen0 = S.dlen[0];
}

// Per frame, one thread: the blocks' bit offsets after the 2-byte header, stored blocks aligned after their 3 type bits; the
// stream length with Adler-32; the file size, or -1 when the stream exceeds its slot.  Writes the zlib header and trailer.
__device__ __forceinline__ void or_byte(uint8_t* z, int64_t byte, unsigned v) {
  atomicOr(reinterpret_cast<unsigned*>(z + (byte & ~3ll)), v << (8 * (byte & 3)));
}

__global__ void png_offsets_kernel(Args a, int F, int64_t out_pitch, int64_t* sizes) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int32_t T = a.fr[f].tokens;
  const int nblocks = T / kBlockSymbols + 1;
  Block* blk = a.blk + (int64_t)f * a.nb;
  int64_t pos = 16;
  for (int k = 0; k < nblocks; ++k) {
    blk[k].off = pos;
    if (blk[k].type == kStored) pos = ((pos + 3 + 7) & ~7ll) + 32 + 8ll * blk[k].stored_len;
    else pos += blk[k].bits;
  }
  const int64_t zlen = (pos + 7) / 8 + 4;
  const int64_t size = zlen + 12 * ((zlen + kChunk - 1) / kChunk) + 45;
  if (zlen + 8 > a.zcap || size > out_pitch) {
    a.fr[f].zlen = -1;
    sizes[f] = -1;
    return;
  }
  a.fr[f].zlen = zlen;
  sizes[f] = size;
  uint8_t* z = a.zbuf + f * a.zcap;
  // zlib's header for the window, then optimize_cmf's rewrite from the data size
  unsigned cmf = (unsigned)(((window_bits(a.n) - 8) << 4) | 8), flg = 0x1f - ((cmf << 8) % 0x1f);
  if (a.n <= 16384) {
    unsigned cinfo = cmf >> 4, half = 1u << (cinfo + 7);
    if (a.n <= half) {
      do half >>= 1, --cinfo;
      while (cinfo > 0 && a.n <= half);
      cmf = (cmf & 0x0f) | (cinfo << 4);
      flg = 0x1f - ((cmf << 8) % 0x1f);
    }
  }
  or_byte(z, 0, cmf);
  or_byte(z, 1, flg);
  const unsigned adler = adler_of_sums(a.fr[f].s1, a.fr[f].s2, a.n);
  for (int i = 0; i < 4; ++i) or_byte(z, zlen - 4 + i, (adler >> (24 - 8 * i)) & 0xff);
}

// Bits v (at most 25 of them) at bit offset off of the zeroed stream.
__device__ __forceinline__ void or_bits(uint8_t* z, int64_t off, unsigned long long v) {
  unsigned* w = reinterpret_cast<unsigned*>(z) + (off >> 5);
  const int s = (int)(off & 31);
  const unsigned long long x = v << s;
  if ((unsigned)x) atomicOr(w, (unsigned)x);
  if ((unsigned)(x >> 32)) atomicOr(w + 1, (unsigned)(x >> 32));
}

__global__ void __launch_bounds__(kPackThreads) png_pack_kernel(Args a) {
  __shared__ int64_t sh[32];
  __shared__ uint16_t lcode[286];
  __shared__ uint8_t llen[286];
  const int f = blockIdx.y, k = blockIdx.x;
  const int32_t T = a.fr[f].tokens;
  if (k >= T / kBlockSymbols + 1 || a.fr[f].zlen < 0) return;
  const Block& B = a.blk[(int64_t)f * a.nb + k];
  uint8_t* z = a.zbuf + f * a.zcap;
  const bool last = k == T / kBlockSymbols;
  const int64_t off = B.off;
  if (B.type == kStored) {
    if (threadIdx.x == 0) or_bits(z, off, last ? 1 : 0);
    const int64_t byte0 = (off + 3 + 7) >> 3;
    const uint32_t L = (uint32_t)B.stored_len;
    const uint8_t* src = a.filt + f * a.fstride + B.start;
    for (int64_t i = threadIdx.x; i < 4 + (int64_t)L; i += blockDim.x) {
      const unsigned v = i == 0 ? L & 0xff : i == 1 ? (L >> 8) & 0xff : i == 2 ? ~L & 0xff : i == 3 ? (~L >> 8) & 0xff : src[i - 4];
      if (v) or_byte(z, byte0 + i, v);
    }
    return;
  }
  for (int i = threadIdx.x; i < 286; i += blockDim.x) lcode[i] = B.lcode[i], llen[i] = B.llen[i];
  const int dl = B.dlen0;
  const unsigned dc = B.dcode0;
  if (threadIdx.x == 0) or_bits(z, off, (B.type == kFixed ? 2 : 4) + (last ? 1 : 0));
  for (int i = threadIdx.x; i < (B.hdr_bits + 7) / 8; i += blockDim.x) or_bits(z, off + 3 + 8ll * i, B.hdr[i]);
  __syncthreads();
  const int32_t t0 = k * kBlockSymbols, t1 = min(T, t0 + kBlockSymbols);
  const int per = (kBlockSymbols + kPackThreads - 1) / kPackThreads;
  const int32_t my0 = min(t1, t0 + (int32_t)threadIdx.x * per), my1 = min(t1, my0 + per);
  const uint16_t* tok = a.tok + (int64_t)f * a.n;
  auto code_of = [&](int v, int& nb) -> unsigned long long {
    if (v < 256) {
      nb = llen[v];
      return lcode[v];
    }
    const int lc = v - 256, c = length_code(lc), xb = kExtraL[c];
    const int ln = llen[257 + c];
    nb = ln + xb + dl;
    return (unsigned long long)lcode[257 + c] | ((unsigned long long)(lc - kBaseLength[c]) << ln) | ((unsigned long long)dc << (ln + xb));
  };
  int64_t mine = 0;
  for (int32_t i = my0; i < my1; ++i) {
    int nb;
    code_of(tok[i], nb);
    mine += nb;
  }
  int64_t total;
  int64_t pos = off + 3 + B.hdr_bits + block_scan(mine, SumS64(), (int64_t)0, sh, &total);
  for (int32_t i = my0; i < my1; ++i) {
    int nb;
    const unsigned long long v = code_of(tok[i], nb);
    or_bits(z, pos, v);
    pos += nb;
  }
  if (threadIdx.x == 0) or_bits(z, off + 3 + B.hdr_bits + total, lcode[256]);
}

// One warp per IDAT chunk of each frame: its length, type, bytes and CRC; chunk 0 adds signature and IHDR, the last IEND.
__global__ void __launch_bounds__(32) png_frame_kernel(Args a, uint8_t* out, int64_t out_pitch) {
  __shared__ uint32_t table[256], x2n[32];
  __shared__ uint32_t part[32];
  const int f = blockIdx.y, c = blockIdx.x, lane = threadIdx.x;
  const int64_t zlen = a.fr[f].zlen;
  if (zlen < 0) return;
  const int64_t nchunks = (zlen + kChunk - 1) / kChunk;
  if (c >= nchunks) return;
  crc_tables(table, x2n, lane);
  uint8_t* o = out + f * out_pitch;
  const uint8_t* z = a.zbuf + f * a.zcap + (int64_t)c * kChunk;
  const int64_t left = zlen - (int64_t)c * kChunk;
  const int len = left < kChunk ? (int)left : kChunk;
  uint8_t* ch = o + 33 + (int64_t)c * (kChunk + 12);
  for (int i = lane; i < len; i += 32) ch[8 + i] = z[i];
  if (lane == 0) {
    put_be32(ch, (uint32_t)len);
    ch[4] = 'I', ch[5] = 'D', ch[6] = 'A', ch[7] = 'T';
  }
  __syncwarp();
  const uint32_t crc = warp_crc(table, x2n, part, ch + 4, len + 4, lane);
  if (lane == 0) {
    put_be32(ch + 8 + len, crc);
    if (c == 0) {
      const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
      for (int i = 0; i < 8; ++i) o[i] = sig[i];
      uint8_t* h = o + 8;
      put_be32(h, 13);
      h[4] = 'I', h[5] = 'H', h[6] = 'D', h[7] = 'R';
      put_be32(h + 8, (uint32_t)a.W);
      put_be32(h + 12, (uint32_t)a.H);
      h[16] = 8, h[17] = a.C == 1 ? 0 : a.C == 3 ? 2 : 6, h[18] = 0, h[19] = 0, h[20] = 0;
      put_be32(h + 21, crc_bytes(table, 0, h + 4, 17));
    }
    if (c == nchunks - 1) {
      uint8_t* e = ch + 12 + len;
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
      for (int i = 0; i < 12; ++i) e[i] = iend[i];
    }
  }
}

}  // namespace
}  // namespace opb

extern "C" int opb_png_workspace_bytes(int32_t F, int32_t H, int32_t W, int32_t C, int64_t* bytes) {
  REQUIRE(__func__, bytes && F > 0 && F <= OPB_PNG_MAX_FRAMES && H > 0 && W > 0 && (C == 1 || C == 3 || C == 4));
  const int64_t n = (int64_t)H * (1 + (int64_t)W * C);
  REQUIRE(__func__, n <= opb::kMaxFiltered);
  *bytes = (int64_t)opb::layout(F, n).total;
  return OPB_OK;
}

extern "C" int opb_png_frame_bytes(int32_t H, int32_t W, int32_t C, int64_t* bytes) {
  REQUIRE(__func__, bytes && H > 0 && W > 0 && (C == 1 || C == 3 || C == 4));
  const int64_t n = (int64_t)H * (1 + (int64_t)W * C);
  REQUIRE(__func__, n <= opb::kMaxFiltered);
  *bytes = opb::png_bound(n);
  return OPB_OK;
}

extern "C" int opb_png_encode(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t F, int32_t H, int32_t W, int32_t C,
                              void* workspace, int64_t workspace_bytes, uint8_t* out, int64_t out_pitch, int64_t* sizes, void* stream) {
  REQUIRE(__func__, frames && workspace && out && sizes);
  REQUIRE(__func__, F > 0 && F <= OPB_PNG_MAX_FRAMES && H > 0 && W > 0 && (C == 1 || C == 3 || C == 4));
  const int64_t n = (int64_t)H * (1 + (int64_t)W * C);
  REQUIRE(__func__, n <= opb::kMaxFiltered);
  REQUIRE(__func__, row_pitch >= (int64_t)W * C && (F == 1 || frame_pitch == 0 || frame_pitch >= (int64_t)H * row_pitch));
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  const opb::PngLayout L = opb::layout(F, n);
  REQUIRE(__func__, workspace_bytes >= (int64_t)L.total);
  REQUIRE(__func__, out_pitch >= opb::png_bound(n));
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = (uint8_t*)workspace;
  opb::Args a;
  a.frames = frames;
  a.frame_pitch = F == 1 ? 0 : frame_pitch;
  a.row_pitch = row_pitch;
  a.H = H, a.W = W, a.C = C;
  a.n = n;
  a.row = 1 + (int64_t)W * C;
  a.nt = L.nt, a.nb = L.nb, a.zcap = L.zcap;
  a.fstride = (int64_t)opb::align256((size_t)n);
  a.filt = w + L.filt;
  a.tok = (uint16_t*)(w + L.tok);
  const size_t tile_part = opb::align256((size_t)F * L.nt * 4);
  a.tile_first = (int32_t*)(w + L.tile);
  a.tile_last = (int32_t*)(w + L.tile + tile_part);
  a.tile_count = (int32_t*)(w + L.tile + 2 * tile_part);
  a.tile_off = (int32_t*)(w + L.tile + 3 * tile_part);
  a.blk = (opb::Block*)(w + L.blk);
  a.fr = (opb::Frame*)(w + L.frame);
  a.zbuf = w + L.zbuf;
  CK(opb::no_handle_error, cudaMemsetAsync(a.fr, 0, (size_t)F * sizeof(opb::Frame), st));
  CK(opb::no_handle_error, cudaMemsetAsync(a.zbuf, 0, (size_t)F * L.zcap, st));
  const dim3 tiles((unsigned)L.nt, (unsigned)F), blocks((unsigned)L.nb, (unsigned)F);
  LAUNCH_NH(__func__, opb::png_filter_kernel, tiles, opb::kTileThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_carry_kernel, (unsigned)F, opb::kScanThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_tokens_kernel<false>, tiles, opb::kTileThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_scan_kernel, (unsigned)F, opb::kScanThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_tokens_kernel<true>, tiles, opb::kTileThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_tree_kernel, blocks, 256, 0, st, a);
  LAUNCH_NH(__func__, opb::png_offsets_kernel, (unsigned)((F + 127) / 128), 128, 0, st, a, (int)F, out_pitch, sizes);
  LAUNCH_NH(__func__, opb::png_pack_kernel, blocks, opb::kPackThreads, 0, st, a);
  const int64_t max_chunks = (L.zcap + opb::kChunk - 1) / opb::kChunk;
  LAUNCH_NH(__func__, opb::png_frame_kernel, dim3((unsigned)max_chunks, (unsigned)F), 32, 0, st, a, out, out_pitch);
  return OPB_OK;
}
