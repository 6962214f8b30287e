// PNG files read as cv2.imread / cv2.imdecode (OpenCV 4.13, libpng 1.6, zlib 1.3) read them with IMREAD_GRAYSCALE or IMREAD_COLOR,
// for F files of one width and height in one call: 8-bit grey, RGB and RGBA files, not interlaced, any zlib stream split into any
// IDAT chunks, every row filter.  The rules -- which files libpng refuses and which of its complaints are only warnings, its window
// handling, the grey and BGR conversions -- and the probes behind them are DESIGN §5.16; the byte model and a Python emulation of
// these kernels are tests/png_decode_reference.py.
//
//   png_offsets_kernel  offsets that decrease anywhere refuse every file
//   png_chunks_kernel   one warp per file: signature, IHDR, chunk order and names, every chunk's CRC-32 (warp_crc), the format
//                       and shape, and the first run of IDAT chunks' data copied into one zlib stream in the workspace
//   png_inflate_kernel  one warp per file: lane 0 decodes up to 32 tokens (literals, matches, stored spans) from shared-memory
//                       tables with the bit buffer in registers, then the warp writes them; zlib's checks on every code set,
//                       block, length and distance, libpng's window and end-of-image rules, Adler-32 and the filter bytes
//   png_rows_kernel     one CTA per row: NONE rows stay, SUB rows are a per-channel prefix sum mod 256 (block_scan of __vadd4)
//   png_chain_kernel    one CTA per run of UP / AVG / PAETH rows that follows a NONE or SUB row (or starts the image): UP rows
//                       across the row, runs of AVG / PAETH rows as a wavefront, one row per thread, one pixel per step
//   png_convert_kernel  the mode's pixels: grey (grey_of of RGB, alpha ignored) with image / 255, or BGR
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "grey.cuh"
#include "host_util.cuh"
#include "png_common.cuh"

namespace opb {
namespace {

constexpr int kPiece = 8192;                 // libpng's IDAT read size: the most input one inflate call sees
constexpr int64_t kMaxFilteredBytes = 1ll << 28;
constexpr int kFastBits = 10;                // lookup-table bits; longer codes take the canonical walk
constexpr int kBatch = 32;                   // tokens lane 0 decodes before the warp writes them
constexpr int kRowThreads = 256;
constexpr int kChainThreads = 256;
constexpr int kInvalidSym = 511;             // a table entry of a code that zlib rejects when it is read

struct FileRec {
  int32_t status, C;                         // OPB_PNG_* and the file's channels
  int64_t idat;                              // file offset of the first IDAT chunk's length field
  int64_t zlen;                              // bytes of the first IDAT run: the zlib stream, at zbuf + offsets[f]
};

__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct DLayout {
  size_t flag, rec, filt, zbuf, total;
  int64_t slot;                              // filtered bytes' slot per file: H * (1 + 4 W), aligned
};

DLayout dlayout(int F, int H, int W, int64_t total_bytes) {
  DLayout L;
  L.slot = (int64_t)align256((size_t)H * (1 + 4 * (size_t)W));
  size_t o = 0;
  L.flag = o; o += 256;
  L.rec = o; o += align256((size_t)F * sizeof(FileRec));
  L.filt = o; o += (size_t)F * L.slot;
  L.zbuf = o; o += align256((size_t)total_bytes);
  L.total = o;
  return L;
}

struct DArgs {
  const uint8_t* data;
  const int64_t* offsets;
  int H, W, mode;
  int64_t zcap, slot;
  int32_t* unordered;                        // set when the offsets decrease anywhere
  FileRec* rec;
  uint8_t* filt;
  uint8_t* zbuf;
  uint8_t* out;
  int64_t out_frame_pitch, out_row_pitch;
  float* image;
  int32_t* status;
};

__device__ __forceinline__ uint32_t be32(const uint8_t* p) {
  return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3];
}
__host__ __device__ constexpr uint32_t tag(char a, char b, char c, char d) {
  return (uint32_t)(uint8_t)a << 24 | (uint32_t)(uint8_t)b << 16 | (uint32_t)(uint8_t)c << 8 | (uint8_t)d;
}
__device__ __forceinline__ bool letter(uint32_t c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }

// ---- chunks ----

// Offsets that decrease anywhere would let files overlap in the workspace's streams: every file is then refused.
__global__ void png_offsets_kernel(DArgs a, int F) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < F && (a.offsets[i] > a.offsets[i + 1] || (i == 0 && a.offsets[0] < 0))) atomicOr(a.unordered, 1);
}

__global__ void __launch_bounds__(32) png_chunks_kernel(DArgs a) {
  __shared__ uint32_t table[256], x2n[32], part[32];
  const int f = blockIdx.x, lane = threadIdx.x;
  crc_tables(table, x2n, lane);
  const int64_t b = a.offsets[f], e = a.offsets[f + 1];
  int status = OPB_PNG_OK, C = 0;
  int64_t idat = -1, zlen = 0;
  if (*a.unordered || b < 0 || e < b || e > a.zcap) status = OPB_PNG_NOT_PNG;
  const uint8_t* p = a.data + (status == OPB_PNG_OK ? b : 0);
  const int64_t len = status == OPB_PNG_OK ? e - b : 0;
  const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  for (int i = 0; i < 8 && status == OPB_PNG_OK; ++i)
    if (len < 8 || p[i] != sig[i]) status = OPB_PNG_NOT_PNG;
  int64_t pos = 8;
  bool idat_done = false;
  for (int k = 0; status == OPB_PNG_OK; ++k) {
    if (len - pos < 12) { status = OPB_PNG_NOT_PNG; break; }           // no IEND: libpng runs out of input
    const uint32_t L = be32(p + pos), type = be32(p + pos + 4);
    if (L > 0x7fffffffu || (int64_t)L > len - pos - 12) { status = OPB_PNG_NOT_PNG; break; }
    if (!letter(type >> 24) || !letter((type >> 16) & 255) || !letter((type >> 8) & 255) || !letter(type & 255)) {
      status = OPB_PNG_NOT_PNG;
      break;
    }
    const uint32_t crc = __shfl_sync(0xffffffffu, warp_crc(table, x2n, part, p + pos + 4, (int64_t)L + 4, lane), 0);
    const bool crc_ok = crc == be32(p + pos + 8 + L);
    const bool critical = !(type & 0x20000000u);
    const uint8_t* d = p + pos + 8;
    if (k == 0) {
      if (type != tag('I', 'H', 'D', 'R') || L != 13) { status = OPB_PNG_NOT_PNG; break; }
      if (!crc_ok) { status = OPB_PNG_BAD_CRC; break; }
      const int depth = d[8], ct = d[9];
      if (depth != 8 || (ct != 0 && ct != 2 && ct != 6) || d[10] || d[11] || d[12]) { status = OPB_PNG_UNSUPPORTED; break; }
      if (be32(d) != (uint32_t)a.W || be32(d + 4) != (uint32_t)a.H) { status = OPB_PNG_BAD_SHAPE; break; }
      C = ct == 0 ? 1 : ct == 2 ? 3 : 4;
    } else if (type == tag('I', 'H', 'D', 'R')) {
      status = OPB_PNG_NOT_PNG;
    } else if (type == tag('I', 'E', 'N', 'D')) {
      if (idat < 0) status = OPB_PNG_NOT_PNG;
      break;                                 // an IEND with a bad CRC is only a warning; bytes after it are not read
    } else if (critical && !crc_ok) {
      status = OPB_PNG_BAD_CRC;
    } else if (type == tag('I', 'D', 'A', 'T')) {
      if (idat < 0) idat = pos;
      if (!idat_done) {                      // IDATs after the first run are ignored, as libpng's "Too many IDATs" warning
        uint8_t* z = a.zbuf + b + zlen;
        for (int64_t i = lane; i < L; i += 32) z[i] = d[i];
        zlen += L;
      }
    } else {
      if (idat >= 0) idat_done = true;
      if (type == tag('P', 'L', 'T', 'E')) {
        if (C == 1 || idat >= 0) status = OPB_PNG_NOT_PNG;
      } else if (critical) {
        status = OPB_PNG_NOT_PNG;            // unhandled critical chunk
      } else if (crc_ok && idat < 0 && a.mode == OPB_PNG_READ_GREY && C > 1 &&
                 ((type == tag('g', 'A', 'M', 'A') && L == 4 && be32(d) != 100000u) || type == tag('s', 'R', 'G', 'B') ||
                  type == tag('i', 'C', 'C', 'P'))) {
        status = OPB_PNG_UNSUPPORTED;        // libpng's rgb_to_gray would work in linear light
      }
    }
    pos += 12 + (int64_t)L;
  }
  if (lane == 0) {
    FileRec& R = a.rec[f];
    R.status = status;
    R.C = C;
    R.idat = idat;
    R.zlen = zlen;
  }
}

// ---- inflate ----

__constant__ uint16_t kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                       4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// A canonical code's decoding tables: fast[i] = symbol | length << 9 for the code that the low kFastBits bits i start with (0:
// a longer code), count / sorted for the canonical walk of longer codes.
struct Table {
  uint16_t fast[1 << kFastBits];
  uint16_t count[16];
  uint16_t sorted[288];
};

struct InflateSmem {
  Table lit, dist;
  uint8_t lens[320];
  uint16_t code[320];
  int32_t tpos[kBatch], tlen[kBatch], tdist[kBatch];   // tdist > 0: match; 0: literal tlen; -1: stored bytes from tsrc
  int64_t tsrc[kBatch];
  int32_t ntok, done;
  int32_t bad;                                         // build_table's verdict
  unsigned long long s1[32], s2[32];
};

// inflate_table's checks and the tables of lens[0 .. n).  kind 0: the code-length code (must be complete), 1: literal/length,
// 2: distance (a single code of length 1, or none at all, is allowed: the missing codes decode as invalid symbols).  Lane 0
// checks and assigns codes, the warp fills the fast table.  Returns false for a set zlib rejects.
__device__ bool build_table(InflateSmem& S, Table& T, const uint8_t* lens, int n, int kind, int lane) {
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) T.count[l] = 0;
    for (int i = 0; i < n; ++i) T.count[lens[i]]++;
    int max = 15;
    while (max > 0 && T.count[max] == 0) --max;
    int left = 1, bad = 0;
    for (int l = 1; l < 16; ++l) {
      left <<= 1;
      left -= T.count[l];
      if (left < 0) bad = 1;                           // over-subscribed
    }
    if (max == 0) bad = kind != 2;                     // no codes: only a distance code may be empty
    else if (left > 0 && (kind == 0 || max != 1)) bad = 1;   // incomplete
    S.bad = bad | ((left > 0) << 1);
    uint16_t offs[16], next[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + T.count[l];
    unsigned c = 0;
    T.count[0] = 0;
    for (int l = 1; l < 16; ++l) next[l] = (uint16_t)(c = (c + T.count[l - 1]) << 1);
    for (int i = 0; i < n; ++i)
      if (lens[i]) {
        T.sorted[offs[lens[i]]++] = (uint16_t)i;
        S.code[i] = (uint16_t)(__brev(next[lens[i]]++) >> (32 - lens[i]));
      }
  }
  __syncwarp();
  const int verdict = S.bad;
  __syncwarp();
  if (verdict & 1) return false;
  const uint16_t fill = (verdict & 2) ? (uint16_t)(kInvalidSym | 1 << 9) : 0;   // an incomplete or empty set's missing 1-bit code
  for (int i = lane; i < (1 << kFastBits); i += 32) T.fast[i] = fill;
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const int l = lens[i];
    if (l == 0 || l > kFastBits) continue;
    for (int j = S.code[i]; j < (1 << kFastBits); j += 1 << l) T.fast[j] = (uint16_t)(i | l << 9);
  }
  __syncwarp();
  return true;
}

// Where libpng's reading stands in the stream.  kImage: rows still to come.  kLastCall: the image is complete and zlib goes on
// in the last row's inflate call (its errors are fatal).  kFinish: libpng's finishing call, one inflate over the next piece
// (errors are warnings; running out of that piece ends it).  kExtra: that call has produced more image data, and libpng keeps
// inflating until the stream ends (errors are warnings; running out of IDAT data is fatal).
enum { kImage = 0, kLastCall = 1, kFinish = 2, kExtra = 3 };
constexpr int kStopped = -1;                           // decoding ended without an error before the stream's end
constexpr int kFinishBuffer = 1024;                    // libpng's finishing call inflates into a buffer of this size

// Lane 0's decoder state.  Positions in the zlib stream are bits (cbit) and bytes; out counts the filtered bytes decoded, past n
// once there is more image data than the image holds (those are not written).
struct Inflater {
  const uint8_t* z;
  int64_t zlen, zbits, cbit;
  unsigned long long buf;
  int nb;
  int64_t rpos;
  // the piece of input libpng has handed zlib: the first IDAT run walked chunk by chunk, each in pieces of kPiece bytes
  const uint8_t* file;
  int64_t pc_data, pc_len, pc_off, pc_z, piece_end;
  int64_t out, n, row, cs_piece, wsize;
  int phase;

  __device__ void next_piece() {                       // after the run's last piece, piece_end stays at zlen
    pc_off += kPiece;
    while (pc_off >= pc_len) {
      if (pc_z + pc_len >= zlen) {
        piece_end = zlen;
        return;
      }
      pc_z += pc_len;
      const int64_t h = pc_data + pc_len + 4;
      pc_len = be32(file + h);
      pc_data = h + 8;
      pc_off = 0;
    }
    piece_end = pc_z + min(pc_len, pc_off + kPiece);
  }
  __device__ void refill() {
    while (nb <= 56 && rpos < zlen) buf |= (unsigned long long)z[rpos++] << nb, nb += 8;
  }
  __device__ unsigned peek(int k) {
    refill();
    return (unsigned)(buf & ((1ull << k) - 1));
  }
  __device__ void skip(int k) {
    buf >>= k;
    nb -= k;
    cbit += k;
  }
  // 0: the next k bits can be read; 1: stop without an error (the finishing call's piece is used up); 2: the IDAT data ends
  // first, which libpng refuses in every phase.  A first bit from a new piece starts a new inflate call at the current output.
  __device__ int need(int k) {
    const int64_t last = (cbit + k - 1) >> 3;
    if (k == 0 || last < piece_end) return 0;
    if (phase == kFinish) return 1;
    cs_piece = out;
    if (phase == kLastCall) {                          // the finishing call loads one more piece
      if (piece_end >= zlen) return 2;
      next_piece();
      phase = kFinish;
      return last >= piece_end ? 1 : 0;
    }
    if (cbit + k > zbits) return 2;
    while (last >= piece_end) next_piece();
    return 0;
  }
  // The last row's call has stopped with image data still to write: the finishing call loads the next piece first when the
  // current one is used up (fatal when the IDAT run is over), and the data it then produces keeps it inflating.
  __device__ int start_extra() {
    if (((cbit + 7) >> 3) >= piece_end) {
      if (piece_end >= zlen) return 2;
      cs_piece = n;
      next_piece();
    }
    phase = kExtra;
    return 0;
  }
  // Before decoded output past the image: 0, or 2 as need().
  __device__ int more_output() {
    if (phase == kLastCall) return start_extra();
    phase = kExtra;
    return 0;
  }
  // The output position where the inflate call writing position p began: one call per row, then kFinishBuffer-byte calls.
  __device__ int64_t call_start(int64_t p) const { return p < n ? p - p % row : n + ((p - n) / kFinishBuffer) * kFinishBuffer; }
  __device__ int64_t next_boundary(int64_t p) const { return p < n ? p - p % row + row : call_start(p) + kFinishBuffer; }
  __device__ unsigned bits(int k) {
    const unsigned v = peek(k);
    skip(k);
    return v;
  }
  __device__ void align_byte() {
    const int r = (int)(cbit & 7);
    if (r) skip(8 - r);
  }
  // The next symbol of T into sym; returns need()'s verdict for its code.
  __device__ int decode(const Table& T, int& sym) {
    unsigned e = T.fast[peek(kFastBits)];
    int l;
    if (e) {
      l = (int)(e >> 9);
      sym = (int)(e & 511);
    } else {                                           // canonical walk (puff's decode) for codes longer than kFastBits
      const unsigned v = peek(15);
      int code = 0, first = 0, index = 0;
      sym = kInvalidSym;
      for (l = 1; l < 16; ++l) {
        code |= (v >> (l - 1)) & 1;
        const int c = T.count[l];
        if (code - c < first) {
          sym = T.sorted[index + (code - first)];
          break;
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
      }
      if (l == 16) l = 15;
    }
    const int r = need(l);
    if (r == 0) skip(l);
    return r;
  }
};

// The status after need()'s verdict r != 0.
__device__ __forceinline__ int stop_status(int r) { return r == 1 ? kStopped : OPB_PNG_TOO_LITTLE_DATA; }

// One warp per file.  The warp runs the block-level steps (header, table builds) together; lane 0 decodes each block's tokens in
// batches of kBatch and the warp writes a batch before the next is decoded.  Broadcasts go through shared memory, each read
// followed by a __syncwarp before lane 0 writes the next.
__global__ void __launch_bounds__(32) png_inflate_kernel(DArgs a) {
  __shared__ InflateSmem S;
  const int f = blockIdx.x, lane = threadIdx.x;
  FileRec& R = a.rec[f];
  if (R.status != OPB_PNG_OK) return;
  const int64_t b = a.offsets[f];
  const int C = R.C;
  uint8_t* o = a.filt + f * a.slot;
  Inflater I;
  I.z = a.zbuf + b;
  I.zlen = R.zlen;
  I.zbits = R.zlen * 8;
  I.cbit = 0, I.buf = 0, I.nb = 0, I.rpos = 0;
  I.file = a.data + b;
  I.pc_data = R.idat + 8;
  I.pc_len = be32(I.file + R.idat);
  I.pc_off = -kPiece, I.pc_z = 0;
  I.next_piece();                                      // the first non-empty chunk's first piece
  I.row = 1 + (int64_t)a.W * C;
  I.n = (int64_t)a.H * I.row;
  I.out = 0, I.cs_piece = 0, I.phase = kImage, I.wsize = 0;
  int status = OPB_PNG_OK;
  bool check = false;                                  // the Adler-32 at the stream's end is read in a fatal phase: compare it
  uint32_t adler = 0;
  // zlib header: FCHECK, CM 8, CINFO <= 7 (libpng takes the window from it), no preset dictionary
  int r = I.need(16);
  if (r) {
    status = stop_status(r);
  } else {
    const unsigned cmf = I.bits(8), flg = I.bits(8);
    if (((cmf << 8) | flg) % 31 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 0x20)) status = OPB_PNG_BAD_DEFLATE;
    I.wsize = 1ll << ((cmf >> 4) + 8);
  }
  bool last = false;
  while (status == OPB_PNG_OK && !last) {
    // ---- block header (warp-uniform through shared memory) ----
    int type = 0;
    if (lane == 0) {
      if ((r = I.need(3))) {
        status = stop_status(r);
      } else {
        last = I.bits(1);
        type = (int)I.bits(2);
        if (type == 3) status = OPB_PNG_BAD_DEFLATE;
      }
      S.ntok = type | last << 2;
      S.bad = status;
    }
    __syncwarp();
    status = S.bad;
    type = S.ntok & 3;
    last = S.ntok >> 2;
    __syncwarp();
    if (status != OPB_PNG_OK) break;
    if (type == 0) {                                   // stored: LEN, NLEN, then the bytes
      if (lane == 0) {
        I.align_byte();
        int64_t L = 0;
        if ((r = I.need(32))) {
          status = stop_status(r);
        } else {
          const unsigned v = I.bits(16), nv = I.bits(16);
          if (v != (~nv & 0xffff)) status = OPB_PNG_BAD_DEFLATE;
          else L = v;
        }
        S.ntok = 0;
        if (L > 0 && status == OPB_PNG_OK) {
          const int64_t byte0 = I.cbit >> 3;
          if (I.phase == kLastCall) {
            if (I.start_extra()) status = OPB_PNG_TOO_LITTLE_DATA;
          } else if (I.phase == kFinish) {
            if (byte0 >= I.piece_end) status = kStopped;   // nothing of the block in the finishing call's piece
            else I.phase = kExtra;
          }
          if (status == OPB_PNG_OK && I.zlen - byte0 < L) status = OPB_PNG_TOO_LITTLE_DATA;   // the IDAT data ends inside it
          if (status == OPB_PNG_OK) {
            int64_t pos = byte0, left = L;
            if (I.phase == kImage) {
              const int64_t w = min(left, I.n - I.out);
              // each piece boundary inside the copy starts a new inflate call at the output reached there
              while (pos + w > I.piece_end) I.cs_piece = I.out + (I.piece_end - pos), I.next_piece();
              S.tpos[0] = (int32_t)I.out, S.tlen[0] = (int32_t)w, S.tdist[0] = -1, S.tsrc[0] = pos;
              S.ntok = 1;
              I.out += w, pos += w, left -= w;
              if (I.out == I.n) {
                I.cbit = pos * 8;
                if (left == 0) I.phase = kLastCall;
                else if (I.start_extra()) status = OPB_PNG_TOO_LITTLE_DATA;
              }
            }
            if (status == OPB_PNG_OK && left > 0) {      // more image data than the image holds: read, not written
              while (pos + left > I.piece_end) I.cs_piece = I.out + (I.piece_end - pos), I.next_piece();
              I.out += left, pos += left;
            }
            I.buf = 0, I.nb = 0, I.rpos = pos, I.cbit = pos * 8;
          }
        }
        S.bad = status;
      }
      __syncwarp();
      status = S.bad;
      if (S.ntok) {
        const int64_t p0 = S.tpos[0], w = S.tlen[0];
        const uint8_t* src = I.z + S.tsrc[0];
        for (int64_t i = lane; i < w; i += 32) o[p0 + i] = src[i];
      }
      __syncwarp();
      if (status != OPB_PNG_OK) break;
      continue;
    }
    // ---- fixed or dynamic codes ----
    if (type == 1) {
      for (int i = lane; i < 288; i += 32) S.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
      __syncwarp();
      build_table(S, S.lit, S.lens, 288, 1, lane);
      for (int i = lane; i < 32; i += 32) S.lens[i] = 5;
      __syncwarp();
      build_table(S, S.dist, S.lens, 32, 2, lane);
    } else {
      int nlen = 0, ndist = 0, ncode = 0;
      if (lane == 0) {
        if ((r = I.need(14))) {
          status = stop_status(r);
        } else {
          nlen = (int)I.bits(5) + 257, ndist = (int)I.bits(5) + 1, ncode = (int)I.bits(4) + 4;
          if (nlen > 286 || ndist > 30) status = OPB_PNG_BAD_DEFLATE;
        }
        for (int i = 0; i < 19; ++i) S.lens[i] = 0;
        for (int i = 0; i < ncode && status == OPB_PNG_OK; ++i) {
          if ((r = I.need(3))) status = stop_status(r);
          else S.lens[kClOrder[i]] = (uint8_t)I.bits(3);
        }
        S.bad = status;
        S.tlen[0] = nlen, S.tlen[1] = ndist;
      }
      __syncwarp();
      status = S.bad;
      nlen = S.tlen[0], ndist = S.tlen[1];
      __syncwarp();
      if (status != OPB_PNG_OK) break;
      if (!build_table(S, S.lit, S.lens, 19, 0, lane)) { status = OPB_PNG_BAD_DEFLATE; break; }
      if (lane == 0) {                                 // the code-length code's table is built: its lengths may go
        uint8_t* lens = S.lens;
        int have = 0;
        while (have < nlen + ndist && status == OPB_PNG_OK) {
          int sym;
          if ((r = I.decode(S.lit, sym))) { status = stop_status(r); break; }
          if (sym < 16) { lens[have++] = (uint8_t)sym; continue; }
          const int xb = sym == 16 ? 2 : sym == 17 ? 3 : 7;
          if ((r = I.need(xb))) { status = stop_status(r); break; }
          if (sym == 16 && have == 0) { status = OPB_PNG_BAD_DEFLATE; break; }
          const int rep = (int)I.bits(xb) + (sym == 16 ? 3 : sym == 17 ? 3 : 11);
          const uint8_t v = sym == 16 ? lens[have - 1] : 0;
          if (have + rep > nlen + ndist) { status = OPB_PNG_BAD_DEFLATE; break; }
          for (int i = 0; i < rep; ++i) lens[have++] = v;
        }
        if (status == OPB_PNG_OK && lens[256] == 0) status = OPB_PNG_BAD_DEFLATE;   // no end-of-block code
        S.bad = status;
      }
      __syncwarp();
      status = S.bad;
      __syncwarp();
      if (status != OPB_PNG_OK) break;
      if (!build_table(S, S.lit, S.lens, nlen, 1, lane)) { status = OPB_PNG_BAD_DEFLATE; break; }
      for (int i = lane; i < ndist; i += 32) S.lens[i] = S.lens[nlen + i];
      __syncwarp();
      if (!build_table(S, S.dist, S.lens, ndist, 2, lane)) { status = OPB_PNG_BAD_DEFLATE; break; }
    }
    // ---- the block's tokens ----
    for (;;) {
      if (lane == 0) {
        int nt = 0, eob = 0;
        while (nt < kBatch) {
          int sym;
          if ((r = I.decode(S.lit, sym))) { status = stop_status(r); break; }
          if (sym >= 286) { status = OPB_PNG_BAD_DEFLATE; break; }
          if (sym == 256) { eob = 1; break; }
          if (sym < 256) {
            if (I.phase == kImage) {
              S.tpos[nt] = (int32_t)I.out, S.tlen[nt] = sym, S.tdist[nt] = 0;
              ++nt;
              if (++I.out == I.n) I.phase = kLastCall;
            } else {
              if ((r = I.more_output())) { status = stop_status(r); break; }
              ++I.out;
            }
            continue;
          }
          const int lc = sym - 257, lx = kLenExtra[lc];
          if ((r = I.need(lx))) { status = stop_status(r); break; }
          const int L = kLenBase[lc] + (int)I.bits(lx);
          int ds;
          if ((r = I.decode(S.dist, ds))) { status = stop_status(r); break; }
          if (ds >= 30) { status = OPB_PNG_BAD_DEFLATE; break; }
          const int dx = kDistExtra[ds];
          if ((r = I.need(dx))) { status = stop_status(r); break; }
          const int64_t d = kDistBase[ds] + (int64_t)I.bits(dx);
          if (I.phase != kImage && (r = I.more_output())) { status = stop_status(r); break; }
          // zlib reaches back over its window plus what the current inflate call has written, and checks again where a match
          // goes on into the next call: q is where the match stops, at the first refused position if any
          const int64_t p = I.out, cs = max(I.call_start(p), I.cs_piece);
          int64_t q = p + L;
          bool bad = false;
          if (d > p - cs + min(I.wsize, cs)) q = p, bad = true;
          else if (d > I.wsize && I.next_boundary(p) < q) q = I.next_boundary(p), bad = true;
          if (p < I.n && min(q, I.n) > p) {
            S.tpos[nt] = (int32_t)p, S.tlen[nt] = (int32_t)(min(q, I.n) - p), S.tdist[nt] = (int32_t)d;
            ++nt;
          }
          I.out = q;
          if (I.phase == kImage && q >= I.n) {
            if (q > I.n || bad) {                        // the rest goes to the finishing call
              if ((r = I.start_extra())) { status = stop_status(r); break; }
            } else {
              I.phase = kLastCall;
            }
          }
          if (bad) { status = OPB_PNG_BAD_DEFLATE; break; }
        }
        S.ntok = nt, S.done = eob, S.bad = status;
      }
      __syncwarp();
      const int nt = S.ntok, eob = S.done;
      status = S.bad;
      if (lane < nt && S.tdist[lane] == 0) o[S.tpos[lane]] = (uint8_t)S.tlen[lane];
      __syncwarp();
      for (int t = 0; t < nt; ++t) {
        const int64_t d = S.tdist[t];
        if (d <= 0) continue;
        const int64_t p = S.tpos[t];
        for (int64_t j = lane; j < S.tlen[t]; j += 32) o[p + j] = o[p - d + j % d];
        __syncwarp();
      }
      __syncwarp();
      if (status != OPB_PNG_OK || eob) break;
    }
    if (status != OPB_PNG_OK) break;
  }
  // ---- the stream's end: the Adler-32, compared when it is read in a fatal phase ----
  __syncwarp();
  if (lane == 0) {
    if (status == OPB_PNG_OK) {
      I.align_byte();
      if ((r = I.need(32))) {
        status = stop_status(r);
      } else {
        const unsigned v = I.bits(8) << 24;
        adler = v | I.bits(8) << 16;
        adler |= I.bits(8) << 8;
        adler |= I.bits(8);
        check = I.phase <= kLastCall;
        if (I.out < I.n) status = OPB_PNG_TOO_LITTLE_DATA;   // checked after the Adler-32, which zlib reads first
      }
    }
    if (status == kStopped || (I.phase >= kFinish && status == OPB_PNG_BAD_DEFLATE)) status = OPB_PNG_OK;   // only warnings
    S.bad = status, S.done = check, S.ntok = (int32_t)min(I.out, I.n), S.tsrc[0] = adler;
  }
  __syncwarp();
  status = S.bad;
  const int64_t produced = S.ntok;
  if ((status == OPB_PNG_OK || status == OPB_PNG_TOO_LITTLE_DATA) && S.done) {
    unsigned long long s1 = 0, s2 = 0;
    for (int64_t i = lane; i < produced; i += 32) s1 += o[i], s2 += (unsigned long long)(produced - i) * o[i];
    S.s1[lane] = s1, S.s2[lane] = s2;
    __syncwarp();
    if (lane == 0) {
      for (int l = 1; l < 32; ++l) s1 += S.s1[l], s2 += S.s2[l];
      if (adler_of_sums(s1, s2, produced) != (uint32_t)S.tsrc[0]) S.bad = OPB_PNG_BAD_ADLER;
    }
    __syncwarp();
    status = S.bad;
  }
  if (status == OPB_PNG_OK) {                          // filter bytes: 0 .. 4
    const int64_t row = 1 + (int64_t)a.W * C;
    bool badf = false;
    for (int y = lane; y < a.H; y += 32) badf |= o[y * row] > 4;
    if (__any_sync(0xffffffffu, badf)) status = OPB_PNG_BAD_FILTER;
  }
  if (lane == 0) R.status = status;
}

// ---- unfilter and convert ----

struct Vadd4 { __device__ uint32_t operator()(uint32_t x, uint32_t y) const { return __vadd4(x, y); } };

__device__ __forceinline__ uint32_t load_px(const uint8_t* p, int C) {
  uint32_t v = 0;
  for (int c = 0; c < C; ++c) v |= (uint32_t)p[c] << (8 * c);
  return v;
}
__device__ __forceinline__ void store_px(uint8_t* p, int C, uint32_t v) {
  for (int c = 0; c < C; ++c) p[c] = (uint8_t)(v >> (8 * c));
}

// One CTA per row of each file: SUB rows become their per-channel prefix sums mod 256 in place (pixels packed in 32-bit words,
// added bytewise).  NONE rows need nothing; the other filters are png_chain_kernel's.
__global__ void __launch_bounds__(kRowThreads) png_rows_kernel(DArgs a) {
  __shared__ uint32_t sh[32];
  const int f = blockIdx.y, y = blockIdx.x;
  const FileRec& R = a.rec[f];
  if (R.status != OPB_PNG_OK) return;
  const int C = R.C;
  uint8_t* row = a.filt + f * a.slot + (int64_t)y * (1 + (int64_t)a.W * C);
  if (row[0] != 1) return;
  uint8_t* px = row + 1;
  constexpr int kPer = 8;
  uint32_t carry = 0;
  for (int x0 = 0; x0 < a.W; x0 += kRowThreads * kPer) {
    const int xs = x0 + threadIdx.x * kPer;
    uint32_t v[kPer], acc = 0;
    for (int k = 0; k < kPer; ++k) {
      v[k] = xs + k < a.W ? load_px(px + (int64_t)(xs + k) * C, C) : 0u;
      acc = __vadd4(acc, v[k]);
      v[k] = acc;
    }
    uint32_t total;
    const uint32_t exc = __vadd4(carry, block_scan(acc, Vadd4(), 0u, sh, &total));
    for (int k = 0; k < kPer; ++k)
      if (xs + k < a.W) store_px(px + (int64_t)(xs + k) * C, C, __vadd4(exc, v[k]));
    carry = __vadd4(carry, total);
  }
}

__device__ __forceinline__ uint8_t paeth(int l, int u, int ul) {
  const int p = l + u - ul, pa = abs(p - l), pb = abs(p - u), pc = abs(p - ul);
  return (uint8_t)(pa <= pb && pa <= pc ? l : pb <= pc ? u : ul);
}

// One CTA per row that starts a run of UP / AVG / PAETH rows (row 0, or a row after a NONE or SUB row): the run's rows in order,
// UP rows across the row, each stretch of AVG / PAETH rows as a wavefront -- thread t reconstructs row a + t, pixel s - t at step
// s, after the row above has done that pixel -- in rounds of kChainThreads rows.
__global__ void __launch_bounds__(kChainThreads) png_chain_kernel(DArgs a) {
  const int f = blockIdx.y, y0 = blockIdx.x;
  const FileRec& R = a.rec[f];
  if (R.status != OPB_PNG_OK) return;
  const int C = R.C, W = a.W, H = a.H;
  const int64_t rb = 1 + (int64_t)W * C;
  uint8_t* base = a.filt + f * a.slot;
  auto ftype = [&](int y) { return base[(int64_t)y * rb]; };
  if (ftype(y0) < 2 || (y0 > 0 && ftype(y0 - 1) >= 2)) return;
  int y = y0;
  while (y < H && ftype(y) >= 2) {
    if (ftype(y) == 2) {
      uint8_t* cur = base + (int64_t)y * rb + 1;
      if (y > 0)
        for (int64_t i = threadIdx.x; i < (int64_t)W * C; i += blockDim.x) cur[i] = (uint8_t)(cur[i] + cur[i - rb]);
      __syncthreads();
      ++y;
      continue;
    }
    int y1 = y;
    while (y1 < H && ftype(y1) >= 3) ++y1;
    for (int r0 = y; r0 < y1; r0 += kChainThreads) {
      const int my = r0 + threadIdx.x;
      const bool mine = my < y1;
      const int rows = min(kChainThreads, y1 - r0);
      uint8_t* cur = base + (int64_t)my * rb + 1;
      const uint8_t* up = cur - rb;
      const bool has_up = my > 0;
      const bool is_avg = mine && ftype(my) == 3;
      for (int s = 0; s < W + rows - 1; ++s) {
        const int x = s - (int)threadIdx.x;
        if (mine && x >= 0 && x < W) {
          uint8_t* c = cur + (int64_t)x * C;
          for (int ch = 0; ch < C; ++ch) {
            const int l = x > 0 ? c[ch - C] : 0, u = has_up ? up[(int64_t)x * C + ch] : 0;
            const int ul = x > 0 && has_up ? up[(int64_t)(x - 1) * C + ch] : 0;
            c[ch] = (uint8_t)(c[ch] + (is_avg ? (l + u) >> 1 : paeth(l, u, ul)));
          }
        }
        __syncthreads();
      }
    }
    y = y1;
  }
}

// One thread per pixel of each decoded file: grey (a grey file's bytes, else grey_of of R, G, B) and image / 255, or BGR.
__global__ void __launch_bounds__(256) png_convert_kernel(DArgs a) {
  const int f = blockIdx.y;
  const FileRec& R = a.rec[f];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)a.H * a.W) {
    if (i == (int64_t)a.H * a.W) a.status[f] = R.status;
    return;
  }
  if (R.status != OPB_PNG_OK) return;
  const int C = R.C;
  const int y = (int)(i / a.W), x = (int)(i - (int64_t)y * a.W);
  const uint8_t* p = a.filt + f * a.slot + (int64_t)y * (1 + (int64_t)a.W * C) + 1 + (int64_t)x * C;
  uint8_t* o = a.out + f * a.out_frame_pitch + y * a.out_row_pitch;
  if (a.mode == OPB_PNG_READ_GREY) {
    const uint32_t g = C == 1 ? p[0] : grey_of(p[0], p[1], p[2], true);
    o[x] = (uint8_t)g;
    if (a.image) a.image[(int64_t)f * a.H * a.W + i] = __fdiv_rn((float)g, 255.f);
  } else {
    o += (int64_t)x * 3;
    if (C == 1) o[0] = o[1] = o[2] = p[0];
    else o[0] = p[2], o[1] = p[1], o[2] = p[0];
  }
}

}  // namespace
}  // namespace opb

extern "C" int opb_png_decode_workspace_bytes(int32_t F, int32_t H, int32_t W, int64_t total_bytes, int64_t* bytes) {
  REQUIRE(__func__, bytes && F > 0 && F <= OPB_PNG_MAX_FRAMES && H > 0 && W > 0 && total_bytes >= 0);
  REQUIRE(__func__, (int64_t)H * (1 + 4 * (int64_t)W) <= opb::kMaxFilteredBytes);
  *bytes = (int64_t)opb::dlayout(F, H, W, total_bytes).total;
  return OPB_OK;
}

extern "C" int opb_png_decode(const uint8_t* data, const int64_t* offsets, int32_t F, int32_t H, int32_t W, int32_t mode, void* workspace,
                              int64_t workspace_bytes, uint8_t* out, int64_t out_frame_pitch, int64_t out_row_pitch, float* image,
                              int32_t* status, void* stream) {
  REQUIRE(__func__, data && offsets && workspace && out && status);
  REQUIRE(__func__, F > 0 && F <= OPB_PNG_MAX_FRAMES && H > 0 && W > 0);
  REQUIRE(__func__, (int64_t)H * (1 + 4 * (int64_t)W) <= opb::kMaxFilteredBytes);
  REQUIRE(__func__, mode == OPB_PNG_READ_GREY || mode == OPB_PNG_READ_BGR);
  REQUIRE(__func__, image == nullptr || mode == OPB_PNG_READ_GREY);
  const int64_t px = mode == OPB_PNG_READ_GREY ? 1 : 3;
  REQUIRE(__func__, out_row_pitch >= (int64_t)W * px && (F == 1 || out_frame_pitch >= (int64_t)H * out_row_pitch));
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  const opb::DLayout L = opb::dlayout(F, H, W, 0);
  REQUIRE(__func__, workspace_bytes >= (int64_t)L.total);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = (uint8_t*)workspace;
  opb::DArgs a;
  a.data = data;
  a.offsets = offsets;
  a.H = H, a.W = W, a.mode = mode;
  a.zcap = workspace_bytes - (int64_t)L.zbuf;
  a.slot = L.slot;
  a.unordered = (int32_t*)(w + L.flag);
  a.rec = (opb::FileRec*)(w + L.rec);
  a.filt = w + L.filt;
  a.zbuf = w + L.zbuf;
  a.out = out;
  a.out_frame_pitch = F == 1 ? 0 : out_frame_pitch;
  a.out_row_pitch = out_row_pitch;
  a.image = image;
  a.status = status;
  const int64_t pixels = (int64_t)H * W;
  CK(opb::no_handle_error, cudaMemsetAsync(a.unordered, 0, sizeof(int32_t), st));
  LAUNCH_NH(__func__, opb::png_offsets_kernel, (unsigned)((F + 255) / 256), 256, 0, st, a, (int)F);
  LAUNCH_NH(__func__, opb::png_chunks_kernel, (unsigned)F, 32, 0, st, a);
  LAUNCH_NH(__func__, opb::png_inflate_kernel, (unsigned)F, 32, 0, st, a);
  LAUNCH_NH(__func__, opb::png_rows_kernel, dim3((unsigned)H, (unsigned)F), opb::kRowThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_chain_kernel, dim3((unsigned)H, (unsigned)F), opb::kChainThreads, 0, st, a);
  LAUNCH_NH(__func__, opb::png_convert_kernel, dim3((unsigned)((pixels + 1 + 255) / 256), (unsigned)F), 256, 0, st, a);
  return OPB_OK;
}
