"""Models of the PNG reader (csrc/png_decode.cu): what cv2.imdecode / cv2.imread (OpenCV 4.13, libpng 1.6, zlib 1.3) return for a
PNG file, with the reader's status codes.

- ``model_decode`` is the byte model: the chunk walk and CRC-32s, ``zlib`` for the stream, a numpy unfilter of the five row
  filters and cv2's grey / BGR conversions.  Its deflate verdict comes from ``inflate`` below, which holds libpng's rules.
- ``inflate`` is a pure-Python emulation of png_inflate_kernel: the same tables (a 10-bit lookup and the canonical walk), the same
  checks in zlib's order and the same status codes, with libpng's two rules on top (DESIGN §5.16):
  * libpng inflates one row per call and hands zlib the IDAT data in pieces of 8192 bytes per chunk; zlib accepts a distance up
    to its window (from CINFO) plus what the current call has written.  So a distance past the window is accepted inside a
    row (and inside one piece), and refused across a row or piece boundary.
  * After the last row: what zlib reads in that same call is checked as before (errors and a bad Adler-32 are fatal).  Then
    libpng's finishing call inflates once more, loading the next piece if the last one is used up (fatal when the IDAT run
    is over); its errors are only warnings.  If that call produces no image data, reading ends there.  If it does (more
    image data than the image holds), libpng keeps inflating to the stream's end: errors stay warnings, and running out of
    IDAT data is fatal.
- ``png_file`` and ``Deflater`` build test files: chunk splits, ancillary chunks and hand-made deflate streams.
"""
import struct
import zlib

import numpy as np

from tests import grey_reference

OK, NOT_PNG, BAD_CRC, UNSUPPORTED, BAD_SHAPE, BAD_DEFLATE, BAD_ADLER, TOO_LITTLE, BAD_FILTER = range(9)
GREY, BGR = 0, 1                         # cv2.IMREAD_GRAYSCALE, cv2.IMREAD_COLOR
PIECE = 8192
SIGNATURE = b"\x89PNG\r\n\x1a\n"

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
             12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FAST = 10
INVALID = 511


# ---- building files ----

def chunk(kind: bytes, data: bytes, crc=None) -> bytes:
    c = zlib.crc32(kind + data) if crc is None else crc
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", c & 0xffffffff)


def ihdr(H, W, ct, depth=8, interlace=0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ct, 0, 0, interlace))


def png_file(H, W, ct, stream: bytes, split=None, before=b"", after=b"", iend=True) -> bytes:
    """A PNG file of a zlib stream: IDAT chunks of `split` bytes (or one chunk), chunks `before` and `after` the IDATs."""
    out = SIGNATURE + ihdr(H, W, ct) + before
    split = split or max(1, len(stream))
    for i in range(0, max(1, len(stream)), split):
        out += chunk(b"IDAT", stream[i:i + split])
    return out + after + (chunk(b"IEND", b"") if iend else b"")


def channels(ct: int) -> int:
    return {0: 1, 2: 3, 6: 4}[ct]


def filter_rows(pixels: np.ndarray, filters) -> bytes:
    """The filtered bytes of uint8 [H, W, C] pixels in PNG order (RGB(A)), row y with filter filters[y]."""
    H, W, C = pixels.shape
    prev = np.zeros(W * C, np.int32)
    out = bytearray()
    for y in range(H):
        cur = pixels[y].reshape(-1).astype(np.int32)
        left = np.concatenate([np.zeros(C, np.int32), cur[:-C]])
        ul = np.concatenate([np.zeros(C, np.int32), prev[:-C]])
        f = int(filters[y])
        if f == 0:
            v = cur
        elif f == 1:
            v = cur - left
        elif f == 2:
            v = cur - prev
        elif f == 3:
            v = cur - (left + prev) // 2
        else:
            v = cur - paeth(left, prev, ul)
        out.append(f)
        out += (v & 255).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


class Deflater:
    """A hand-made deflate stream, for streams zlib would not write: blocks of literals and matches with fixed codes, stored
    blocks, raw bits, any header and trailer."""

    def __init__(self, cinfo=7):
        self.acc, self.n, self.out = 0, 0, bytearray()
        cmf = (cinfo << 4) | 8
        self.header = bytes([cmf, 31 - ((cmf << 8) % 31)])

    def bits(self, v, n):
        self.acc |= v << self.n
        self.n += n

    def code(self, c, n):                # a Huffman code, most significant bit first
        self.bits(int(format(c, f"0{n}b")[::-1], 2), n)

    def fixed_sym(self, v):
        if v < 144:
            self.code(0x30 + v, 8)
        elif v < 256:
            self.code(0x190 + v - 144, 9)
        elif v < 280:
            self.code(v - 256, 7)
        else:
            self.code(0xc0 + v - 280, 8)

    def fixed_block(self, tokens, last):
        """tokens: ints (literals) and (length, distance) pairs; the output is tracked for the Adler-32."""
        self.bits(int(last), 1)
        self.bits(1, 2)
        for t in tokens:
            if isinstance(t, int):
                self.fixed_sym(t)
                self.out.append(t)
                continue
            L, d = t
            c = max(i for i in range(29) if LEN_BASE[i] <= L) if L < 258 else 28
            self.fixed_sym(257 + c)
            self.bits(L - LEN_BASE[c], LEN_EXTRA[c])
            k = max(i for i in range(30) if DIST_BASE[i] <= d)
            self.code(k, 5)
            self.bits(d - DIST_BASE[k], DIST_EXTRA[k])
            for _ in range(L):
                self.out.append(self.out[-d] if d <= len(self.out) else 0)
        self.fixed_sym(256)

    def stored_block(self, data: bytes, last):
        self.bits(int(last), 1)
        self.bits(0, 2)
        self.n = (self.n + 7) // 8 * 8
        self.bits(len(data) | ((len(data) ^ 0xffff) << 16), 32)
        for b in data:
            self.bits(b, 8)
        self.out += data

    def stream(self, adler=None) -> bytes:
        body = self.acc.to_bytes((self.n + 7) // 8, "little")
        a = zlib.adler32(bytes(self.out)) if adler is None else adler
        return self.header + body + struct.pack(">I", a)


# ---- the chunk walk (png_chunks_kernel) ----

def walk_chunks(buf: bytes, H: int, W: int, mode: int):
    """(status, channels, first IDAT chunk's offset, the first IDAT run's data)."""
    n = len(buf)
    if n < 8 or buf[:8] != SIGNATURE:
        return NOT_PNG, 0, -1, b""
    pos, k, C, idat, done, z = 8, 0, 0, -1, False, bytearray()
    while True:
        if n - pos < 12:
            return NOT_PNG, C, idat, bytes(z)
        L, kind = struct.unpack(">I", buf[pos:pos + 4])[0], buf[pos + 4:pos + 8]
        if L > 0x7fffffff or L > n - pos - 12 or not all(chr(c).isalpha() and c < 128 for c in kind):
            return NOT_PNG, C, idat, bytes(z)
        d = buf[pos + 8:pos + 8 + L]
        crc_ok = zlib.crc32(kind + d) == struct.unpack(">I", buf[pos + 8 + L:pos + 12 + L])[0]
        critical = not (kind[0] & 0x20)
        if k == 0:
            if kind != b"IHDR" or L != 13:
                return NOT_PNG, C, idat, bytes(z)
            if not crc_ok:
                return BAD_CRC, C, idat, bytes(z)
            w, h, depth, ct, comp, filt, inter = struct.unpack(">IIBBBBB", d)
            if depth != 8 or ct not in (0, 2, 6) or comp or filt or inter:
                return UNSUPPORTED, C, idat, bytes(z)
            if (w, h) != (W, H):
                return BAD_SHAPE, C, idat, bytes(z)
            C = channels(ct)
        elif kind == b"IHDR":
            return NOT_PNG, C, idat, bytes(z)
        elif kind == b"IEND":            # its CRC is only a warning; bytes after it are not read
            return (NOT_PNG if idat < 0 else OK), C, idat, bytes(z)
        elif critical and not crc_ok:
            return BAD_CRC, C, idat, bytes(z)
        elif kind == b"IDAT":
            if idat < 0:
                idat = pos
            if not done:
                z += d
        else:
            done = done or idat >= 0
            if kind == b"PLTE":
                if C == 1 or idat >= 0:
                    return NOT_PNG, C, idat, bytes(z)
            elif critical:
                return NOT_PNG, C, idat, bytes(z)
            elif (crc_ok and idat < 0 and mode == GREY and C > 1 and
                  ((kind == b"gAMA" and L == 4 and struct.unpack(">I", d)[0] != 100000) or kind in (b"sRGB", b"iCCP"))):
                return UNSUPPORTED, C, idat, bytes(z)
        pos += 12 + L
        k += 1


def pieces(buf: bytes, idat: int, zlen: int):
    """The end (in stream bytes) of every piece libpng hands zlib: each IDAT chunk of the first run in pieces of PIECE bytes."""
    ends, z, pos = [], 0, idat
    while z < zlen:
        L = struct.unpack(">I", buf[pos:pos + 4])[0]
        for o in range(0, L, PIECE):
            ends.append(z + min(L, o + PIECE))
        z += L
        pos += 12 + L
    return ends


# ---- the inflate emulation (png_inflate_kernel) ----

class Table:
    def __init__(self):
        self.fast = [0] * (1 << FAST)
        self.count = [0] * 16
        self.sorted = []


def build_table(lens, kind):
    """inflate_table's verdict and tables of lens: kind 0 the code-length code, 1 literal/length, 2 distance.  None: rejected."""
    T = Table()
    for v in lens:
        T.count[v] += 1
    mx = max([l for l in range(1, 16) if T.count[l]], default=0)
    left, bad = 1, False
    for l in range(1, 16):
        left = (left << 1) - T.count[l]
        bad |= left < 0
    if mx == 0:
        bad = kind != 2
    elif left > 0 and (kind == 0 or mx != 1):
        bad = True
    if bad:
        return None
    T.count[0] = 0
    nxt, c = [0] * 16, 0
    for l in range(1, 16):
        c = (c + T.count[l - 1]) << 1
        nxt[l] = c
    T.sorted = [i for l in range(1, 16) for i in range(len(lens)) if lens[i] == l]
    if left > 0:
        T.fast = [INVALID | 1 << 9] * (1 << FAST)
    for i, l in enumerate(lens):
        if not l:
            continue
        code = int(format(nxt[l], f"0{l}b")[::-1], 2)
        nxt[l] += 1
        if l <= FAST:
            for j in range(code, 1 << FAST, 1 << l):
                T.fast[j] = i | l << 9
    return T


# libpng's phases (png_inflate_kernel): rows still to come; the last row's inflate call; the finishing call's one piece; more
# image data than the image holds, which keeps the finishing call inflating to the stream's end.
IMAGE, LAST_CALL, FINISH, EXTRA = range(4)
FINISH_BUFFER = 1024


class _Stop(Exception):
    def __init__(self, status):
        self.status = status


class Inflater:
    def __init__(self, z: bytes, piece_ends, n: int, row: int):
        self.z, self.zlen, self.zbits, self.cbit = z, len(z), 8 * len(z), 0
        self.ends, self.pi = piece_ends, 0
        self.piece_end = piece_ends[0] if piece_ends else 0
        self.out, self.n, self.row, self.cs_piece, self.phase, self.wsize = 0, n, row, 0, IMAGE, 0
        self.filt = bytearray()          # the image's filtered bytes (output past n is counted, not kept)

    def next_piece(self):
        self.pi += 1
        self.piece_end = self.ends[self.pi] if self.pi < len(self.ends) else self.zlen

    def peek(self, k):
        v = 0
        for i in range(k):
            b = self.cbit + i
            if b < self.zbits:
                v |= ((self.z[b >> 3] >> (b & 7)) & 1) << i
        return v

    def need(self, k):
        """Raise _Stop unless the next k bits can be read (as Inflater::need)."""
        last = (self.cbit + k - 1) >> 3
        if k == 0 or last < self.piece_end:
            return
        if self.phase == FINISH:
            raise _Stop(None)
        self.cs_piece = self.out
        if self.phase == LAST_CALL:
            if self.piece_end >= self.zlen:
                raise _Stop(TOO_LITTLE)
            self.next_piece()
            self.phase = FINISH
            if last >= self.piece_end:
                raise _Stop(None)
            return
        if self.cbit + k > self.zbits:
            raise _Stop(TOO_LITTLE)
        while last >= self.piece_end:
            self.next_piece()

    def start_extra(self):
        if (self.cbit + 7) >> 3 >= self.piece_end:
            if self.piece_end >= self.zlen:
                raise _Stop(TOO_LITTLE)
            self.cs_piece = self.n
            self.next_piece()
        self.phase = EXTRA

    def more_output(self):
        if self.phase == LAST_CALL:
            self.start_extra()
        self.phase = EXTRA

    def call_start(self, p):
        return p - p % self.row if p < self.n else self.n + (p - self.n) // FINISH_BUFFER * FINISH_BUFFER

    def next_boundary(self, p):
        return p - p % self.row + self.row if p < self.n else self.call_start(p) + FINISH_BUFFER

    def bits(self, k):
        self.need(k)
        v = self.peek(k)
        self.cbit += k
        return v

    def decode(self, T):
        e = T.fast[self.peek(FAST)]
        if e:
            l, sym = e >> 9, e & 511
        else:
            v, code, first, index, sym = self.peek(15), 0, 0, 0, INVALID
            for l in range(1, 16):
                code |= (v >> (l - 1)) & 1
                c = T.count[l]
                if code - c < first:
                    sym = T.sorted[index + code - first]
                    break
                index += c
                first = (first + c) << 1
                code <<= 1
        self.need(l)
        self.cbit += l
        return sym


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def inflate(z: bytes, piece_ends, n: int, row: int):
    """(status, filtered bytes of the image written) of a zlib stream read as png_inflate_kernel reads it; n = H * row."""
    I = Inflater(z, piece_ends, n, row)
    try:
        status = _inflate(I, z, n, row)
    except _Stop as s:
        status = s.status
    if status is None or (I.phase >= FINISH and status == BAD_DEFLATE):
        status = OK                      # the finishing call's errors are only warnings
    return status, bytes(I.filt)


def _inflate(I, z, n, row):
    cmf, flg = I.bits(8), I.bits(8)
    if ((cmf << 8) | flg) % 31 or (cmf & 15) != 8 or (cmf >> 4) > 7 or flg & 0x20:
        return BAD_DEFLATE
    I.wsize = 1 << ((cmf >> 4) + 8)
    last = False
    while not last:
        last, kind = I.bits(1), I.bits(2)
        if kind == 3:
            return BAD_DEFLATE
        if kind == 0:
            I.cbit = (I.cbit + 7) // 8 * 8
            v, nv = I.bits(16), I.bits(16)
            if v != (~nv & 0xffff):
                return BAD_DEFLATE
            if v == 0:
                continue
            byte0 = I.cbit >> 3
            if I.phase == LAST_CALL:
                I.start_extra()
            elif I.phase == FINISH:
                if byte0 >= I.piece_end:
                    return None
                I.phase = EXTRA
            if len(z) - byte0 < v:
                return TOO_LITTLE
            pos, left = byte0, v
            if I.phase == IMAGE:
                w = min(left, n - I.out)
                while pos + w > I.piece_end:
                    I.cs_piece = I.out + (I.piece_end - pos)
                    I.next_piece()
                I.filt += z[pos:pos + w]
                I.out, pos, left = I.out + w, pos + w, left - w
                if I.out == n:
                    I.cbit = pos * 8
                    if left == 0:
                        I.phase = LAST_CALL
                    else:
                        I.start_extra()
            if left:
                while pos + left > I.piece_end:
                    I.cs_piece = I.out + (I.piece_end - pos)
                    I.next_piece()
                I.out, pos = I.out + left, pos + left
            I.cbit = pos * 8
            continue
        if kind == 1:
            lit, dist = build_table(FIXED_LIT, 1), build_table([5] * 32, 2)
        else:
            nlen, ndist, ncode = I.bits(5) + 257, I.bits(5) + 1, I.bits(4) + 4
            if nlen > 286 or ndist > 30:
                return BAD_DEFLATE
            cl = [0] * 19
            for i in range(ncode):
                cl[CL_ORDER[i]] = I.bits(3)
            T = build_table(cl, 0)
            if T is None:
                return BAD_DEFLATE
            lens = []
            while len(lens) < nlen + ndist:
                sym = I.decode(T)
                if sym < 16:
                    lens.append(sym)
                    continue
                xb = {16: 2, 17: 3, 18: 7}[sym]
                I.need(xb)
                if sym == 16 and not lens:
                    return BAD_DEFLATE
                rep = I.bits(xb) + (11 if sym == 18 else 3)
                if len(lens) + rep > nlen + ndist:
                    return BAD_DEFLATE
                lens += [lens[-1] if sym == 16 else 0] * rep
            if lens[256] == 0:
                return BAD_DEFLATE
            lit = build_table(lens[:nlen], 1)
            if lit is None:
                return BAD_DEFLATE
            dist = build_table(lens[nlen:], 2)
            if dist is None:
                return BAD_DEFLATE
        while True:
            sym = I.decode(lit)
            if sym >= 286:
                return BAD_DEFLATE
            if sym == 256:
                break
            if sym < 256:
                if I.phase == IMAGE:
                    I.filt.append(sym)
                    I.out += 1
                    if I.out == n:
                        I.phase = LAST_CALL
                else:
                    I.more_output()
                    I.out += 1
                continue
            L = LEN_BASE[sym - 257] + I.bits(LEN_EXTRA[sym - 257])
            ds = I.decode(dist)
            if ds >= 30:
                return BAD_DEFLATE
            d = DIST_BASE[ds] + I.bits(DIST_EXTRA[ds])
            if I.phase != IMAGE:
                I.more_output()
            p = I.out
            cs = max(I.call_start(p), I.cs_piece)
            q, bad = p + L, False
            if d > p - cs + min(I.wsize, cs):
                q, bad = p, True
            elif d > I.wsize and I.next_boundary(p) < q:
                q, bad = I.next_boundary(p), True
            for i in range(p, min(q, n)):
                I.filt.append(I.filt[i - d])
            I.out = q
            if I.phase == IMAGE and q >= n:
                if q > n or bad:
                    I.start_extra()
                else:
                    I.phase = LAST_CALL
            if bad:
                return BAD_DEFLATE
    I.cbit = (I.cbit + 7) // 8 * 8
    a = I.bits(32)
    adler = int.from_bytes(a.to_bytes(4, "little"), "big")
    if I.phase <= LAST_CALL and zlib.adler32(bytes(I.filt)) != adler:
        return BAD_ADLER
    return TOO_LITTLE if I.out < n else OK


# ---- unfilter and convert ----

def unfilter(filt: bytes, H: int, W: int, C: int) -> np.ndarray:
    """uint8 [H, W, C] pixels in PNG order from the filtered bytes (numpy, one row at a time)."""
    rows = np.frombuffer(filt, np.uint8).reshape(H, 1 + W * C)
    out = np.zeros((H, W * C), np.int32)
    prev = np.zeros(W * C, np.int32)
    for y in range(H):
        f, v = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        if f == 0:
            cur = v
        elif f == 1:
            cur = np.cumsum(v.reshape(W, C), axis=0).reshape(-1) & 255
        elif f == 2:
            cur = (v + prev) & 255
        else:
            cur = np.zeros(W * C, np.int32)
            for x in range(W * C):
                left = cur[x - C] if x >= C else 0
                ul = prev[x - C] if x >= C else 0
                pr = (left + prev[x]) >> 1 if f == 3 else int(paeth(left, prev[x], ul))
                cur[x] = (v[x] + pr) & 255
        out[y] = cur
        prev = cur
    return out.astype(np.uint8).reshape(H, W, C)


def convert(pixels: np.ndarray, mode: int) -> np.ndarray:
    """cv2's pixels of PNG-order [H, W, C] pixels: IMREAD_GRAYSCALE [H, W], IMREAD_COLOR BGR [H, W, 3]."""
    C = pixels.shape[-1]
    if mode == GREY:
        return pixels[..., 0].copy() if C == 1 else grey_reference.grey_from_bgr(pixels[..., 2::-1])
    if C == 1:
        return np.repeat(pixels, 3, axis=-1)
    return np.ascontiguousarray(pixels[..., 2::-1])


def model_decode(buf: bytes, mode: int, H=None, W=None, emulate=True):
    """(status, pixels or None) of one file read at H x W (the file's own IHDR when None).  emulate=False takes the stream
    verdict from zlib alone (valid streams only; fast on large files)."""
    if H is None:
        if len(buf) < 24:
            return NOT_PNG, None
        W, H = struct.unpack(">II", buf[16:24])
    status, C, idat, z = walk_chunks(buf, H, W, mode)
    if status != OK:
        return status, None
    row = 1 + W * C
    n = H * row
    if emulate:
        status, filt = inflate(z, pieces(buf, idat, len(z)), n, row)
        if status != OK:
            return status, None
    else:
        filt = zlib.decompressobj().decompress(z)[:n]
        if len(filt) < n:
            return TOO_LITTLE, None
    rows = np.frombuffer(filt, np.uint8)[::row]
    if (rows > 4).any():
        return BAD_FILTER, None
    return OK, convert(unfilter(filt, H, W, C), mode)


# ---- test files ----

def image(rng, H, W, C):
    """Pixels with flat, noisy and repeated parts, so every filter and every kind of token appears."""
    img = rng.integers(0, 256, (H, W, C), np.uint8)
    img[: H // 3] = img[: H // 3] // 16 * 16
    img[H // 3: H // 2, :] = img[H // 3: H // 3 + 1, :]
    return img


def cv2_corpus(rng, sizes=((1, 1), (1, 7), (5, 1), (3, 5), (17, 31), (40, 40), (64, 100))):
    """(name, file) pairs written by cv2.imencode: grey / BGR / BGRA, every compression level and strategy."""
    import cv2
    params = [[]] + [[cv2.IMWRITE_PNG_COMPRESSION, c] for c in range(10)] + [[cv2.IMWRITE_PNG_STRATEGY, s] for s in range(5)]
    out = []
    for H, W in sizes:
        for C in (1, 3, 4):
            img = image(rng, H, W, C)
            for p in params:
                out.append((f"cv2 {H}x{W}x{C} {p}", cv2.imencode(".png", img if C > 1 else img[..., 0], p)[1].tobytes()))
    return out


def zlib_corpus(rng, H=24, W=37):
    """(name, file) pairs of zlib.compressobj streams over every wbits 9-15, strategy and a spread of levels, with row filters
    chosen at random per row, in IDAT chunks of random sizes (down to 1 byte), with ancillary chunks before and after."""
    out = []
    for C, ct in ((1, 0), (3, 2), (4, 6)):
        img = image(rng, H, W, C)
        for wbits in range(9, 16):
            for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
                level = int(rng.integers(0, 10))
                raw = filter_rows(img, rng.integers(0, 5, H))
                co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
                z = co.compress(raw) + co.flush()
                split = int(rng.choice([1, 7, 100, 1000, len(z)]))
                anc = chunk(b"tEXt", b"k\0v") + chunk(b"pHYs", bytes(9))
                out.append((f"zlib C={C} wbits={wbits} strategy={strategy} level={level} split={split}",
                            png_file(H, W, ct, z, split, before=anc, after=anc)))
    return out


def malformed(rng):
    """(name, file, H, W, expected status) of files libpng refuses or only warns about."""
    H, W = 12, 20
    img = image(rng, H, W, 3)
    raw = filter_rows(img, [1] * H)
    n = len(raw)
    z = zlib.compress(raw, 6)
    cases = []

    def add(name, f, st):
        cases.append((name, f, H, W, st))

    add("valid", png_file(H, W, 2, z), OK)
    add("bad signature", b"\x88" + png_file(H, W, 2, z)[1:], NOT_PNG)
    add("truncated file", png_file(H, W, 2, z)[:-20], NOT_PNG)
    add("no IEND", png_file(H, W, 2, z, iend=False), NOT_PNG)
    add("bytes after IEND", png_file(H, W, 2, z) + b"junk", OK)
    add("IHDR CRC", SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0), 7) + chunk(b"IDAT", z) + chunk(b"IEND", b""),
        BAD_CRC)
    idat_bad = SIGNATURE + ihdr(H, W, 2) + chunk(b"IDAT", z, 5) + chunk(b"IEND", b"")
    add("IDAT CRC", idat_bad, BAD_CRC)
    add("ancillary CRC before", png_file(H, W, 2, z, before=chunk(b"tEXt", b"a\0b", 5)), OK)
    add("ancillary CRC after", png_file(H, W, 2, z, after=chunk(b"tEXt", b"a\0b", 5)), OK)
    add("IEND CRC", png_file(H, W, 2, z)[:-4] + b"\0\0\0\0", OK)
    add("unknown critical chunk", png_file(H, W, 2, z, before=chunk(b"ABCD", b"x")), NOT_PNG)
    add("unknown ancillary chunk", png_file(H, W, 2, z, before=chunk(b"abCD", b"x")), OK)
    add("chunk between IDATs", png_file(H, W, 2, z[:50], after=chunk(b"tEXt", b"a\0b") + chunk(b"IDAT", z[50:])), TOO_LITTLE)
    add("16-bit", SIGNATURE + ihdr(H, W, 2, depth=16) + chunk(b"IDAT", z) + chunk(b"IEND", b""), UNSUPPORTED)
    add("interlaced", SIGNATURE + ihdr(H, W, 2, interlace=1) + chunk(b"IDAT", z) + chunk(b"IEND", b""), UNSUPPORTED)
    add("palette", SIGNATURE + ihdr(H, W, 3) + chunk(b"IDAT", z) + chunk(b"IEND", b""), UNSUPPORTED)
    cases.append(("other shape", png_file(H, W, 2, z), H, W + 1, BAD_SHAPE))
    add("bad header check", png_file(H, W, 2, bytes([z[0], z[1] ^ 1]) + z[2:]), BAD_DEFLATE)
    add("preset dictionary", png_file(H, W, 2, bytes([0x78, 0x20 | (31 - (0x7820 % 31))]) + z[2:]), BAD_DEFLATE)
    add("bad Adler-32", png_file(H, W, 2, z[:-1] + bytes([z[-1] ^ 1])), BAD_ADLER)
    add("bad Adler-32 in the next chunk", png_file(H, W, 2, z[:-4], after=chunk(b"IDAT", z[-4:][:3] + bytes([z[-1] ^ 1]))), OK)
    add("no Adler-32", png_file(H, W, 2, z[:-4]), TOO_LITTLE)
    add("truncated stream", png_file(H, W, 2, z[: len(z) // 2]), TOO_LITTLE)
    add("too little data", png_file(H, W, 2, zlib.compress(raw[:-5])), TOO_LITTLE)
    add("too much data", png_file(H, W, 2, zlib.compress(raw + bytes(70))), OK)
    add("bad filter byte", png_file(H, W, 2, zlib.compress(raw[:61] + b"\x05" + raw[62:])), BAD_FILTER)
    for name, build, st in [
        ("block type 3", lambda d: d.bits(0b111, 3), BAD_DEFLATE),
        ("stored length check", lambda d: (d.bits(1, 3), d.bits(0, 5), d.bits(5 | (7 << 16), 32)), BAD_DEFLATE),
        ("literal code 286", lambda d: (d.bits(3, 3), d.fixed_sym(286)), BAD_DEFLATE),
        ("distance code 30", lambda d: (d.bits(3, 3), d.fixed_sym(0), d.fixed_sym(257), d.code(30, 5)), BAD_DEFLATE),
        ("distance before the output", lambda d: (d.bits(3, 3), d.fixed_sym(0), d.fixed_sym(257), d.code(1, 5)), BAD_DEFLATE),
        # dynamic headers: HLIT 257, HDIST 1, HCLEN 4+15, code-length lengths below
        ("oversubscribed code lengths", lambda d: (d.bits(5, 3), d.bits(0, 5), d.bits(0, 5), d.bits(15, 4),
                                                   [d.bits(1, 3) for _ in range(19)]), BAD_DEFLATE),
        ("incomplete code lengths", lambda d: (d.bits(5, 3), d.bits(0, 5), d.bits(0, 5), d.bits(15, 4),
                                               [d.bits(2 if i < 3 else 0, 3) for i in range(19)]), BAD_DEFLATE),
        ("too many length codes", lambda d: (d.bits(5, 3), d.bits(30, 5), d.bits(0, 5), d.bits(15, 4)), BAD_DEFLATE),
    ]:
        d = Deflater()
        build(d)
        add(name, png_file(H, W, 2, d.stream()), st)
    # literal/length lengths: symbols 0..255 and 256 at lengths that over-subscribe / leave incomplete / miss the end of block
    for name, lens, st in [("oversubscribed literal code", [8] * 256 + [8] + [1], BAD_DEFLATE),
                           ("incomplete literal code", [9] * 256 + [9], BAD_DEFLATE),
                           ("no end-of-block code", [8] * 256 + [0] + [8], BAD_DEFLATE),
                           ("incomplete distance code", None, BAD_DEFLATE)]:
        d = Deflater()
        if lens is None:                 # a complete literal code, distances with two codes of length 2: incomplete
            lens, dl = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, [2, 2]
        else:
            dl = [1]
        _dynamic_header(d, lens[:286] if len(lens) > 286 else lens, dl)
        add(name, png_file(H, W, 2, d.stream()), st)
    # libpng's window: a distance past CINFO's window inside one row is accepted, across rows refused
    row = [0] + rng.integers(0, 256, 999).tolist()
    for cinfo, rows, st in [(1, 1, OK), (1, 2, BAD_DEFLATE), (2, 2, OK)]:
        d = Deflater(cinfo)
        if rows == 1:                    # 1000 bytes, then 1000 more from 1000 back (the window is 512)
            toks = row + [(258, 1000)] * 3 + [(226, 1000)]
            Wd = 1999
        else:                            # row 1 is row 0, from 1000 back
            toks = row + [0] + [(258, 1000)] * 3 + [(225, 1000)]
            Wd = 999
        d.fixed_block(toks, True)
        cases.append((f"distance past the window, cinfo={cinfo}, rows={rows}", png_file(rows, Wd, 0, d.stream()), rows, Wd, st))
    # more image data than the image holds, then a truncated stream: the finishing call runs out of IDAT data
    for extra in (1, 70, 300):
        add(f"{extra} bytes too many, then no Adler-32", png_file(H, W, 2, zlib.compress(raw + bytes(extra))[:-4]), TOO_LITTLE)
    # no image data after the last row and half an Adler-32: in later pieces the finishing call stops with one piece, in the
    # same piece the stream runs out
    row32 = b"\0" + bytes((7 * i * i + 3) & 255 for i in range(32))
    co = zlib.compressobj(9, zlib.DEFLATED, 13, 9, zlib.Z_FILTERED)
    z32 = (co.compress(row32) + co.flush())[:-2]
    for split, st in [(1, OK), (3, OK), (None, TOO_LITTLE)]:
        cases.append((f"half an Adler-32, IDAT chunks of {split}", png_file(1, 32, 0, z32, split), 1, 32, st))
    # after the last row: the Adler-32 in the same 8192-byte piece is checked, in the next piece it is not
    for m, st in [(8180, BAD_ADLER), (8185, OK), (8186, BAD_ADLER)]:
        d = Deflater()
        data = b"\0" + rng.integers(0, 256, m - 1, np.uint8).tobytes()
        d.stored_block(data, True)
        s = d.stream()
        s = s[:-4] + bytes([s[-4] ^ 1]) + s[-3:]
        cases.append((f"bad Adler-32 at stream byte {len(s) - 4}", png_file(1, m - 1, 0, s), 1, m - 1, st))
    return cases


def _dynamic_header(d: Deflater, lens, dlens):
    """A dynamic block header for literal/length lengths `lens` and distance lengths `dlens`, every code length sent with a
    4-bit code-length code (lengths 0-15 at length 4), then one end-of-block when the code has one."""
    d.bits(0b101, 3)
    d.bits(len(lens) - 257, 5)
    d.bits(len(dlens) - 1, 5)
    d.bits(15, 4)
    cl = [4 if s < 16 else 0 for s in range(19)]
    for s in CL_ORDER:
        d.bits(cl[s], 3)
    for v in list(lens) + list(dlens):
        d.code(v, 4)


def fuzzed(rng, count):
    """(name, file) pairs of small files whose zlib streams have bit flips, truncation, replaced bytes or appended junk, split
    into IDAT chunks of 1, 3 or 50 bytes or one chunk."""
    out = []
    for k in range(count):
        H, W = int(rng.integers(1, 6)), int(rng.integers(1, 40))
        C, ct = [(1, 0), (3, 2), (4, 6)][k % 3]
        raw = filter_rows(image(rng, H, W, C), rng.integers(0, 5, H))
        co = zlib.compressobj(int(rng.integers(0, 10)), zlib.DEFLATED, int(rng.integers(9, 16)), 9, int(rng.integers(0, 5)))
        z = bytearray(co.compress(raw) + co.flush())
        kind = k % 4
        if kind == 0:
            for _ in range(int(rng.integers(1, 4))):
                i = int(rng.integers(0, len(z) * 8))
                z[i >> 3] ^= 1 << (i & 7)
        elif kind == 1:
            z = z[:int(rng.integers(2, len(z)))]
        elif kind == 2:
            z[int(rng.integers(2, len(z)))] = int(rng.integers(0, 256))
        else:
            z += rng.integers(0, 256, int(rng.integers(1, 20)), np.uint8).tobytes()
        split = [1, 3, 50, None][int(rng.integers(0, 4))]
        out.append((f"fuzz {k}: {H}x{W}x{C} kind {kind} split {split}", png_file(H, W, ct, bytes(z), split)))
    return out
