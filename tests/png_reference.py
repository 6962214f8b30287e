"""Byte model of ``cv2.imencode('.png', img)`` (OpenCV 4.13, libpng, zlib 1.3) and a numpy emulation of the device encoder
(``csrc/png.cu``): the test oracle of ``onepose_b200/png.py``.

``encode`` is the model.  cv2 writes 8-bit grey, BGR or BGRA with libpng's SUB filter on every row (NONE when the image is one
pixel wide: libpng drops SUB there), deflate level 1 with Z_RLE at memLevel 8, the window libpng's ``png_deflate_claim`` picks
from the filtered size, the header ``optimize_cmf`` rewrites, IDAT chunks of 8192 bytes and no ancillary chunks.  The model
feeds one filtered row per ``compress()`` call, as ``png_write_row`` feeds ``deflate(Z_NO_FLUSH)``.

``emulate_zlib`` restates what zlib's ``deflate_rle`` and ``trees.c`` make of those bytes with whole-array operations, in the
decomposition the device uses: greedy distance-1 tokens from run lengths, blocks of 16383 symbols, per-block histograms,
zlib's ``build_tree`` / ``gen_bitlen`` / ``scan_tree`` / ``send_tree``, the stored / fixed / dynamic choice, and bit offsets by
prefix sums.  A block may be stored whenever storing wins: a stored block of 16383 symbols or fewer that beats the fixed
codes spans at most 24575 bytes (DESIGN §5.15), within the 32506 bytes zlib keeps behind its position after a slide, and a
window below 32 KB never slides."""
import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
IDAT_BYTES = 8192
BLOCK_SYMBOLS = 16383          # zlib's sym_end at memLevel 8: (lit_bufsize - 1)
COLOUR_TYPE = {1: 0, 3: 2, 4: 6}


# ---- the model ----

def _as_hwc(img):
    a = np.asarray(img)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3, 4)):
        raise ValueError(f"img must be uint8 [H, W], [H, W, 3] or [H, W, 4], got {a.dtype} {a.shape}")
    return a[:, :, None] if a.ndim == 2 else a


def filtered(img):
    """The filtered rows uint8 [H, 1 + W C]: the filter byte (1 = SUB, 0 = NONE when W = 1), then each byte minus the byte
    one pixel to its left mod 256, the first pixel unchanged; BGR(A) stored as RGB(A)."""
    a = _as_hwc(img)
    H, W, C = a.shape
    if C >= 3:
        a = a[:, :, [2, 1, 0, 3][:C]]
    rows = np.ascontiguousarray(a).reshape(H, W * C)
    f = rows.copy()
    f[:, C:] = rows[:, C:] - rows[:, :-C]
    return np.concatenate([np.full((H, 1), 1 if W > 1 else 0, np.uint8), f], axis=1)


def window_bits(n):
    """png_deflate_claim: 15, halved while n + 262 fits in the half window when n <= 16384; zlib runs 8 as 9."""
    wb = 15
    if n <= 16384:
        half = 1 << (wb - 1)
        while n + 262 <= half:
            half >>= 1
            wb -= 1
    return max(wb, 9)


def optimize_cmf(z, n):
    """libpng's optimize_cmf: the CINFO nibble from the data size alone (no +262), FCHECK recomputed."""
    z = bytearray(z)
    if n <= 16384 and (z[0] & 0x0F) == 8 and (z[0] & 0xF0) <= 0x70:
        cinfo = z[0] >> 4
        half = 1 << (cinfo + 7)
        if n <= half:
            while True:
                half >>= 1
                cinfo -= 1
                if not (cinfo > 0 and n <= half):
                    break
            z[0] = (z[0] & 0x0F) | (cinfo << 4)
            t = z[1] & 0xE0
            z[1] = t + 0x1F - ((z[0] << 8) + t) % 0x1F
    return bytes(z)


def zlib_stream(filt):
    """zlib.compressobj(1, DEFLATED, window_bits, 8, Z_RLE) fed one row per call, with optimize_cmf's header."""
    n = filt.size
    co = zlib.compressobj(1, zlib.DEFLATED, window_bits(n), 8, zlib.Z_RLE)
    z = b"".join(co.compress(r.tobytes()) for r in filt) + co.flush()
    return optimize_cmf(z, n)


def chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))


def frame_png(z, H, W, C):
    """Signature, IHDR, the zlib stream in IDAT chunks of 8192 bytes, IEND."""
    out = [SIGNATURE, chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, COLOUR_TYPE[C], 0, 0, 0))]
    out += [chunk(b"IDAT", z[i:i + IDAT_BYTES]) for i in range(0, len(z), IDAT_BYTES)]
    out.append(chunk(b"IEND", b""))
    return b"".join(out)


def encode(img):
    """The bytes cv2.imencode('.png', img)[1] holds."""
    a = _as_hwc(img)
    H, W, C = a.shape
    return frame_png(zlib_stream(filtered(a)), H, W, C)


def deflate_bound(n):
    """zlib 1.3's deflateBound for level 1, memLevel 8 and window_bits(n) with the zlib wrapper."""
    if window_bits(n) == 15:
        return n + (n >> 12) + (n >> 14) + (n >> 25) + 13
    return n + (n >> 3) + (n >> 8) + (n >> 9) + 4 + 6


def png_bound(n):
    """The most bytes a frame of n filtered bytes takes: deflateBound, 12 per IDAT chunk, 45 for signature, IHDR and IEND."""
    z = deflate_bound(n)
    return z + 12 * ((z + IDAT_BYTES - 1) // IDAT_BYTES) + 45


# ---- the emulation of the device encoder ----

EXTRA_LBITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
BASE_LENGTH = [0]
for _c in range(28):
    BASE_LENGTH.append(BASE_LENGTH[-1] + (1 << EXTRA_LBITS[_c]))
BASE_LENGTH[28] = 255          # code 285: match length 258 without extra bits (zlib's tr_static_init)
LENGTH_CODE = np.zeros(256, np.int64)
for _c in range(28):
    LENGTH_CODE[BASE_LENGTH[_c]:BASE_LENGTH[_c] + (1 << EXTRA_LBITS[_c])] = _c
LENGTH_CODE[255] = 28
STATIC_LLEN = np.array([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
STATIC_DLEN = np.full(30, 5)


def tokens(s):
    """deflate_rle's greedy tokens of the byte string s (uint8 [n]): (position, length) per token, length 1 for a literal.
    Within a run of L equal bytes the first is a literal; the L - 1 repeats become matches of 258 while 258 remain, then one
    match of the rest if it is 3 or more, else literals.  Runs are found by comparison with the left neighbour."""
    n = s.size
    i = np.arange(n)
    head = np.ones(n, bool)
    head[1:] = s[1:] != s[:-1]
    start = np.maximum.accumulate(np.where(head, i, 0))
    nxt = np.where(np.r_[head[1:], True], i + 1, n)              # position after i when i ends a run
    end = np.minimum.accumulate(nxt[::-1])[::-1]
    k = i - start
    r = end - start - 1
    q, m = r // 258, r % 258
    j = k - 1
    c, t = j // 258, j % 258
    full = (k >= 1) & (c < q) & (t == 0)
    last = (k >= 1) & (c == q)
    tail_match = last & (m >= 3) & (t == 0)
    tail_lit = last & (m < 3)
    first = k == 0
    is_tok = first | full | tail_match | tail_lit
    length = np.where(full, 258, np.where(tail_match, m, 1))
    return i[is_tok], length[is_tok]


def _pqdownheap(heap, heap_len, freq, depth, k):
    v = heap[k]
    j = k << 1
    while j <= heap_len:
        if j < heap_len and (freq[heap[j + 1]] < freq[heap[j]] or
                             (freq[heap[j + 1]] == freq[heap[j]] and depth[heap[j + 1]] <= depth[heap[j]])):
            j += 1
        if freq[v] < freq[heap[j]] or (freq[v] == freq[heap[j]] and depth[v] <= depth[heap[j]]):
            break
        heap[k] = heap[j]
        k = j
        j <<= 1
    heap[k] = v


def build_tree(freq_in, stree, extra, base, max_length):
    """zlib's build_tree and gen_bitlen: code lengths, max_code and the opt_len / static_len contributions."""
    elems = len(freq_in)
    freq = [0] * (2 * elems + 1)
    freq[:elems] = [int(f) for f in freq_in]
    depth = [0] * (2 * elems + 1)
    dad = [0] * (2 * elems + 1)
    ln = [0] * (2 * elems + 1)
    heap_size = 2 * 286 + 1
    heap = [0] * heap_size
    heap_len, heap_max = 0, heap_size
    opt = stat = 0
    max_code = -1
    for n in range(elems):
        if freq[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
    while heap_len < 2:
        if max_code < 2:
            max_code += 1
            node = max_code
        else:
            node = 0
        heap_len += 1
        heap[heap_len] = node
        freq[node] = 1
        depth[node] = 0
        opt -= 1
        if stree is not None:
            stat -= int(stree[node])
    for n in range(heap_len // 2, 0, -1):
        _pqdownheap(heap, heap_len, freq, depth, n)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[heap_len]
        heap_len -= 1
        _pqdownheap(heap, heap_len, freq, depth, 1)
        m = heap[1]
        heap_max -= 1
        heap[heap_max] = n
        heap_max -= 1
        heap[heap_max] = m
        freq[node] = freq[n] + freq[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        _pqdownheap(heap, heap_len, freq, depth, 1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]
    # gen_bitlen
    bl_count = [0] * (max_length + 1)
    ln[heap[heap_max]] = 0
    overflow = 0
    for h in range(heap_max + 1, heap_size):
        n = heap[h]
        bits = ln[dad[n]] + 1
        if bits > max_length:
            bits = max_length
            overflow += 1
        ln[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xbits = extra[n - base] if n >= base else 0
        opt += freq[n] * (bits + xbits)
        if stree is not None:
            stat += freq[n] * (int(stree[n]) + xbits)
    if overflow:
        while overflow > 0:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
        h = heap_size
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if ln[m] != bits:
                    opt += (bits - ln[m]) * freq[m]
                    ln[m] = bits
                n -= 1
    lens = np.array([ln[n] if n <= max_code and freq[n] else 0 for n in range(elems)])
    return lens, max_code, opt, stat


def canonical_codes(lens):
    """gen_codes: the canonical code of each length, bit-reversed for LSB-first output."""
    lens = np.asarray(lens)
    bl_count = np.bincount(lens, minlength=16)
    bl_count[0] = 0
    next_code, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + int(bl_count[b - 1])) << 1
        next_code[b] = code
    codes = np.zeros(len(lens), np.int64)
    for n, L in enumerate(lens):
        if L:
            c = next_code[L]
            next_code[L] += 1
            codes[n] = int(format(c, f"0{L}b")[::-1], 2)
    return codes


def _tree_runs(lens, max_code):
    """scan_tree / send_tree's run encoding of lens[0 .. max_code]: (symbol, extra value, extra bits) per item."""
    out = []
    prevlen, nextlen, count = -1, int(lens[0]), 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        curlen = nextlen
        nextlen = int(lens[n + 1]) if n + 1 <= max_code else 0xFFFF
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            out += [(curlen, 0, 0)] * count
        elif curlen != 0:
            if curlen != prevlen:
                out.append((curlen, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


def block_codes(lfreq, dfreq):
    """_tr_flush_block's trees for one block: (lit lens, dist lens, header items [(value, bits)], opt_len, static_len)."""
    llens, lmax, lopt, lstat = build_tree(lfreq, STATIC_LLEN, EXTRA_LBITS, 257, 15)
    dlens, dmax, dopt, dstat = build_tree(dfreq, STATIC_DLEN, EXTRA_DBITS, 0, 15)
    runs = _tree_runs(llens, lmax) + _tree_runs(dlens, dmax)
    blfreq = np.bincount([r[0] for r in runs], minlength=19)
    bllens, _, blopt, _ = build_tree(blfreq, None, EXTRA_BLBITS, 0, 7)
    max_blindex = 18
    while max_blindex >= 3 and bllens[BL_ORDER[max_blindex]] == 0:
        max_blindex -= 1
    opt = lopt + dopt + blopt + 3 * (max_blindex + 1) + 5 + 5 + 4
    blcodes = canonical_codes(bllens)
    header = [(lmax + 1 - 257, 5), (dmax + 1 - 1, 5), (max_blindex + 1 - 4, 4)]
    header += [(int(bllens[BL_ORDER[r]]), 3) for r in range(max_blindex + 1)]
    for sym, xv, xb in runs:
        header.append((int(blcodes[sym]), int(bllens[sym])))
        if xb:
            header.append((xv, xb))
    return llens, dlens, header, opt, lstat + dstat


def _pack(values, bits):
    """LSB-first bit string of the (value, bit count) items, as zlib's send_bits."""
    values = np.asarray(values, np.int64)
    bits = np.asarray(bits, np.int64)
    total = int(bits.sum())
    if total == 0:
        return np.zeros(0, np.uint8)
    owner = np.repeat(np.arange(len(bits)), bits)
    within = np.arange(total) - np.repeat(np.cumsum(bits) - bits, bits)
    return ((values[owner] >> within) & 1).astype(np.uint8)


def adler32(s):
    s = s.astype(np.int64)
    n = s.size
    a = (1 + int(s.sum())) % 65521
    b = (n + int(((n - np.arange(n)) * s).sum())) % 65521
    return (b << 16) | a


def emulate_zlib(filt):
    """The zlib stream (with optimize_cmf's header) the device writes for the filtered rows: equal to zlib_stream(filt)."""
    s = np.ascontiguousarray(filt).reshape(-1)
    n = s.size
    pos, length = tokens(s)
    match = length >= 3
    sym = np.where(match, 257 + LENGTH_CODE[np.maximum(length - 3, 0)], s[pos].astype(np.int64))
    T = pos.size
    nblocks = T // BLOCK_SYMBOLS + 1
    bitstream = []
    for k in range(nblocks):
        a, b = k * BLOCK_SYMBOLS, min((k + 1) * BLOCK_SYMBOLS, T)
        last = k == nblocks - 1
        bsym, bmatch, blen = sym[a:b], match[a:b], length[a:b]
        lfreq = np.bincount(bsym, minlength=286)
        lfreq[256] += 1
        dfreq = np.zeros(30, np.int64)
        dfreq[0] = int(bmatch.sum())
        llens, dlens, header, opt, stat = block_codes(lfreq, dfreq)
        opt_lenb, static_lenb = (opt + 3 + 7) >> 3, (stat + 3 + 7) >> 3
        opt_lenb = min(opt_lenb, static_lenb)
        start = int(pos[a]) if b > a else n
        stored_len = (int(pos[b - 1] + blen[-1]) if b > a else n) - start
        if stored_len + 4 <= opt_lenb:
            bitstream.append(_pack([last], [3]))
            used = sum(x.size for x in bitstream) + 16
            pad = -used % 8
            data = np.r_[np.array([stored_len & 255, stored_len >> 8, ~stored_len & 255, (~stored_len >> 8) & 255], np.int64),
                         s[start:start + stored_len].astype(np.int64)]
            bitstream.append(np.r_[np.zeros(pad, np.uint8), _pack(data, np.full(data.size, 8))])
            continue
        if static_lenb == opt_lenb:
            bitstream.append(_pack([2 + last], [3]))
            llens, dlens = STATIC_LLEN, STATIC_DLEN
        else:
            bitstream.append(_pack([4 + last] + [v for v, _ in header], [3] + [w for _, w in header]))
        lcodes, dcodes = canonical_codes(llens), canonical_codes(dlens)
        xl = np.where(bmatch, np.array(EXTRA_LBITS)[np.maximum(bsym - 257, 0)], 0)
        xv = np.where(bmatch, np.maximum(blen - 3, 0) - np.array(BASE_LENGTH)[np.maximum(bsym - 257, 0)], 0)
        vals = np.stack([lcodes[bsym], xv, np.full(bsym.size, dcodes[0])], 1).reshape(-1)
        nb = np.stack([llens[bsym], xl, np.where(bmatch, dlens[0], 0)], 1).reshape(-1)
        bitstream.append(_pack(np.r_[vals, lcodes[256]], np.r_[nb, llens[256]]))
    bits = np.concatenate(bitstream)
    body = np.packbits(np.r_[bits, np.zeros(-bits.size % 8, np.uint8)], bitorder="little").tobytes()
    wb = window_bits(n)
    cmf = ((wb - 8) << 4) | 8
    head = bytes([cmf, 0x1F - (cmf << 8) % 0x1F])
    return optimize_cmf(head + body + struct.pack(">I", adler32(s)), n)


def fibonacci_row():
    """A one-row grey image whose SUB-filtered bytes hold literal counts 2, 3, 5, 8, ... (no byte next to an equal one, so
    every byte is a literal): with the filter byte and the end-of-block code (one each), zlib's Huffman tree for them is one
    chain deeper than 15 bits and gen_bitlen's repair runs."""
    counts = [2, 3]
    while sum(counts) + counts[-1] + counts[-2] < 16000:
        counts.append(counts[-1] + counts[-2])
    syms = np.arange(len(counts)) * 7 + 2
    seq = np.repeat(syms[::-1], counts[::-1])
    d = np.empty_like(seq)
    half = (seq.size + 1) // 2
    d[0::2], d[1::2] = seq[:half], seq[half:]
    return np.cumsum(d.astype(np.uint64)).astype(np.uint8)[None, :]       # row 0's SUB bytes are d
