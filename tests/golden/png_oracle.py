"""Host restatement, from the format definitions, of the PNG file `tecogan_b200/csrc/png.cu` writes for an RGB uint8
frame (the bytes `cv2.imwrite` writes: libpng with zlib's run-length strategy, `tests/test_png_host.py` pins both).

Stages, each one a step of the device encoder:
  filter_stream  rows -> S: filter byte 1 (Sub, bpp 3) and the byte differences; rows of width 1 use filter 0 (None)
  tokenize       S -> literals and distance-1 matches: each maximal run of equal bytes is a literal, then matches of
                 258 over the rest of the run, then one match of the remainder if it is at least 3, else literals
  split_blocks   a block ends after every 16 383 symbols and after the last one (an exact multiple leaves an empty
                 final block)
  build_tree     deflate's length-limited Huffman code as zlib's trees.c builds it: a binary heap ordered by
                 (frequency, depth), at least two codes per tree, over-long codes pushed back to the limit
  block_choice   stored, static or dynamic: the shortest, ties going to static over dynamic and stored first
  zlib_stream    2-byte header (window bits from the filtered size), the blocks bit-packed LSB first, Adler-32
  png_file       signature, IHDR, the stream cut into 8 192-byte IDAT chunks, IEND
Plain Python and numpy; slow but exact, for frames up to a few megabytes.
"""
import struct

import numpy as np

BLOCK_SYMBOLS = 16383                     # symbols per deflate block (zlib's literal buffer of 16 384, minus one)
IDAT_BYTES = 8192
MAX_BITS, MAX_BL_BITS = 15, 7
L_CODES, D_CODES, BL_CODES = 286, 30, 19
END_BLOCK = 256
BL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258)
LEN_EXTRA = (0,) * 8 + (1,) * 4 + (2,) * 4 + (3,) * 4 + (4,) * 4 + (5,) * 4 + (0,)
BL_EXTRA = (0,) * 16 + (2, 3, 7)
STATIC_LLEN = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8       # RFC 1951 3.2.6, 288 codes
STATIC_DLEN = [5] * 30


def length_code(length):
    """Match length 3..258 -> (index 0..28 of the length code 257 + index, extra bits value, extra bit count)."""
    if length == 258:
        return 28, 0, 0
    i = max(k for k in range(28) if LEN_BASE[k] <= length)
    return i, length - LEN_BASE[i], LEN_EXTRA[i]


# ---------------------------------------------------------------------------------------------------- filter, tokens
def filter_stream(rgb):
    """[H, W, 3] uint8 RGB -> S: per row the filter byte, then the row's bytes (Sub differences when W > 1)."""
    h, w, _ = rgb.shape
    rows = rgb.reshape(h, 3 * w).astype(np.int32)
    if w > 1:
        rows = np.concatenate([rows[:, :3], (rows[:, 3:] - rows[:, :-3]) & 255], axis=1)
    ftype = np.full((h, 1), 1 if w > 1 else 0, np.int32)
    return np.concatenate([ftype, rows], axis=1).reshape(-1).astype(np.uint8)


def tokenize(s):
    """S -> list of tokens: (0, byte) literal or (1, length) distance-1 match."""
    s = np.asarray(s, np.uint8)
    starts = np.flatnonzero(np.concatenate([[True], s[1:] != s[:-1]]))
    ends = np.append(starts[1:], len(s))
    out = []
    for r, e in zip(starts.tolist(), ends.tolist()):
        b = int(s[r])
        out.append((0, b))
        tail = e - r - 1
        out += [(1, 258)] * (tail // 258)
        rem = tail % 258
        if rem >= 3:
            out.append((1, rem))
        else:
            out += [(0, b)] * rem
    return out


def split_blocks(tokens):
    nb = len(tokens) // BLOCK_SYMBOLS + 1
    return [tokens[i * BLOCK_SYMBOLS:(i + 1) * BLOCK_SYMBOLS] for i in range(nb)]


# ---------------------------------------------------------------------------------------------------- Huffman trees
def build_tree(freq, max_length, static_len=None, extra=None, extra_base=0):
    """freq: list of symbol counts.  Returns (lens, max_code, opt, stat):
    code lengths, the largest code with a length, and the bits of the symbols under this code and under `static_len`
    (extra bits included)."""
    elems = len(freq)
    nodes = 2 * elems + 1
    f = list(freq) + [0] * (nodes - elems)
    depth = [0] * nodes
    dad = [0] * nodes
    heap = [0] * nodes
    heap_len, heap_max = 0, nodes
    max_code = -1
    opt = stat = 0
    for n in range(elems):
        if f[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
    while heap_len < 2:                     # a tree has at least two codes: add code max_code + 1 while < 2, else 0
        if max_code < 2:
            max_code += 1
            node = max_code
        else:
            node = 0
        heap_len += 1
        heap[heap_len] = node
        f[node] = 1
        opt -= 1
        if static_len is not None:
            stat -= static_len[node]

    def smaller(a, b):
        return f[a] < f[b] or (f[a] == f[b] and depth[a] <= depth[b])

    def down(k):
        v = heap[k]
        j = k << 1
        while j <= heap_len:
            if j < heap_len and smaller(heap[j + 1], heap[j]):
                j += 1
            if smaller(v, heap[j]):
                break
            heap[k] = heap[j]
            k = j
            j <<= 1
        heap[k] = v

    for k in range(heap_len // 2, 0, -1):
        down(k)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[heap_len]
        heap_len -= 1
        down(1)
        m = heap[1]
        heap_max -= 1
        heap[heap_max] = n
        heap_max -= 1
        heap[heap_max] = m
        f[node] = f[n] + f[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        down(1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]

    # lengths from the root down, clamped at max_length
    lens = [0] * nodes
    bl_count = [0] * (max_length + 1)
    overflow = 0
    for h in range(heap_max + 1, nodes):
        n = heap[h]
        bits = lens[dad[n]] + 1
        if bits > max_length:
            bits = max_length
            overflow += 1
        lens[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xb = extra[n - extra_base] if extra is not None and n >= extra_base else 0
        opt += f[n] * (bits + xb)
        if static_len is not None:
            stat += f[n] * (static_len[n] + xb)
    if overflow:
        while overflow > 0:                 # move a leaf down from the deepest level that has one above the limit
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
        h = nodes                           # hand the new lengths out in heap order (most frequent last)
        for bits in range(max_length, 0, -1):
            cnt = bl_count[bits]
            while cnt:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if lens[m] != bits:
                    opt += (bits - lens[m]) * f[m]
                    lens[m] = bits
                cnt -= 1
    return lens[:elems], max_code, opt, stat


def canonical_codes(lens):
    """Code lengths -> bit-reversed canonical codes (deflate sends Huffman codes most significant bit first)."""
    bl_count = [0] * (MAX_BITS + 1)
    for l in lens:
        if l:
            bl_count[l] += 1
    nxt = [0] * (MAX_BITS + 1)
    code = 0
    for bits in range(1, MAX_BITS + 1):
        code = (code + bl_count[bits - 1]) << 1
        nxt[bits] = code
    codes = [0] * len(lens)
    for n, l in enumerate(lens):
        if l:
            c = nxt[l]
            nxt[l] += 1
            codes[n] = int(format(c, "0%db" % l)[::-1], 2)
    return codes


def length_runs(lens, max_code):
    """Run-length code of lens[0..max_code] with the bit-length alphabet: list of (symbol, extra value, extra bits)."""
    out = []
    prev = -1
    n = 0
    count = 0
    nextlen = lens[0]
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        cur = nextlen
        nextlen = lens[n + 1] if n < max_code else -1
        count += 1
        if count < max_count and cur == nextlen:
            continue
        if count < min_count:
            out += [(cur, 0, 0)] * count
        elif cur != 0:
            if cur != prev:
                out.append((cur, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count = 0
        prev = cur
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif cur == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


# ---------------------------------------------------------------------------------------------------- blocks
class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, value, bits):
        self.acc |= value << self.n
        self.n += bits
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)


def block_plan(block):
    """One block's trees and its bit counts.  Returns a dict with kind 'stored' | 'static' | 'dynamic'."""
    lfreq = [0] * L_CODES
    dfreq = [0] * D_CODES
    lfreq[END_BLOCK] = 1
    for kind, v in block:
        if kind == 0:
            lfreq[v] += 1
        else:
            lfreq[257 + length_code(v)[0]] += 1
            dfreq[0] += 1
    llens, lmax, lopt, lstat = build_tree(lfreq, MAX_BITS, STATIC_LLEN, LEN_EXTRA, 257)
    dlens, dmax, dopt, dstat = build_tree(dfreq, MAX_BITS, STATIC_DLEN, None, 0)
    runs = length_runs(llens, lmax) + length_runs(dlens, dmax)
    blfreq = [0] * BL_CODES
    for sym, _, _ in runs:
        blfreq[sym] += 1
    bllens, _, blopt, _ = build_tree(blfreq, MAX_BL_BITS, None, BL_EXTRA, 0)
    max_blindex = max([3] + [i for i in range(3, BL_CODES) if bllens[BL_ORDER[i]]])
    opt = lopt + dopt + blopt + 3 * (max_blindex + 1) + 5 + 5 + 4
    stat = lstat + dstat
    opt_bytes = (opt + 3 + 7) >> 3
    static_bytes = (stat + 3 + 7) >> 3
    stored_len = sum(1 if k == 0 else v for k, v in block)
    if static_bytes <= opt_bytes:
        opt_bytes = static_bytes
    if stored_len + 4 <= opt_bytes:
        kind = "stored"
    elif static_bytes == opt_bytes:
        kind = "static"
    else:
        kind = "dynamic"
    return dict(kind=kind, llens=llens, lmax=lmax, dlens=dlens, dmax=dmax, bllens=bllens, runs=runs,
                max_blindex=max_blindex, stored_len=stored_len)


def write_block(bw, block, plan, raw, last):
    kind = plan["kind"]
    if kind == "stored":
        bw.put(last, 3)
        bw.align()
        n = plan["stored_len"]
        bw.put(n, 16)
        bw.put(n ^ 0xFFFF, 16)
        for b in raw:
            bw.put(int(b), 8)
        return
    if kind == "static":
        bw.put(2 + last, 3)
        llens, dlens = STATIC_LLEN, STATIC_DLEN
    else:
        bw.put(4 + last, 3)
        bl = plan["bllens"]
        bw.put(plan["lmax"] + 1 - 257, 5)
        bw.put(plan["dmax"] + 1 - 1, 5)
        bw.put(plan["max_blindex"] + 1 - 4, 4)
        for i in range(plan["max_blindex"] + 1):
            bw.put(bl[BL_ORDER[i]], 3)
        blcodes = canonical_codes(bl)
        for sym, xv, xb in plan["runs"]:
            bw.put(blcodes[sym], bl[sym])
            if xb:
                bw.put(xv, xb)
        llens, dlens = plan["llens"], plan["dlens"]
    lcodes, dcodes = canonical_codes(llens), canonical_codes(dlens)
    for kind_, v in block:
        if kind_ == 0:
            bw.put(lcodes[v], llens[v])
        else:
            i, xv, xb = length_code(v)
            bw.put(lcodes[257 + i], llens[257 + i])
            if xb:
                bw.put(xv, xb)
            bw.put(dcodes[0], dlens[0])
    bw.put(lcodes[END_BLOCK], llens[END_BLOCK])


def deflate_rle(s):
    """Raw deflate body of S (no zlib header or trailer)."""
    s = np.asarray(s, np.uint8)
    bw = BitWriter()
    blocks = split_blocks(tokenize(s))
    pos = 0
    for i, blk in enumerate(blocks):
        plan = block_plan(blk)
        n = plan["stored_len"]
        write_block(bw, blk, plan, s[pos:pos + n], 1 if i == len(blocks) - 1 else 0)
        pos += n
    bw.align()
    return bytes(bw.out)


# ---------------------------------------------------------------------------------------------------- zlib, PNG
def window_bits(n):
    """Window bits in the zlib header for n filtered bytes: the smallest window holding them, between 8 and 15."""
    w = 8
    while w < 15 and (1 << w) < n:
        w += 1
    return w


def zlib_header(n):
    cmf = ((window_bits(n) - 8) << 4) | 8
    flg = 31 - (cmf * 256) % 31                # FLEVEL 0, no dictionary
    return bytes([cmf, flg])


def adler32(s):
    s = np.asarray(s, np.uint8).astype(np.int64)
    n = len(s)
    a = (1 + int(s.sum())) % 65521
    b = (n + int(((n - np.arange(n)) * s).sum())) % 65521
    return (b << 16) | a


_CRC = []
for _i in range(256):
    _c = _i
    for _ in range(8):
        _c = (_c >> 1) ^ 0xEDB88320 if _c & 1 else _c >> 1
    _CRC.append(_c)


def crc32(data):
    c = 0xFFFFFFFF
    for b in data:
        c = _CRC[(c ^ b) & 255] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", crc32(tag + data))


def zlib_stream(s):
    return zlib_header(len(s)) + deflate_rle(s) + struct.pack(">I", adler32(s))


def png_file(rgb):
    """[H, W, 3] uint8 RGB -> the PNG file's bytes."""
    h, w, _ = rgb.shape
    z = zlib_stream(filter_stream(rgb))
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
    for i in range(0, len(z), IDAT_BYTES):
        out += chunk(b"IDAT", z[i:i + IDAT_BYTES])
    return out + chunk(b"IEND", b"")


def unfilter_sub(s, h, w):
    """Inverse of filter_stream for W > 1: the RGB frame whose filtered stream is S (S's filter bytes must be 1)."""
    rows = np.asarray(s, np.uint8).reshape(h, 3 * w + 1)
    assert (rows[:, 0] == 1).all()
    d = rows[:, 1:].astype(np.int64).reshape(h, w, 3)
    return (np.cumsum(d, axis=1) & 255).astype(np.uint8)
