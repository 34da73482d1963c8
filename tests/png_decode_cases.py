"""PNG files for the device decoder's tests (tests/test_png_decode_host.py, tests/test_gpu_png_decode.py): what
cv2.imwrite writes at every compression level and strategy, and -- from a writer here -- what it never writes: chosen
filter types, every colour type and bit depth the device takes, zlib levels and window sizes, flush points, split and
empty IDAT chunks among ancillary chunks, and one file per class the device hands back to cv2.  numpy, zlib and cv2."""
import os
import struct
import zlib

import numpy as np

from tests import png_cases as PC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CALENDAR = [os.path.join(GOLDEN, "calendar_lr_%04d.png" % k) for k in (1, 2)]   # reference LR/calendar, 8-bit RGB, Sub
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(kind)))


def ihdr(h, w, colour, depth, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, colour, 0, 0, interlace))


def pack_rows(px, w, colour, depth):
    """[h, w * channels] sample values -> [h, rowbytes] packed bytes (samples below 8 bits MSB first)."""
    px = np.asarray(px, np.int64)
    h = px.shape[0]
    if depth == 8:
        return px.astype(np.uint8)
    bits = np.zeros((h, px.shape[1] * depth), np.uint8)
    for k in range(depth):
        bits[:, k::depth] = (px >> (depth - 1 - k)) & 1
    return np.packbits(bits, axis=1)


def filter_rows(rows, bpp, types):
    """Unfiltered [h, rowbytes] rows -> filtered bytes (filter byte + row) with types[y] per row."""
    h, rb = rows.shape
    out = np.zeros((h, rb + 1), np.uint8)
    r = rows.astype(np.int64)
    for y in range(h):
        f = types[y % len(types)]
        up = r[y - 1] if y else np.zeros(rb, np.int64)
        left = np.concatenate([np.zeros(bpp, np.int64), r[y, :-bpp]]) if rb > bpp else np.zeros(rb, np.int64)
        left = left[:rb]
        ul = np.concatenate([np.zeros(bpp, np.int64), up[:-bpp]])[:rb] if rb > bpp else np.zeros(rb, np.int64)
        if f == 0:
            pred = 0
        elif f == 1:
            pred = left
        elif f == 2:
            pred = up
        elif f == 3:
            pred = (left + up) >> 1
        else:
            p = left + up - ul
            pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
            pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
        out[y, 0] = f
        out[y, 1:] = (r[y] - pred) & 255
    return out.tobytes()


def compress(raw, level=6, wbits=15, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits)
    if not flush_every:
        return c.compress(raw) + c.flush()
    out = b""
    for k in range(0, len(raw), flush_every):
        out += c.compress(raw[k:k + flush_every]) + c.flush(flush)
    return out + c.flush()


def png_file(h, w, colour, depth, zdata, plte=None, split=None, before=(), between=(), after=(), interlace=0):
    """A PNG file around `zdata`: `before` chunks after IHDR, the PLTE, `between` chunks, IDAT chunks of `split` bytes
    (None: one chunk; 0: alternating 1-byte and empty chunks), `after` chunks, IEND."""
    out = b"\x89PNG\r\n\x1a\n" + ihdr(h, w, colour, depth, interlace) + b"".join(before)
    if plte is not None:
        out += chunk(b"PLTE", bytes(np.asarray(plte, np.uint8).reshape(-1)))
    out += b"".join(between)
    if split is None:
        parts = [zdata]
    elif split == 0:
        parts = []
        for b in zdata:
            parts += [bytes([b]), b""]
    else:
        parts = [zdata[k:k + split] for k in range(0, len(zdata), split)] or [b""]
    return out + b"".join(chunk(b"IDAT", p) for p in parts) + b"".join(after) + chunk(b"IEND", b"")


def image(h, w, colour, depth, seed, plte_n=None):
    """Seeded samples [h, w * channels] and the palette (colour type 3)."""
    g = np.random.default_rng(seed)
    ch = CHANNELS[colour]
    hi = (1 << depth) if colour != 3 else min(1 << depth, plte_n or (1 << depth))
    base = PC.smooth(h, w, seed).astype(np.int64)
    if colour in (2, 6, 4, 0) and depth == 8:
        px = np.concatenate([base, g.integers(0, 256, (h, w, 1))], 2)[:, :, :ch] if ch != 1 else base[:, :, :1]
        if colour == 4:
            px = np.concatenate([base[:, :, :1], g.integers(0, 256, (h, w, 1))], 2)
        px = px.reshape(h, w * ch)
    else:
        px = (base[:, :, 0] * hi // 256).reshape(h, w)
    plte = g.integers(0, 256, (plte_n or (1 << depth), 3)) if colour == 3 else None
    return px, plte


def made(h, w, colour, depth, seed, types=(1,), level=6, wbits=15, plte_n=None, **kw):
    px, plte = image(h, w, colour, depth, seed, plte_n)
    rows = pack_rows(px, w, colour, depth)
    bpp = max(1, CHANNELS[colour] * depth // 8)
    raw = filter_rows(rows, bpp, types)
    zkw = {k: kw.pop(k) for k in ("flush_every", "flush") if k in kw}
    return png_file(h, w, colour, depth, compress(raw, level, wbits, **zkw), plte, **kw)


class _BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):                                 # LSB first
        self.bits += [(v >> k) & 1 for k in range(n)]

    def code(self, c, n):                                # Huffman codes go MSB first
        self.bits += [(c >> (n - 1 - k)) & 1 for k in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def bytes(self):
        self.align()
        b = np.packbits(np.array(self.bits, np.uint8).reshape(-1, 8)[:, ::-1], axis=1).reshape(-1)
        return b.tobytes()


def _canonical(lengths):
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = []
    for l in lengths:
        out.append((nxt[l], l) if l else None)
        if l:
            nxt[l] += 1
    return out


def _index(bases, v):
    return max(i for i, b in enumerate(bases) if b <= v)


def deflate_tokens(tokens, lit_lens=None, dist_lens=None, cl_syms=None, wbits=15):
    """A zlib stream of one final block holding `tokens` (a byte value or a (length, distance) pair): fixed Huffman
    codes, or a dynamic block with the given code lengths, sent as the code-length symbols `cl_syms` ((symbol, extra)
    pairs) under a fixed complete code-length code."""
    from tests.golden import inflate_oracle as O
    bw = _BitWriter()
    cmf = ((wbits - 8) << 4) | 8
    bw.put(cmf, 8)
    bw.put(31 - (cmf * 256) % 31, 8)
    if lit_lens is None:
        lit_lens, dist_lens = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, [5] * 30
        bw.put(1, 1)
        bw.put(1, 2)
    else:
        bw.put(1, 1)
        bw.put(2, 2)
        bw.put(len(lit_lens) - 257, 5)
        bw.put(len(dist_lens) - 1, 5)
        cl = [4] * 13 + [5] * 6                          # a complete code over all 19 symbols
        bw.put(19 - 4, 4)
        for s in O.CL_ORDER:
            bw.put(cl[s], 3)
        clc = _canonical(cl)
        for s, x in cl_syms:
            bw.code(*clc[s])
            if s >= 16:
                bw.put(x, {16: 2, 17: 3, 18: 7}[s])
    lc, dc = _canonical(lit_lens), _canonical(dist_lens)
    out = bytearray()
    for t in tokens:
        if isinstance(t, int):
            bw.code(*lc[t])
            out.append(t)
            continue
        n, d = t
        i = _index(O.LEN_BASE, n) if n != 257 else 27
        bw.code(*lc[257 + i])
        bw.put(n - O.LEN_BASE[i], O.LEN_EXTRA[i])
        j = _index(O.DIST_BASE, d)
        bw.code(*dc[j])
        bw.put(d - O.DIST_BASE[j], O.DIST_EXTRA[j])
        for _ in range(n):
            out.append(out[-d])
    bw.code(*lc[256])
    a, b = 1, 0
    for x in out:
        a = (a + x) % 65521
        b = (b + a) % 65521
    return bw.bytes() + struct.pack(">I", (b << 16) | a), bytes(out)


def _runs(sym, n, rep):
    """Code-length symbols for n copies of length `sym` (repeat code 16) or of zero (17 / 18)."""
    out = []
    if sym:
        out.append((sym, 0))
        n -= 1
        while n >= 3:
            k = min(6, n)
            out.append((16, k - 3))
            n -= k
        out += [(sym, 0)] * n
        return out
    while n >= 11:
        k = min(138, n)
        out.append((18, k - 11))
        n -= k
    if n >= 3:
        out.append((17, n - 3))
        n = 0
    return out + [(0, 0)] * n


def crafted_fixed():
    """One grey row through fixed codes: lengths 3, 257 and 258, every distance code up to 32 768, distance 1 and
    distances shorter than the length."""
    from tests.golden import inflate_oracle as O
    g = np.random.default_rng(120)
    toks = [0] + [int(v) for v in g.integers(0, 256, 300)]
    n = 301
    toks += [(3, 1), (257, 2), (258, 7)]
    n += 3 + 257 + 258
    while n < 32768 + 10:
        toks.append((258, 300))
        n += 258
    for j, base in enumerate(O.DIST_BASE):
        d = min(base + (1 << O.DIST_EXTRA[j]) - 1, 32768)
        toks.append((3 + j, d))
        n += 3 + j
    toks.append((10, 32768))
    z, raw = deflate_tokens(toks)
    return png_file(1, len(raw) - 1, 0, 8, z)


def crafted_one_distance():
    """A dynamic block whose distance code has one code of length 1, with repeat codes 16, 17 and 18."""
    lit = [9] * 256 + [5] * 14 + [8] * 16
    dist = [0] * 30
    dist[11] = 1                                         # distances 49 .. 64
    syms = _runs(9, 256, 16) + _runs(5, 14, 16) + _runs(8, 16, 16) + _runs(0, 11, 0) + [(1, 0)] + _runs(0, 18, 0)
    g = np.random.default_rng(121)
    toks = [0] + [int(v) for v in g.integers(0, 256, 80)]
    toks += [(3, 50), (40, 64), (258, 49), (11, 60)]
    z, raw = deflate_tokens(toks, lit, dist, syms)
    return png_file(1, len(raw) - 1, 0, 8, z)


def stored_blocks():
    """Two grey rows of 40 000 in stored blocks of 65 535 bytes and the rest, after an empty one."""
    raw = filter_rows(np.random.default_rng(97).integers(0, 256, (2, 40000)), 1, (0, 2))
    z = b"\x78\x01" + b"\x00\x00\x00\xff\xff"
    for k in range(0, len(raw), 65535):
        part = raw[k:k + 65535]
        z += bytes([k + 65535 >= len(raw)]) + struct.pack("<HH", len(part), len(part) ^ 0xFFFF) + part
    return png_file(2, 40000, 0, 8, z + struct.pack(">I", zlib.adler32(raw)))


def crafted_long_code():
    """A dynamic block whose literal / length code is a chain of lengths 1 .. 15: the end-of-block code and the length-3
    code are 15 bits long."""
    lit = [0] * 258
    for k in range(14):
        lit[k] = k + 1
    lit[256] = lit[257] = 15
    dist = [1]
    syms = [(l, 0) for l in lit[:14]] + _runs(0, 256 - 14, 0) + [(15, 0), (15, 0), (1, 0)]
    g = np.random.default_rng(122)
    toks = [0] + [int(v) for v in g.integers(1, 14, 200)] + [(3, 1), 5, (3, 1)]
    z, raw = deflate_tokens(toks, lit, dist, syms)
    return png_file(1, len(raw) - 1, 0, 8, z)


def _cv2_png(frame, level, strategy):
    import cv2
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(frame[:, :, ::-1]),
                           [cv2.IMWRITE_PNG_COMPRESSION, level, cv2.IMWRITE_PNG_STRATEGY, strategy])
    assert ok
    return buf.tobytes()


def _exif_orientation(v):
    ifd = struct.pack(">HHHIHH", 1, 0x0112, 3, 1, v, 0) + struct.pack(">I", 0)
    return chunk(b"eXIf", b"MM\x00\x2a" + struct.pack(">I", 8) + ifd)


def _far_distance():
    """Repeats 700 bytes apart inside a stream whose header claims a 512-byte window."""
    w = 80
    g = np.random.default_rng(3)
    block = g.integers(0, 256, (3, 3 * w), dtype=np.uint8)
    rows = np.concatenate([block] * 4)
    raw = filter_rows(rows, 3, (0,))
    z = bytearray(compress(raw, 9, 15))
    cmf = 0x18                                           # CINFO 1: 512-byte window
    z[0] = cmf
    z[1] = (31 - (cmf * 256) % 31) % 31                  # FCHECK for FLEVEL 0, no dictionary
    return png_file(12, w, 2, 8, bytes(z))


def device_cases():
    """name -> file bytes the device decodes."""
    import cv2
    c = {}
    frame = PC.smooth(37, 53, 21)
    low = PC.low_entropy(29, 41, 22)
    for level in range(10):
        for name, strat in (("default", cv2.IMWRITE_PNG_STRATEGY_DEFAULT), ("filtered", cv2.IMWRITE_PNG_STRATEGY_FILTERED),
                            ("huffman", cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY), ("rle", cv2.IMWRITE_PNG_STRATEGY_RLE),
                            ("fixed", cv2.IMWRITE_PNG_STRATEGY_FIXED)):
            c["cv2_l%d_%s" % (level, name)] = _cv2_png(frame if level % 2 else low, level, strat)
    for f in range(5):
        for colour, depth in ((0, 8), (4, 8), (2, 8), (6, 8)):
            c["filter%d_c%d" % (f, colour)] = made(19, 23, colour, depth, 30 + f, types=(f,))
    c["filter_mixed_rgb"] = made(40, 33, 2, 8, 40, types=(0, 1, 2, 3, 4, 4, 3, 1, 2))
    c["filter_mixed_rgba"] = made(40, 31, 6, 8, 41, types=(4, 3, 2, 1, 0))
    c["filter_mixed_grey2"] = made(25, 37, 0, 2, 42, types=(3, 4, 1, 2))
    for colour, depths in ((0, (1, 2, 4, 8)), (3, (1, 2, 4, 8))):
        for depth in depths:
            for w in (1, 7, 13):
                c["c%d_d%d_w%d" % (colour, depth, w)] = made(11, w, colour, depth, 50 + depth + w, types=(0, 1, 2, 3, 4))
    c["palette_short"] = made(9, 17, 3, 8, 60, plte_n=5)
    c["palette_trns"] = made(9, 17, 3, 4, 61, before=(chunk(b"tRNS", bytes([0, 128, 255])),))
    c["grey_trns"] = made(9, 17, 0, 8, 62, before=(chunk(b"tRNS", b"\x00\x07"),))
    for level in range(10):
        c["zlib_l%d" % level] = made(30, 45, 2, 8, 70 + level, types=(0, 1, 4), level=level)
    for wbits in range(9, 16):
        c["zlib_w%d" % wbits] = made(33, 61, 2, 8, 80 + wbits, types=(2, 3), level=9, wbits=wbits)
    c["sync_flush"] = made(31, 40, 2, 8, 90, flush_every=333, flush=zlib.Z_SYNC_FLUSH)
    c["full_flush"] = made(31, 40, 6, 8, 91, flush_every=500, flush=zlib.Z_FULL_FLUSH)
    c["idat_1byte_empty"] = made(7, 9, 2, 8, 92, split=0)
    c["idat_split_7"] = made(21, 19, 2, 8, 93, split=7)
    c["ancillary"] = made(21, 19, 2, 8, 94, split=100,
                          before=(chunk(b"gAMA", struct.pack(">I", 45455)), chunk(b"sBIT", b"\x05\x06\x05")),
                          between=(chunk(b"pHYs", struct.pack(">IIB", 2835, 2835, 1)), chunk(b"tEXt", b"Title\x00x")),
                          after=(chunk(b"tIME", bytes([7, 234, 10, 17, 12, 0, 0])),))
    c["palette_ancillary_1byte"] = made(9, 14, 3, 4, 96, split=0, before=(chunk(b"sRGB", b"\x00"),),
                                        between=(chunk(b"tRNS", bytes([10, 20])), chunk(b"bKGD", b"\x01")))
    c["stored_64k"] = stored_blocks()
    c["noise_576x720"] = _cv2_png(PC.noise(576, 720, 14), 1, cv2.IMWRITE_PNG_STRATEGY_RLE)
    c["smooth_cv2"] = _cv2_png(PC.smooth(128, 128, 2), 3, cv2.IMWRITE_PNG_STRATEGY_DEFAULT)
    c["long_codes"] = _cv2_png(PC.long_codes()[:, :600], 9, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY)
    c["crafted_fixed"] = crafted_fixed()
    c["crafted_one_distance"] = crafted_one_distance()
    c["crafted_long_code"] = crafted_long_code()
    for k, p in enumerate(CALENDAR):
        c["calendar_%d" % k] = open(p, "rb").read()
    return c


def fallback_cases():
    """name -> (file bytes, device status or None): None for files the host routes to cv2 without the device, else
    the status the device reports before the file goes to cv2 (include/teco.h)."""
    import cv2
    ok = made(12, 20, 2, 8, 100)
    px, _ = image(12, 20, 2, 8, 101)
    raw = filter_rows(pack_rows(px, 20, 2, 8), 3, (1,))
    z = compress(raw, 6)
    g = np.random.default_rng(102)
    c = {}
    ok16, buf = cv2.imencode(".png", g.integers(0, 65536, (9, 11, 3)).astype(np.uint16))
    c["depth16"] = (buf.tobytes(), None)
    c["interlaced"] = (png_file(1, 1, 2, 8, compress(b"\x00\x10\x20\x30"), interlace=1), None)
    c["exif6"] = (png_file(12, 20, 2, 8, z, before=(_exif_orientation(6),)), None)
    bad = bytearray(ok)
    bad[-13] ^= 0xFF                                     # last byte of the IDAT chunk's CRC
    c["bad_idat_crc"] = (bytes(bad), None)
    c["idat_interrupted"] = (png_file(12, 20, 2, 8, z[:9], after=(chunk(b"tEXt", b"a\x00b"), chunk(b"IDAT", z[9:]))), None)
    c["actl"] = (png_file(12, 20, 2, 8, z, before=(chunk(b"acTL", struct.pack(">II", 1, 0)),)), None)
    c["truncated"] = (png_file(12, 20, 2, 8, z[:len(z) // 2]), 6)
    c["adler"] = (png_file(12, 20, 2, 8, z[:-1] + bytes([z[-1] ^ 1])), 9)
    c["trailing"] = (png_file(12, 20, 2, 8, z + b"\x00\x00"), 10)
    c["far_distance"] = (_far_distance(), 5)
    c["filter5"] = (png_file(12, 20, 2, 8, compress(bytes([5]) + raw[1:])), 11)
    pal = np.array([[0, 0, 0], [255, 0, 0]], np.uint8)
    c["palette_index"] = (png_file(4, 6, 3, 2, compress(filter_rows(pack_rows(np.full((4, 6), 3), 6, 3, 2), 1, (0,))), pal), 12)
    return c
