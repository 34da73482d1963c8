"""JPEG as cv2.imwrite writes it with cv2's defaults, restated on the host from ITU-T T.81 and the arithmetic DESIGN.md
section 4.6 lists: baseline, quality 95, 4:2:0, fixed-point colour conversion, h2v2 averaging, the islow integer FDCT,
rounded division, the Annex K Huffman tables.  numpy only.  tests/test_jpeg_host.py checks it against cv2.imencode.

encode(rgb, stats) returns the file; a `stats` dict collects which code paths the frame reached (dummy blocks, the bottom
row rule, ZRL, blocks without EOB, 0xFF stuffing, padding lengths, size categories) for the coverage test.
"""
import numpy as np

QUALITY = 95

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])      # zigzag position -> row-major index

# T.81 Annex K, Tables K.1 (luminance) and K.2 (chrominance), row-major
LUMA_BASE = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                      14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                      49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
CHROMA_BASE = np.array([17, 18, 24, 47] + [99] * 4 + [18, 21, 26, 66] + [99] * 4 + [24, 26, 56] + [99] * 5 +
                       [47, 66] + [99] * 38)

# T.81 Annex K.3, Tables K.3 - K.6: number of codes of each length 1..16, then the symbols in code order
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], list(bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f0243362728209"
    "0a161718191a25262728292a3435363738393a434445464748494a535455565758595a636465"
    "666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9ea"
    "f1f2f3f4f5f6f7f8f9fa")))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], list(bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a16"
    "2434e125f11718191a262728292a35363738393a434445464748494a535455565758595a63"
    "6465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6"
    "a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8"
    "e9eaf2f3f4f5f6f7f8f9fa")))


def quant_table(base):
    """libjpeg's scaling for quality >= 50: base * (200 - 2q) / 100, rounded half up, clamped to 1..255."""
    return np.clip((np.asarray(base) * (200 - 2 * QUALITY) + 50) // 100, 1, 255)


def huffman_codes(table):
    """symbol -> (code, length), T.81 Annex C: canonical codes in order of length."""
    bits, vals = table
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def _fix(x, frac):
    return int(x * (1 << frac) + 0.5)


def ycc(rgb):
    """Y, Cb, Cr planes (int64) from R, G, B: 16 fractional bits; Y rounds half up, Cb and Cr with 2^15 - 1."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    f = lambda x: _fix(x, 16)
    y = (f(.299) * r + f(.587) * g + f(.114) * b + (1 << 15)) >> 16
    cb = (-f(.16874) * r - f(.33126) * g + f(.5) * b + (128 << 16) + (1 << 15) - 1) >> 16
    cr = (f(.5) * r - f(.41869) * g - f(.08131) * b + (128 << 16) + (1 << 15) - 1) >> 16
    return y, cb, cr


def downsample(c, mw, mh):
    """h2v2 chroma: columns repeated to 16 per MCU, rows to an even count; (2x2 sum + 1, 2, 1, 2, ..) >> 2 along each
    row; then the last downsampled row repeated to 8 per MCU."""
    h, w = c.shape
    c = np.pad(c, ((0, h % 2), (0, 16 * mw - w)), mode="edge")
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    bias = np.tile([1, 2], s.shape[1] // 2)[None, :]
    d = (s + bias) >> 2
    return np.pad(d, ((0, 8 * mh - d.shape[0]), (0, 0)), mode="edge")


def _pass(v, second):
    """One islow pass over axis 0 of v (8 x ...): CONST_BITS 13, PASS1_BITS 2, round half up."""
    f = lambda x: _fix(x, 13)
    n = 13 + 2 if second else 13 - 2
    desc = lambda x, b: (x + (1 << (b - 1))) >> b
    t0, t7, t1, t6 = v[0] + v[7], v[0] - v[7], v[1] + v[6], v[1] - v[6]
    t2, t5, t3, t4 = v[2] + v[5], v[2] - v[5], v[3] + v[4], v[3] - v[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    o[0] = desc(t10 + t11, 2) if second else (t10 + t11) << 2
    o[4] = desc(t10 - t11, 2) if second else (t10 - t11) << 2
    e = (t12 + t13) * f(0.541196100)
    o[2] = desc(e + t13 * f(0.765366865), n)
    o[6] = desc(e - t12 * f(1.847759065), n)
    z5 = (t4 + t5 + t6 + t7) * f(1.175875602)
    z1, z2 = -(t4 + t7) * f(0.899976223), -(t5 + t6) * f(2.562915447)
    z3, z4 = -(t4 + t6) * f(1.961570560) + z5, -(t5 + t7) * f(0.390180644) + z5
    o[7] = desc(t4 * f(0.298631336) + z1 + z3, n)
    o[5] = desc(t5 * f(2.053119869) + z2 + z4, n)
    o[3] = desc(t6 * f(3.072711026) + z2 + z3, n)
    o[1] = desc(t7 * f(1.501321110) + z1 + z4, n)
    return np.stack(o)


def fdct(blocks):
    """[..., 8, 8] samples already centred (-128) -> the islow FDCT, scaled by 8, int64."""
    b = np.moveaxis(blocks.astype(np.int64), (-2, -1), (0, 1))      # [row, col, ...]
    b = np.stack([_pass(b[i], False) for i in range(8)])              # rows: pass over columns
    b = np.stack([_pass(b[:, j], True) for j in range(8)], 1)         # columns
    return np.moveaxis(b, (0, 1), (-2, -1))


def quantise(coef, table):
    """sign(c) * ((|c| + d/2) // d), d = 8 Q (the FDCT's scale)."""
    d = 8 * np.asarray(table, np.int64).reshape(8, 8)
    return np.sign(coef) * ((np.abs(coef) + d // 2) // d)


def _blocks(plane, nby, nbx):
    return plane[:8 * nby, :8 * nbx].reshape(nby, 8, nbx, 8).transpose(0, 2, 1, 3)


def scan_blocks(rgb, stats=None):
    """[mh, mw, 6, 64] quantised coefficients in zigzag order, MCU by MCU: Y00 Y01 Y10 Y11 Cb Cr, dummy blocks
    included."""
    h, w, _ = rgb.shape
    mw, mh, bw, bh = -(-w // 16), -(-h // 16), -(-w // 8), -(-h // 8)
    y, cb, cr = ycc(rgb)
    yp = np.pad(y, ((0, 8 * bh - h), (0, 8 * bw - w)), mode="edge")
    ql, qc = quant_table(LUMA_BASE), quant_table(CHROMA_BASE)
    zq = lambda blocks, q: quantise(fdct(blocks - 128), q).reshape(blocks.shape[:-2] + (64,))[..., ZIGZAG]
    yq = zq(_blocks(yp, bh, bw), ql)
    out = np.zeros((mh, mw, 6, 64), np.int64)
    real = np.zeros((2 * mh, 2 * mw), bool)
    real[:bh, :bw] = True
    full = np.zeros((2 * mh, 2 * mw, 64), np.int64)
    full[:bh, :bw] = yq
    for k in range(4):
        dy, dx = k >> 1, k & 1
        out[:, :, k] = full[dy::2, dx::2]
        dummy = ~real[dy::2, dx::2]
        if k:                                           # a dummy takes the DC of the block before it in the MCU
            out[:, :, k, 0] = np.where(dummy, out[:, :, k - 1, 0], out[:, :, k, 0])
    out[:, :, 4] = zq(_blocks(downsample(cb, mw, mh), mh, mw), qc)
    out[:, :, 5] = zq(_blocks(downsample(cr, mw, mh), mh, mw), qc)
    if stats is not None:
        stats["dummy_right"] = stats.get("dummy_right", 0) + int((~real[:, bw:]).sum())
        stats["dummy_bottom"] = stats.get("dummy_bottom", 0) + int((~real[bh:, :]).sum())
        stats.setdefault("odd", set()).update(k for k, n in (("W", w), ("H", h)) if n % 2)
        stats.setdefault("biases", set()).update({1, 2} if mw else set())
        if h % 2 == 0 and h % 16:
            # repeating image rows to 16 per MCU before downsampling would give other chroma rows
            alt = lambda c: downsample(np.pad(c, ((0, 16 * mh - h), (0, 0)), mode="edge"), mw, mh)
            if not (np.array_equal(alt(cb), downsample(cb, mw, mh)) and np.array_equal(alt(cr), downsample(cr, mw, mh))):
                stats["bottom_rule"] = stats.get("bottom_rule", 0) + 1
    return out


class _Bits:
    """MSB-first bit writer; every 0xFF byte is followed by 0x00."""

    def __init__(self):
        self.data, self.acc, self.n, self.ff = bytearray(), 0, 0, 0

    def put(self, v, n):
        self.acc = (self.acc << n) | v
        self.n += n
        while self.n >= 8:
            self.n -= 8
            byte = (self.acc >> self.n) & 255
            self.data.append(byte)
            if byte == 0xFF:
                self.data.append(0)
                self.ff += 1
        self.acc &= (1 << self.n) - 1

    def pad(self):
        """Fill the last byte with 1-bits; returns how many."""
        k = (8 - self.n) % 8
        self.put((1 << k) - 1, k)
        return k


def _category(v):
    return int(abs(int(v))).bit_length()


def _amplitude(v, s):
    return int(v) if v >= 0 else int(v) + (1 << s) - 1


def entropy_code(mcus, stats=None):
    """The scan's entropy-coded bytes (stuffed, padded) for [mh, mw, 6, 64] zigzag coefficients."""
    dc = [huffman_codes(DC_LUMA), huffman_codes(DC_CHROMA)]
    ac = [huffman_codes(AC_LUMA), huffman_codes(AC_CHROMA)]
    out, pred = _Bits(), [0, 0, 0]
    zrl = no_eob = dc_only = 0
    max_dc = max_ac = 0
    for blk, k in zip(mcus.reshape(-1, 64), np.tile(np.arange(6), mcus.shape[0] * mcus.shape[1])):
        comp, t = (0, 0) if k < 4 else (k - 3, 1)
        diff = int(blk[0]) - pred[comp]
        pred[comp] = int(blk[0])
        s = _category(diff)
        max_dc = max(max_dc, s)
        code, n = dc[t][s]
        out.put((code << s) | _amplitude(diff, s), n + s)
        nz = np.flatnonzero(blk[1:]) + 1
        last = 0
        for pos in nz:
            run = pos - last - 1
            while run >= 16:
                out.put(*ac[t][0xF0])
                zrl += 1
                run -= 16
            v = blk[pos]
            s = _category(v)
            max_ac = max(max_ac, s)
            code, n = ac[t][(run << 4) | s]
            out.put((code << s) | _amplitude(v, s), n + s)
            last = pos
        if last < 63:
            out.put(*ac[t][0x00])
            dc_only += int(last == 0)
        else:
            no_eob += 1
    pad = out.pad()
    if stats is not None:
        stats["zrl"] = stats.get("zrl", 0) + zrl
        stats["no_eob"] = stats.get("no_eob", 0) + no_eob
        stats["dc_only"] = stats.get("dc_only", 0) + dc_only
        stats["ff"] = stats.get("ff", 0) + out.ff
        stats.setdefault("pad", set()).add(pad)
        stats["max_dc_cat"] = max(stats.get("max_dc_cat", 0), max_dc)
        stats["max_ac_cat"] = max(stats.get("max_ac_cat", 0), max_ac)
    return bytes(out.data)


def header(h, w):
    """SOI, APP0 (JFIF 1.01, no units, 1:1), DQT 0 and 1 (zigzag), SOF0 (4:2:0), DHT DC0 AC0 DC1 AC1, SOS."""
    be16 = lambda v: int(v).to_bytes(2, "big")
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0" + be16(16) + b"JFIF\x00" + bytes([1, 1, 0]) + be16(1) + be16(1) + bytes([0, 0])
    for tid, base in ((0, LUMA_BASE), (1, CHROMA_BASE)):
        out += b"\xff\xdb" + be16(67) + bytes([tid]) + bytes(int(q) for q in quant_table(base)[ZIGZAG])
    out += b"\xff\xc0" + be16(17) + bytes([8]) + be16(h) + be16(w) + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for tc, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        out += b"\xff\xc4" + be16(3 + 16 + len(vals)) + bytes([tc]) + bytes(bits) + bytes(vals)
    out += b"\xff\xda" + be16(12) + bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


def encode(rgb, stats=None):
    """[H, W, 3] uint8 RGB -> the bytes of cv2.imwrite(path.jpg, BGR copy) with cv2's defaults."""
    h, w = rgb.shape[:2]
    return header(h, w) + entropy_code(scan_blocks(rgb, stats), stats) + b"\xff\xd9"
