"""Inflate (RFC 1951) inside a zlib stream (RFC 1950), restated in pure Python for the PNG decoder's tests, plus the PNG
stages after it (unfilter, expand to RGB) in numpy.  inflate() returns the bytes and what the stream used: block types
and stored lengths, match lengths and distance codes, code lengths and code-length symbols, distance codes per block --
so tests/test_png_decode_host.py can show that its cases reach every feature of the format."""
import collections

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class InflateError(ValueError):
    pass


class _Bits:
    def __init__(self, data):
        self.data, self.pos, self.bit = data, 0, 0        # byte position, bit within it

    def get(self, n):
        v = 0
        for k in range(n):
            if self.pos >= len(self.data):
                raise InflateError("stream ends early")
            v |= ((self.data[self.pos] >> self.bit) & 1) << k
            self.bit += 1
            if self.bit == 8:
                self.pos, self.bit = self.pos + 1, 0
        return v

    def align(self):
        if self.bit:
            self.pos, self.bit = self.pos + 1, 0


def _code(lengths):
    """Canonical Huffman code of `lengths`: {(length, code): symbol}, and whether it is complete.  Over-subscribed
    codes raise."""
    count = collections.Counter(l for l in lengths if l)
    left = 1
    for l in range(1, 16):
        left = 2 * left - count.get(l, 0)
        if left < 0:
            raise InflateError("over-subscribed code")
    code, nxt = 0, {}
    for l in range(1, 16):
        code = (code + count.get(l - 1, 0)) << 1
        nxt[l] = code
    table = {}
    for s, l in enumerate(lengths):
        if l:
            table[(l, nxt[l])] = s
            nxt[l] += 1
    return table, left == 0, max(lengths) if lengths else 0


def _decode(b, table):
    code = 0
    for l in range(1, 16):
        code = (code << 1) | b.get(1)
        s = table.get((l, code))
        if s is not None:
            return s, l
    raise InflateError("bit pattern outside the code")


def inflate(data):
    """zlib stream -> (bytes, stats).  Raises InflateError where zlib fails, and for what the device refuses on top:
    incomplete literal / length codes, distances beyond the header's window, data after the Adler-32."""
    data = bytes(data)
    b = _Bits(data)
    cmf, flg = b.get(8), b.get(8)
    if cmf & 15 != 8 or cmf >> 4 > 7 or (cmf * 256 + flg) % 31 or flg & 32:
        raise InflateError("zlib header")
    window = 1 << ((cmf >> 4) + 8)
    out = bytearray()
    st = collections.defaultdict(collections.Counter)
    st["window"][window] += 1
    last = 0
    while not last:
        last, btype = b.get(1), b.get(2)
        st["block"][btype] += 1
        if btype == 0:
            b.align()
            n, nn = b.get(16), b.get(16)
            if n != nn ^ 0xFFFF:
                raise InflateError("stored length")
            st["stored_len"][n] += 1
            if b.pos + n > len(data):
                raise InflateError("stream ends early")
            out += data[b.pos:b.pos + n]
            b.pos += n
            continue
        if btype == 3:
            raise InflateError("block type 3")
        if btype == 1:
            lit, _, _ = _code([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
            dist, _, _ = _code([5] * 32)
        else:
            nlen, ndist, ncl = b.get(5) + 257, b.get(5) + 1, b.get(4) + 4
            if nlen > 286 or ndist > 30:
                raise InflateError("too many symbols")
            cl = [0] * 19
            for i in range(ncl):
                cl[CL_ORDER[i]] = b.get(3)
            clc, whole, _ = _code(cl)
            if not whole:
                raise InflateError("incomplete code-length code")
            lens = []
            while len(lens) < nlen + ndist:
                s, _ = _decode(b, clc)
                st["cl_symbol"][s] += 1
                if s < 16:
                    lens.append(s)
                elif s == 16:
                    if not lens:
                        raise InflateError("repeat without a length")
                    lens += [lens[-1]] * (3 + b.get(2))
                elif s == 17:
                    lens += [0] * (3 + b.get(3))
                else:
                    lens += [0] * (11 + b.get(7))
            if len(lens) > nlen + ndist:
                raise InflateError("repeat beyond the lengths")
            if lens[256] == 0:
                raise InflateError("no end-of-block code")
            lit, whole, lmax = _code(lens[:nlen])
            if not whole:
                raise InflateError("incomplete literal / length code")
            dl = lens[nlen:]
            dist, dwhole, dmax = _code(dl)
            used = sum(1 for l in dl if l)
            if not dwhole and not (used == 0 or (used == 1 and dmax == 1)):
                raise InflateError("incomplete distance code")
            st["max_code_len"][max(lmax, dmax)] += 1
            st["dist_codes_in_block"][used] += 1
        while True:
            s, _ = _decode(b, lit)
            if s < 256:
                out.append(s)
                continue
            if s == 256:
                break
            if s > 285:
                raise InflateError("length symbol %d" % s)
            length = LEN_BASE[s - 257] + b.get(LEN_EXTRA[s - 257])
            ds, _ = _decode(b, dist)
            if ds > 29:
                raise InflateError("distance symbol %d" % ds)
            d = DIST_BASE[ds] + b.get(DIST_EXTRA[ds])
            if d > len(out) or d > window:
                raise InflateError("distance too far back")
            st["len_code"][s] += 1
            st["length"][length] += 1
            st["dist_code"][ds] += 1
            st["distance"][min(d, 33)] += 1            # 1 .. 32 exactly, 33: longer
            if d < length:
                st["overlap"][1] += 1
            for _ in range(length):
                out.append(out[-d])
    b.align()
    adler = b.get(32)
    want = int.from_bytes(adler.to_bytes(4, "little"), "big")
    a, s2 = 1, 0
    for x in out:
        a = (a + x) % 65521
        s2 = (s2 + a) % 65521
    if (s2 << 16 | a) != want:
        raise InflateError("Adler-32")
    if b.pos != len(data):
        raise InflateError("data after the stream")
    return bytes(out), st


def unfilter(raw, h, rowbytes, bpp):
    """Filtered rows (filter byte + rowbytes each) -> [h, rowbytes] uint8; counts (filter, bpp) pairs into `seen`."""
    raw = np.frombuffer(raw, np.uint8).reshape(h, rowbytes + 1)
    out = np.zeros((h, rowbytes), np.int64)
    filters = []
    for y in range(h):
        f, cur = int(raw[y, 0]), raw[y, 1:].astype(np.int64)
        if f > 4:
            raise InflateError("filter type %d" % f)
        filters.append(f)
        up = out[y - 1] if y else np.zeros(rowbytes, np.int64)
        if f == 0:
            row = cur
        elif f == 2:
            row = (cur + up) & 255
        else:
            row = np.zeros(rowbytes, np.int64)
            for i in range(rowbytes):
                a = row[i - bpp] if i >= bpp else 0
                c = up[i - bpp] if i >= bpp else 0
                if f == 1:
                    p = a
                elif f == 3:
                    p = (a + up[i]) >> 1
                else:
                    pp = a + up[i] - c
                    pa, pb, pc = abs(pp - a), abs(pp - up[i]), abs(pp - c)
                    p = a if pa <= pb and pa <= pc else up[i] if pb <= pc else c
                row[i] = (cur[i] + p) & 255
        out[y] = row
    return out.astype(np.uint8), filters


def expand(rows, w, colour, depth, plte=None):
    """Unfiltered rows -> [h, w, 3] uint8 RGB as cv2.imread gives it."""
    h = rows.shape[0]
    if depth < 8:
        bits = np.unpackbits(rows, axis=1).reshape(h, -1)
        idx = np.zeros((h, w), np.int64)
        for k in range(depth):
            idx = idx * 2 + bits[:, k:w * depth:depth]
        v = idx
    else:
        v = rows.astype(np.int64)
    if colour == 0:
        g = v[:, :w] * (255 // ((1 << depth) - 1))
        return np.repeat(g[:, :, None], 3, 2).astype(np.uint8)
    if colour == 3:
        pal = np.frombuffer(plte, np.uint8).reshape(-1, 3)
        idx = v[:, :w]
        if idx.max() >= len(pal):
            raise InflateError("palette index")
        return pal[idx]
    ch = {2: 3, 4: 2, 6: 4}[colour]
    px = v.reshape(h, w, ch)
    if colour == 4:
        return np.repeat(px[:, :, :1], 3, 2).astype(np.uint8)
    return px[:, :, :3].astype(np.uint8)


def decode(stream):
    """A parsed PNG (tecogan_b200.png.Stream) -> (RGB frame, inflate stats, filter types per row)."""
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[stream.colour]
    rowbytes = (stream.w * ch * stream.depth + 7) // 8
    raw, st = inflate(stream.idat)
    if len(raw) != stream.h * (rowbytes + 1):
        raise InflateError("%d bytes, the image has %d" % (len(raw), stream.h * (rowbytes + 1)))
    bpp = max(1, ch * stream.depth // 8)
    rows, filters = unfilter(raw, stream.h, rowbytes, bpp)
    return expand(rows, stream.w, stream.colour, stream.depth, stream.plte), st, filters
