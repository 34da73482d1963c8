"""The device GIF encoder (tecogan_b200/csrc/gif.cu, DESIGN.md section 4.8) restated in numpy and pure Python, plus the
reference's summary quantisation, for the encoder's tests.

encode(frames) takes a uint8 [T, H, W, 3] RGB animation and returns (file bytes, info).  info records what the encoding
went through -- palette size, split ties, nearest-colour ties, code widths, mid-stream Clears, sub-block counts -- so the
tests can show that their cases reach every branch of the specification:

  palette   median cut over every pixel of every frame, up to 256 boxes; split the splittable box (two or more distinct
            colours) with the most pixels (ties: lowest box index) on its axis of largest max - min (ties: R, G, B) at
            the smallest v in [min, max - 1] with 2 count(axis <= v) >= count (none: v = max - 1); pixels with axis <= v
            stay, the rest form a new last box; entry = per-channel (sum + n / 2) / n.
  dither    per frame, raster order, no error carried between frames: c = clamp(src + err, 0, 255); nearest real entry
            by squared RGB distance (ties: lowest index); e = c - pal; (2e) / 4 to the right, e / 4 lower-left and
            e / 4 below, C division (truncation), targets outside the frame dropped.
  LZW       minimum code size 8, Clear 256, EOI 257; Clear first at width 9; greedy longest match; after each emitted
            code the width grows when the next free code equals 1 << width (width < 12); when the table holds 4096
            codes, Clear at width 12 and reset; the pending code, then EOI; LSB-first; 255-byte sub-blocks, 0 ends.
  file      GIF89a, W x H screen, 0xF7 (256-entry global table, black padding), NETSCAPE2.0 loop 0, per frame a
            Graphic Control Extension (no transparency, 33 cs) and a full-frame descriptor without a local table, 0x3B.
"""
import struct

import numpy as np

DELAY_CS = 33


def convert_image_dtype(x, deprocess=False):
    """tf.image.convert_image_dtype(x, uint8, saturate=True) in float32, after (x + 1) / 2 when `deprocess`."""
    x = np.asarray(x, dtype=np.float32)
    if deprocess:
        x = (x + np.float32(1)) / np.float32(2)
    with np.errstate(invalid="ignore"):
        y = x * np.float32(255.5)
        y = np.where(np.isnan(y), np.float32(0), y)
    return np.trunc(np.clip(y, 0, 255)).astype(np.uint8)


def median_cut(pixels, info=None):
    """pixels [P, 3] uint8 -> palette [n, 3] uint8 (1 <= n <= 256)."""
    px = np.asarray(pixels, dtype=np.uint8).reshape(-1, 3)
    boxes, stats = [], []

    def add(i, b):
        s = (len(b), b.min(0).astype(int), b.max(0).astype(int))
        if i == len(boxes):
            boxes.append(b)
            stats.append(s)
        else:
            boxes[i], stats[i] = b, s

    add(0, px)
    ties = {"box": 0, "axis": 0, "no_v": 0}
    while len(boxes) < 256:
        split = [(n, i) for i, (n, lo, hi) in enumerate(stats) if (hi > lo).any()]
        if not split:
            break
        best_n = max(n for n, _ in split)
        tied = [i for n, i in split if n == best_n]
        best = tied[0]                                       # the lowest box index
        if len(tied) > 1:
            ties["box"] += 1
        b = boxes[best]
        _, lo, hi = stats[best]
        rng = hi - lo
        axis = int(np.argmax(rng))                        # argmax takes the first maximum: R, then G, then B
        if (rng == rng[axis]).sum() > 1:
            ties["axis"] += 1
        hist = np.bincount(b[:, axis], minlength=256)
        cum = np.cumsum(hist)
        v = hi[axis] - 1
        cand = [u for u in range(lo[axis], hi[axis]) if 2 * cum[u] >= len(b)]
        if cand:
            v = cand[0]
        else:
            ties["no_v"] += 1
        keep = b[:, axis] <= v
        add(best, b[keep])
        add(len(boxes), b[~keep])
    pal = np.array([[(int(b[:, c].astype(np.int64).sum()) + len(b) // 2) // len(b) for c in range(3)] for b in boxes],
                   dtype=np.uint8)
    if info is not None:
        info.update(boxes=len(boxes), split_ties=ties)
    return pal


def dither(frame, pal, info=None):
    """frame [H, W, 3] uint8, pal [n, 3] -> indices [H, W] uint8 (Sierra-2-4A, the rules above)."""
    h, w, _ = frame.shape
    p = pal.astype(np.int64)
    src = frame.astype(np.int64)
    err = np.zeros((h + 1, w + 2, 3), dtype=np.int64)          # column offset 1: x - 1 and x + 1 stay in range
    out = np.zeros((h, w), dtype=np.uint8)
    ties = 0
    for y in range(h):
        for x in range(w):
            c = np.clip(src[y, x] + err[y, x + 1], 0, 255)
            d = ((p - c) ** 2).sum(1)
            i = int(np.argmin(d))                                # the first minimum: the lowest index
            if (d == d[i]).sum() > 1:
                ties += 1
            out[y, x] = i
            e = c - p[i]
            if x + 1 < w:
                err[y, x + 2] += _cdiv(2 * e, 4)
            if y + 1 < h:
                if x > 0:
                    err[y + 1, x] += _cdiv(e, 4)
                err[y + 1, x + 1] += _cdiv(e, 4)
    if info is not None:
        info["nearest_ties"] = info.get("nearest_ties", 0) + ties
    return out


def _cdiv(a, b):
    """C integer division (truncation toward zero), elementwise."""
    q = np.abs(a) // b
    return np.where(a < 0, -q, q)


def lzw(indices, info=None):
    """indices (uint8, raster order) -> the GIF LZW byte stream at minimum code size 8 (before sub-blocking)."""
    data = bytes(np.asarray(indices, dtype=np.uint8).reshape(-1))
    CLEAR, EOI = 256, 257
    out = bytearray()
    acc = nacc = 0
    widths = set()
    clears = 0

    def emit(code, width):
        nonlocal acc, nacc
        acc |= code << nacc
        nacc += width
        widths.add(width)
        while nacc >= 8:
            out.append(acc & 0xFF)
            acc >>= 8
            nacc -= 8

    width, nxt, table = 9, 258, {}
    emit(CLEAR, width)
    cur = data[0]
    for c in data[1:]:
        k = (cur << 8) | c
        code = table.get(k)
        if code is not None:
            cur = code
            continue
        emit(cur, width)
        if nxt == (1 << width) and width < 12:
            width += 1
        table[k] = nxt
        nxt += 1
        if nxt == 4096:
            emit(CLEAR, 12)
            clears += 1
            width, nxt, table = 9, 258, {}
        cur = c
    emit(cur, width)
    if nxt == (1 << width) and width < 12:
        width += 1
    emit(EOI, width)
    if nacc:
        out.append(acc & 0xFF)
    if info is not None:
        info.setdefault("widths", set()).update(widths)
        info["clears"] = info.get("clears", 0) + clears
    return bytes(out)


def sub_blocks(data):
    out = bytearray()
    for i in range(0, len(data), 255):
        chunk = data[i:i + 255]
        out.append(len(chunk))
        out += chunk
    out.append(0)
    return bytes(out)


def encode(frames, info=None):
    """frames [T, H, W, 3] uint8 RGB -> (GIF89a file bytes, info dict)."""
    frames = np.asarray(frames, dtype=np.uint8)
    if frames.ndim != 4 or frames.shape[3] != 3:
        raise ValueError("expected [T, H, W, 3], got %s" % (frames.shape,))
    t, h, w, _ = frames.shape
    if t < 1 or not (1 <= h <= 65535 and 1 <= w <= 65535):
        raise ValueError("bad animation shape %s" % (frames.shape,))
    info = {} if info is None else info
    pal = median_cut(frames.reshape(-1, 3), info)
    info["palette"] = pal
    table = np.zeros((256, 3), dtype=np.uint8)
    table[:len(pal)] = pal
    out = bytearray(b"GIF89a" + struct.pack("<HHBBB", w, h, 0xF7, 0, 0) + table.tobytes())
    out += b"\x21\xFF\x0BNETSCAPE2.0\x03\x01\x00\x00\x00"
    dithered = []
    nblocks = []
    for f in frames:
        idx = dither(f, pal, info)
        dithered.append(idx)
        z = lzw(idx, info)
        nblocks.append((len(z) + 254) // 255)
        out += b"\x21\xF9\x04\x00" + struct.pack("<H", DELAY_CS) + b"\x00\x00"
        out += b"\x2C" + struct.pack("<HHHHB", 0, 0, w, h, 0) + b"\x08" + sub_blocks(z)
    out += b"\x3B"
    info["dithered"] = np.stack(dithered)                     # [T, H, W] indices
    info["sub_blocks"] = nblocks
    return bytes(out), info


def decoded_frames(info):
    """The RGB frames a decoder must produce: palette[dithered]."""
    return info["palette"][info["dithered"]]
