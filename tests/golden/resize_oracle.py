"""Host restatement, in numpy, of `cv2.resize(frame, (w_out, h_out), interpolation=cv2.INTER_LANCZOS4)` on a uint8
3-channel frame (cv2 4.13.0, fixed-point path): the resize behind `main.py --outscale`.
`tecogan_b200/csrc/resize.cu` computes the same numbers from the tables `tecogan_b200/resize.py` builds (DESIGN.md
section 4.11).  The coefficients are computed here one scalar at a time, in the order cv2's source gives them, so that
this file and the package's vectorised tables are two independent restatements.

  position  per output index d (columns; rows alike): scale = 1 / (n_out / n_in) in double,
            f = float((d + 0.5) * scale - 0.5), s = floor(f), f -= s in float.
  taps      source indices s - 3 .. s + 4, each clamped into [0, n_in - 1].
  weights   interpolateLanczos4(f): y0 = -(f + 3) * pi / 4 (f + 3 in float), s0 = sin(y0), c0 = cos(y0); tap i has
            t = float(f + 3 - i) and weight 1e30f when |t| < 1e-6f, else float((cs[i][0] s0 + cs[i][1] c0) / y^2) with
            y = -t * pi / 4; the eight are summed in float and scaled by 1.f / sum; then int16(round_half_even(w * 2048)).
  passes    horizontal int32 sum of src * alpha per channel, vertical int32 sum of beta * row,
            out = clamp((v + (1 << 21)) >> 22, 0, 255).
"""
import math

import numpy as np

S45 = 0.70710678118654752440084436210485
CS = [(1.0, 0.0), (-S45, -S45), (0.0, 1.0), (S45, -S45), (-1.0, 0.0), (S45, S45), (0.0, -1.0), (-S45, S45)]
COEF_SCALE = 2048
F32 = np.float32


def lanczos4_weights(f):
    """cv2's interpolateLanczos4 for one float32 fraction f in [0, 1): eight float32 weights."""
    f = F32(f)
    f3 = F32(f + F32(3))
    y0 = -float(f3) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    w = []
    total = F32(0)
    for i in range(8):
        t = F32(f3 - F32(i))
        if abs(t) >= F32(1e-6):
            y = -float(t) * math.pi * 0.25
            wi = F32((CS[i][0] * s0 + CS[i][1] * c0) / (y * y))
        else:
            wi = F32(1e30)
        w.append(wi)
        total = F32(total + wi)
    inv = F32(F32(1) / total)
    return [F32(wi * inv) for wi in w]


def to_fixed(w):
    """saturate_cast<short>(w * 2048): round half to even, saturated to int16."""
    v = np.rint(np.float32(w) * np.float32(COEF_SCALE))
    return int(min(max(v, -32768), 32767))


def axis_table(n_in, n_out):
    """(base int32 [n_out], taps int32 [n_out, 8] clamped source indices, coef int16 [n_out, 8]) for one axis."""
    scale = 1.0 / (float(n_out) / float(n_in))
    base = np.empty(n_out, np.int32)
    taps = np.empty((n_out, 8), np.int32)
    coef = np.empty((n_out, 8), np.int16)
    for d in range(n_out):
        f = F32((d + 0.5) * scale - 0.5)
        s = math.floor(f)
        f = F32(f - F32(s))
        base[d] = s
        for j in range(8):
            taps[d, j] = min(max(s - 3 + j, 0), n_in - 1)
        coef[d] = [to_fixed(w) for w in lanczos4_weights(f)]
    return base, taps, coef


def resize(frame, h_out, w_out):
    """uint8 [H, W, 3] -> uint8 [h_out, w_out, 3] equal to cv2.resize(frame, (w_out, h_out), INTER_LANCZOS4).  cv2 copies
    a frame whose size does not change; the identity coefficients give the same bytes, and this path is not special."""
    f = np.asarray(frame)
    if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
        raise ValueError("resize: need a uint8 [H, W, 3] frame, got %s %s" % (f.dtype, f.shape))
    H, W = f.shape[:2]
    _, xt, xc = axis_table(W, w_out)
    _, yt, yc = axis_table(H, h_out)
    src = f.astype(np.int64)
    horiz = np.zeros((H, w_out, 3), np.int64)
    for j in range(8):
        horiz += src[:, xt[:, j], :] * xc[:, j].astype(np.int64)[None, :, None]
    vert = np.zeros((h_out, w_out, 3), np.int64)
    for k in range(8):
        vert += horiz[yt[:, k]] * yc[:, k].astype(np.int64)[:, None, None]
    assert np.abs(horiz).max(initial=0) < 2 ** 31 and np.abs(vert).max(initial=0) < 2 ** 31   # int32 in cv2 and the kernel
    return np.clip((vert + (1 << 21)) >> 22, 0, 255).astype(np.uint8)
