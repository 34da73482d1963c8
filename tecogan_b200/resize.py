"""Output scale of the inference command (`main.py --outscale s`, DESIGN.md section 4.11): the file size a scale gives,
and the coefficient tables of cv2 4.13's fixed-point INTER_LANCZOS4 resize that teco_resize_lanczos4_u8 applies.

The tables need libm's double sin / cos and are O(W + H), so they are computed here, on the host, once per (input
size, output size); the kernel does integer work only.  Per output index d of an axis, in cv2's arithmetic:
scale = 1 / (n_out / n_in) in double, f = float((d + 0.5) * scale - 0.5), s = floor(f), f -= s in float; the taps are
the source indices s - 3 .. s + 4 clamped into the frame, weighted by interpolateLanczos4(f) converted to int16
round_half_even(w * 2048)."""
import functools
import math

import numpy as np

MIN_OUTSCALE, MAX_OUTSCALE = 1.0, 16.0
_S45 = 0.70710678118654752440084436210485
_CS = np.array([(1, 0), (-_S45, -_S45), (0, 1), (_S45, -_S45), (-1, 0), (_S45, _S45), (0, -1), (-_S45, _S45)])


def check_outscale(s):
    """ValueError unless 1 <= s <= 16: at s = 1 the 4x frame is down-scaled 4x, the most the kernel takes."""
    if not (MIN_OUTSCALE <= s <= MAX_OUTSCALE):
        raise ValueError("--outscale must be in [%g, %g], got %r" % (MIN_OUTSCALE, MAX_OUTSCALE, s))


def out_size(h, w, s):
    """(h_out, w_out) = (int(h * s), int(w * s)) for an h x w LR input: Real-ESRGAN's --outscale rule."""
    return int(h * s), int(w * s)


def axis_table(n_in, n_out):
    """(base int32 [n_out], coef int16 [n_out, 8]) of one axis: tap j of output d reads source index
    clamp(base[d] - 3 + j, 0, n_in - 1) with weight coef[d, j] / 2048."""
    f32 = np.float32
    scale = 1.0 / (float(n_out) / float(n_in))
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
    base = np.floor(f).astype(np.int32)
    f = (f - base.astype(f32)).astype(f32)
    f3 = (f + f32(3)).astype(f32)
    y0 = -f3.astype(np.float64) * math.pi * 0.25
    s0 = np.array([math.sin(v) for v in y0])
    c0 = np.array([math.cos(v) for v in y0])
    t = (f3[:, None] - np.arange(8, dtype=f32)[None, :]).astype(f32)
    y = -t.astype(np.float64) * math.pi * 0.25
    with np.errstate(divide="ignore", invalid="ignore"):
        w = ((_CS[:, 0] * s0[:, None] + _CS[:, 1] * c0[:, None]) / (y * y)).astype(f32)
    w = np.where(np.abs(t) >= f32(1e-6), w, f32(1e30))
    total = np.zeros(n_out, f32)
    for i in range(8):                                     # float sum in tap order, as cv2 adds them
        total = (total + w[:, i]).astype(f32)
    w = (w * (f32(1) / total)[:, None]).astype(f32)
    coef = np.clip(np.rint(w * f32(2048)), -32768, 32767).astype(np.int16)
    return base, coef


@functools.lru_cache(maxsize=16)
def tables(h_in, w_in, h_out, w_out, device):
    """(xtab, ytab): int32 CUDA tensors [w_out, 9] and [h_out, 9] on `device` (a torch.device), each row the base index
    and the eight weights -- the layout teco_resize_lanczos4_u8 reads.  Cached per sizes and device."""
    import torch

    def pack(n_in, n_out):
        base, coef = axis_table(n_in, n_out)
        return torch.from_numpy(np.concatenate([base[:, None], coef.astype(np.int32)], axis=1)).to(device)
    return pack(w_in, w_out), pack(h_in, h_out)
