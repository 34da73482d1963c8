"""Host restatement, in numpy, of the float32 arithmetic of `cv2.GaussianBlur(im, (0, 0), sigmaX=1.5)` on an interleaved
3-channel float32 frame (cv2 4.13.0), and of the inference input the reference builds from it: `blur[::4, ::4] / 255`
(reference lib/dataloader.py:38-43).  `tecogan_b200/csrc/gauss_blur.cu` computes the same numbers (DESIGN.md section 4.9).

  taps        ksize = cvRound(1.5 * 4 * 2 + 1) | 1 = 13, cv2.getGaussianKernel(13, 1.5, CV_32F): TAPS below
  border      BORDER_REFLECT_101 on both axes, cv2's borderInterpolate (the reflection repeats on frames under 7 pixels)
  row pass    element e of an n = 3W float row: s = 0; s = op(k[t], x[e + 3(t - 6)], s) for t = 0..12
  column pass c = k[6] * r[y]; c = op(k[6 + t], r[y + t] + r[y - t], c) for t = 1..6, the pair sum rounded first
  op          fmaf on the vector body of the row, product-then-sum on its tail (`fma_mask` / `column_fma_mask`)

The element index e counts floats of the BGR row cv2 sees: RGB channel c sits at e = 3x + 2 - c.  fmaf is emulated
exactly: the product of two float32 values is exact in float64, and the float64 sum is rounded to odd (TwoSum) so that
its rounding to float32 is the single rounding of a fused multiply-add.
"""
import numpy as np

RADIUS = 6
# cv2.getGaussianKernel(13, 1.5, CV_32F), taps 6..12 (the kernel is symmetric)
HALF = np.array([float.fromhex(h) for h in ("0x1.1058fp-2", "0x1.b42852p-3", "0x1.bfdc88p-4", "0x1.26dd9ep-5",
                                            "0x1.f1e742p-8", "0x1.0d891ap-10", "0x1.763864p-14")], np.float32)
TAPS = np.concatenate([HALF[:0:-1], HALF]).astype(np.float32)


def border101(p, n):
    """cv2.borderInterpolate(p, n, BORDER_REFLECT_101) for n >= 2, elementwise over an int array."""
    p = np.array(p, np.int64)
    while True:
        lo, hi = p < 0, p >= n
        if not (lo.any() or hi.any()):
            return p
        p = np.where(lo, -p, np.where(hi, 2 * n - 2 - p, p))


def fmaf(a, b, c):
    """float32 fused multiply-add a * b + c with one rounding, elementwise (a * b exact in float64)."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bp = s - c64
    err = (c64 - (s - bp)) + (p - bp)                 # TwoSum: s + err == p + c exactly
    bits = s.view(np.int64)
    even = (bits & 1) == 0
    toward = np.where(err > 0, np.inf, -np.inf)
    s = np.where((err != 0) & even, np.nextafter(s, toward), s)   # round to odd: float32 rounding is then exact
    return s.astype(np.float32)


def muladd(a, b, c):
    """float32 a * b rounded, then + c rounded."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    return (a * b).astype(np.float32) + c


def fma_mask(n):
    """bool [n]: the elements of an n-float row whose row pass uses fmaf."""
    body = 8 * (n // 8)
    if n - body >= 4:
        body += 4
    return np.arange(n) < body


def column_fma_mask(n):
    """bool [n]: the elements of an n-float row whose column pass uses fmaf."""
    return np.arange(n) < 8 * (n // 8)


def _op(mask, a, b, c):
    return np.where(mask, fmaf(a, b, c), muladd(a, b, c))


def blur_bgr(im):
    """float32 [H, W, 3] BGR frame (H, W >= 2) -> cv2.GaussianBlur(im, (0, 0), sigmaX=1.5), element for element."""
    im = np.asarray(im, np.float32)
    H, W, C = im.shape
    if H < 2 or W < 2:
        raise ValueError("blur_bgr: frames need H, W >= 2, got %dx%d" % (H, W))
    n = W * C
    x = np.arange(W)
    fm = fma_mask(n).reshape(W, C)
    r = np.zeros((H, W, C), np.float32)
    for t in range(2 * RADIUS + 1):
        src = im[:, border101(x + t - RADIUS, W), :]
        r = _op(fm, TAPS[t], src, r)
    cm = column_fma_mask(n).reshape(W, C)
    y = np.arange(H)
    out = (HALF[0] * r).astype(np.float32)
    for t in range(1, RADIUS + 1):
        pair = r[border101(y + t, H)] + r[border101(y - t, H)]
        out = _op(cm, HALF[t], pair, out)
    return out


def down4_rgb(frame):
    """The reference's HR -> LR input: uint8 or uint16 [H, W, 3] RGB -> float32 [ceil(H/4), ceil(W/4), 3]
    = GaussianBlur(frame as float32)[::4, ::4] / 255 (float32 division), computed in cv2's BGR element order."""
    bgr = np.ascontiguousarray(np.asarray(frame)[:, :, ::-1]).astype(np.float32)
    return np.ascontiguousarray(blur_bgr(bgr)[::4, ::4, ::-1]) / np.float32(255.0)


def reference_input(frame_bgr, down):
    """The parent's host formula on a frame as cv2.imread(path, 3) returns it (BGR, uint8 or uint16), with cv2 itself:
    RGB float32 / 255, blurred and sampled first when `down`."""
    import cv2
    im = frame_bgr.astype(np.float32)[:, :, ::-1]
    if down:
        im = cv2.GaussianBlur(im, (0, 0), sigmaX=1.5)[::4, ::4, ::]
    return np.ascontiguousarray(im / 255.0)
