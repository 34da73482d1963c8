"""Host restatement, in numpy, of cv2.cvtColor(..., COLOR_RGB2YUV_I420) and cv2.cvtColor(..., COLOR_YUV2RGB_I420) on
uint8 frames of even sides (cv2 4.13.0, BT.601 limited range, 20-bit fixed point): the colour conversions behind
`main.py --input_y4m / --output_y4m`.  `tecogan_b200/csrc/yuv.cu` computes the same bytes (DESIGN.md section 4.12).

  I420      [3h/2, w] uint8: the Y plane (h x w), then U (h/2 x w/2), then V (h/2 x w/2), each packed.
  RGB->I420 Y = (269484 R + 528482 G + 102760 B + HALF + (16 << 20)) >> 20 for every pixel;
            U = (-155188 R - 305135 G + 460324 B + HALF + (128 << 20)) >> 20 and
            V = (460324 R - 385875 G - 74448 B + HALF + (128 << 20)) >> 20 from the top-left pixel of each 2x2 block
            (cv2 does not average the block).
  I420->RGB u = U - 128, v = V - 128 of the pixel's 2x2 block, y = max(0, Y - 16) * 1220542;
            R = sat8((y + HALF + 1673527 v) >> 20), G = sat8((y + HALF - 852492 v - 409993 u) >> 20),
            B = sat8((y + HALF + 2116026 u) >> 20).
HALF = 1 << 19; >> is an arithmetic shift.
"""
import numpy as np

S = 20
HALF = 1 << (S - 1)


def _check_even(h, w):
    if h < 2 or w < 2 or h % 2 or w % 2:
        raise ValueError("I420 needs even sides >= 2, got %dx%d" % (h, w))


def rgb_to_i420(rgb):
    """uint8 [h, w, 3] RGB -> uint8 [3h/2, w] I420."""
    h, w = rgb.shape[:2]
    _check_even(h, w)
    r, g, b = (rgb[:, :, c].astype(np.int64) for c in range(3))
    y = (269484 * r + 528482 * g + 102760 * b + HALF + (16 << S)) >> S
    r, g, b = r[::2, ::2], g[::2, ::2], b[::2, ::2]
    u = (-155188 * r - 305135 * g + 460324 * b + HALF + (128 << S)) >> S
    v = (460324 * r - 385875 * g - 74448 * b + HALF + (128 << S)) >> S
    flat = np.concatenate([y.ravel(), u.ravel(), v.ravel()]).astype(np.uint8)
    return flat.reshape(3 * h // 2, w)


def i420_to_rgb(i420):
    """uint8 [3h/2, w] I420 -> uint8 [h, w, 3] RGB."""
    h, w = i420.shape[0] * 2 // 3, i420.shape[1]
    _check_even(h, w)
    if i420.shape[0] != 3 * h // 2:
        raise ValueError("I420 buffers have 3h/2 rows, got %d" % i420.shape[0])
    flat = i420.ravel().astype(np.int64)
    n, q = h * w, (h // 2) * (w // 2)
    Y = flat[:n].reshape(h, w)
    U = flat[n:n + q].reshape(h // 2, w // 2).repeat(2, 0).repeat(2, 1) - 128
    V = flat[n + q:n + 2 * q].reshape(h // 2, w // 2).repeat(2, 0).repeat(2, 1) - 128
    y = np.maximum(Y - 16, 0) * 1220542 + HALF
    r = (y + 1673527 * V) >> S
    g = (y - 852492 * V - 409993 * U) >> S
    b = (y + 2116026 * U) >> S
    return np.clip(np.stack([r, g, b], axis=2), 0, 255).astype(np.uint8)
