"""Host restatement, in numpy, of `cv2.resize(frame, (0, 0), fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)` on a uint8
3-channel frame (cv2 4.13.0): the down-sample the reference's data preparation applies to every training frame
(reference lib/data/video.py:168-173).  `tecogan_b200/csrc/area_down2.cu` computes the same numbers (DESIGN.md section
4.10).

  size     oh = cvRound(H * 0.5), ow = cvRound(W * 0.5), halves rounded to even: 721 -> 360, 5 -> 2, 3 -> 2, 7 -> 4.
           A side of 4k + 1 drops its last source line; a side of 4k + 3 gains an output line over one source line.
  scale    cv2 derives the scale from fx and fy, not from the sizes, so it is exactly 2 on both axes whatever their
           parity, and every size runs cv2's integer-scale ("area fast") path: no fractional weights, no float sums.
  inside   an output whose 2 x 2 source block lies inside the frame: (a + b + c + d + 2) >> 2.
  border   an output on the last row when H = 4k + 3 (every column of it), or on the last column when W = 4k + 3:
           the integer sum of its in-frame sources over their count (2, or 1 at the corner), as a float32, rounded
           half to even.  So a border pair rounds (a + b) / 2 to even, where an inside block rounds its halves up.
"""
import numpy as np


def out_size(n):
    """cv2's saturate_cast<int>(n * 0.5): round half to even."""
    return int(np.rint(n * 0.5))


def area_half(frame):
    """uint8 [H, W, 3] frame, 2 <= H, W -> uint8 [cvRound(H/2), cvRound(W/2), 3] equal to cv2's INTER_AREA resize by
    fx = fy = 0.5.  Channels are independent, so their order does not matter."""
    f = np.asarray(frame)
    if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
        raise ValueError("area_half: need a uint8 [H, W, 3] frame, got %s %s" % (f.dtype, f.shape))
    H, W = f.shape[:2]
    if H < 2 or W < 2:
        raise ValueError("area_half: frames need H, W >= 2, got %dx%d" % (H, W))
    oh, ow = out_size(H), out_size(W)
    fh, fw = H // 2, W // 2                                      # outputs whose block is whole on that axis
    s = f.astype(np.int32)
    out = np.empty((oh, ow, 3), np.uint8)
    q = s[0:2 * fh:2, 0:2 * fw:2] + s[0:2 * fh:2, 1:2 * fw:2] + s[1:2 * fh:2, 0:2 * fw:2] + s[1:2 * fh:2, 1:2 * fw:2]
    out[:min(fh, oh), :min(fw, ow)] = ((q[:oh, :ow] + 2) >> 2).astype(np.uint8)
    if oh > fh:                                                  # last row: one source row, pairs and a corner
        row = s[H - 1]
        pair = row[0:2 * fw:2] + row[1:2 * fw:2]
        out[oh - 1, :min(fw, ow)] = np.rint(pair[:ow].astype(np.float32) / np.float32(2)).astype(np.uint8)
    if ow > fw:                                                  # last column: one source column
        col = s[:, W - 1]
        pair = col[0:2 * fh:2] + col[1:2 * fh:2]
        out[:min(fh, oh), ow - 1] = np.rint(pair[:oh].astype(np.float32) / np.float32(2)).astype(np.uint8)
    if oh > fh and ow > fw:
        out[oh - 1, ow - 1] = f[H - 1, W - 1]
    return out
