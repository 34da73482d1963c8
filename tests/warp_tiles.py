"""Host restatement, in float32 as the kernels compute it, of how the two fused warp + space-to-depth kernels choose a path
for each tile (csrc/warp_s2d_v2.cu::warp_s2d_v2_kernel, csrc/resample.cu::warp_s2d_fused_kernel).

Both kernels bound the HR flow over a tile by the min / max of the 4 x flow_lr samples around it (upscale_four is a convex
combination of them), derive the rows / columns of the previous HR frame that the tile's bilinear queries can touch, and
pick a path from that window:
  * v2 (4 x 32 LR tile, 5 x 33 samples): the whole window staged by bulk copies when it fits the 40 KB stage, in one of four
    variants IY / IX ("no query of the tile can touch a clamp on this axis"); otherwise the tile in two halves of 2 LR rows,
    each staged (S) through its own mbarrier phase or gathered from global memory through L1 (G);
  * v1 (2 x 32 LR tile, 3 x 33 samples): the window in shared memory or a global gather, each with or without the
    `interior` shortcut (no clamp on either axis).
"""
from collections import namedtuple

import numpy as np

f32 = np.float32
V2_TLH, V2_TLW, V2_WIN_FLOATS = 4, 32, 10 * 1024
V1_TLH, V1_TLW, V1_SMEM_FLOATS = 2, 32, 8 * 1024

Window = namedtuple("Window", "y_lo y_hi x_lo x_hi int_y int_x qy_lo qy_hi qx_lo qx_hi")


def window(mny, mxy, mnx, mxx, Yt, nrows, X0, H, W):
    """Source window of HR rows [Yt, Yt + nrows) x columns [X0, X0 + 128) for flow bounds (float32) over the tile: queries
    Y - fy lie in [qy_lo, qy_hi], the floor is clamped to [0, H-2], plus the +1 neighbour; columns in whole groups of four
    pixels (16-byte aligned fp32 RGB rows).  int_y / int_x: every query lies at least one pixel inside [0, size-2]."""
    clampf = lambda v, hi: min(max(v, f32(0)), f32(hi))
    qy_lo, qy_hi = f32(Yt) - mxy, f32(Yt + nrows - 1) - mny
    qx_lo, qx_hi = f32(X0) - mxx, f32(X0 + 4 * V2_TLW - 1) - mnx
    y_lo = int(clampf(np.floor(qy_lo) - f32(1), H - 2))
    y_hi = int(clampf(np.floor(qy_hi) + f32(1), H - 2)) + 1
    x_lo = int(clampf(np.floor(qx_lo) - f32(1), W - 2)) & ~3
    x_hi = min((int(clampf(np.floor(qx_hi) + f32(1), W - 2)) + 1) | 3, W - 1)
    int_y = bool(qy_lo >= 1 and qy_hi <= H - 3)
    int_x = bool(qx_lo >= 1 and qx_hi <= W - 3)
    return Window(y_lo, y_hi, x_lo, x_hi, int_y, int_x, qy_lo, qy_hi, qx_lo, qx_hi)


def v2_staged(v):
    return (v.y_hi - v.y_lo + 1) * (v.x_hi - v.x_lo + 1) * 3 <= V2_WIN_FLOATS


def v1_staged(v):
    n = (v.y_hi - v.y_lo + 1) * (v.x_hi - v.x_lo + 1)
    return n * 3 <= V1_SMEM_FLOATS and n * 2 <= 5 * (4 * V1_TLH) * (4 * V1_TLW)


def tile_bounds(flow4, ly0, lx0, tlh, h, w):
    """min / max of fy, fx over the (tlh + 1) x 33 samples of 4 * flow_lr [fh, fw, 2] (float32) around an LR tile: indices
    clamped to the frame like upscale_four, then mirrored by tf.pad SYMMETRIC (main.py:212)."""
    fh, fw = flow4.shape[:2]
    ii = np.minimum(np.arange(ly0, ly0 + tlh + 1), h - 1)
    jj = np.minimum(np.arange(lx0, lx0 + V2_TLW + 1), w - 1)
    ii = np.where(ii < fh, ii, 2 * fh - 1 - ii)
    jj = np.where(jj < fw, jj, 2 * fw - 1 - jj)
    s = flow4[np.ix_(ii, jj)]
    return s[..., 0].min(), s[..., 0].max(), s[..., 1].min(), s[..., 1].max()


def v2_tiles(flow_lr, h, w):
    """Yields (ly0, lx0, full-tile window, staged, half windows or None) for every tile of one image of warp_s2d_v2_kernel."""
    flow4 = np.asarray(flow_lr, f32) * f32(4)
    H, W = 4 * h, 4 * w
    for ly0 in range(0, h, V2_TLH):
        for lx0 in range(0, w, V2_TLW):
            b = tile_bounds(flow4, ly0, lx0, V2_TLH, h, w)
            v = window(*b, 4 * ly0, 4 * V2_TLH, 4 * lx0, H, W)
            halves = None if v2_staged(v) else [window(*b, 4 * ly0 + 8 * k, 8, 4 * lx0, H, W) for k in range(2)]
            yield ly0, lx0, v, halves


def v1_tiles(flow_lr, h, w):
    """Yields (ly0, lx0, window) for every tile of one image of warp_s2d_fused_kernel."""
    flow4 = np.asarray(flow_lr, f32) * f32(4)
    H, W = 4 * h, 4 * w
    for ly0 in range(0, h, V1_TLH):
        for lx0 in range(0, w, V1_TLW):
            yield ly0, lx0, window(*tile_bounds(flow4, ly0, lx0, V1_TLH, h, w), 4 * ly0, 4 * V1_TLH, 4 * lx0, H, W)


def paths(flow_lr, h, w):
    """Set of the paths the tiles of one image take, e.g. 'v2 full+IY+IX', 'v2 halves S/G', 'v1 smem+interior', and of the
    interior thresholds met with equality by a tile that still takes the unclamped path ('v2 qy_lo==1', 'v1 qx_hi==W-3')."""
    H, W = 4 * h, 4 * w
    out = set()

    def edges(kernel, v, on_y, on_x):
        for name, q, lim, on in (("qy_lo==1", v.qy_lo, 1, on_y), ("qy_hi==H-3", v.qy_hi, H - 3, on_y),
                                 ("qx_lo==1", v.qx_lo, 1, on_x), ("qx_hi==W-3", v.qx_hi, W - 3, on_x)):
            if on and q == lim:
                out.add("%s %s" % (kernel, name))

    for _, _, v, halves in v2_tiles(flow_lr, h, w):
        if halves is None:
            out.add("v2 full" + ("+IY" if v.int_y else "") + ("+IX" if v.int_x else ""))
            edges("v2", v, v.int_y, v.int_x)
        else:
            out.add("v2 halves " + "/".join("S" if v2_staged(hv) else "G" for hv in halves))
    for _, _, v in v1_tiles(flow_lr, h, w):
        interior = v.int_y and v.int_x
        out.add("v1 " + ("smem" if v1_staged(v) else "global") + ("+interior" if interior else ""))
        edges("v1", v, interior, interior)
    return out
