"""Host restatement of the partitions of the fixed-order (*_det) entry points (include/teco.h, DESIGN.md section 4.3).
Every number here is a function of the call's shapes: the partitions take no device property, so a run on any H100
splits, and therefore sums, the same way."""

WG_ROWS, WG_COLS, WG_DET_CTAS = 8, 16, 264      # conv_wgrad_tc.cu
DET_SMS, BK = 132, 16                           # conv_simt.cu
DET_BN_BLOCKS, DET_LOSS_BLOCKS, TPB = 264, 2112, 256   # eltwise.cu
WD_SCAN = 1024                                  # resample.cu


def cdiv(a, b):
    return -(-a // b)


def wgrad_tc(N, H, W, cin, cout):
    """(splits, tiles per split) of teco_conv3x3_wgrad_tc_det: split x runs tiles [x * tpc, (x + 1) * tpc)."""
    tiles = N * cdiv(W, WG_COLS) * cdiv(H, WG_ROWS)
    pairs = cdiv(cin, 64) * cdiv(cout, 64)
    splits = min(cdiv(WG_DET_CTAS, pairs), tiles)
    tpc = cdiv(tiles, splits)
    return cdiv(tiles, tpc), tpc


def wgrad_tc_bytes(N, H, W, cin, cout):
    return wgrad_tc(N, H, W, cin, cout)[0] * 9 * cin * cout * 4


def wgrad_f32(M, KH, KW, Cin, Cout):
    """(splits, pixels per split) of teco_conv2d_wgrad_f32_det over M output pixels."""
    base = cdiv(Cin, 64) * KH * KW * cdiv(Cout, 64)
    splits = cdiv(4 * DET_SMS, base)
    splits = max(1, min(splits, cdiv(M, 256), 65535))
    pps = cdiv(cdiv(M, splits), BK) * BK
    return cdiv(M, pps), pps


def bias(M, C):
    """(blocks, pixels per block) of the fixed-order bias gradient; each block runs 256 // C pixel lanes."""
    ppb = 8 * (256 // C)
    blocks = cdiv(M, ppb)
    if blocks > 16 * DET_SMS:
        blocks = 16 * DET_SMS
        ppb = cdiv(M, blocks)
        blocks = cdiv(M, ppb)
    return blocks, ppb


def wgrad_f32_bytes(M, KH, KW, Cin, Cout, with_bias):
    return (wgrad_f32(M, KH, KW, Cin, Cout)[0] * KH * KW * Cin * Cout + (bias(M, Cout)[0] * Cout if with_bias else 0)) * 4


def bn(npix):
    """(blocks, pixels per block) of the fixed-order batch-norm statistics and their gradient."""
    blocks = min(cdiv(npix, 1024), DET_BN_BLOCKS)
    ppb = cdiv(npix, blocks)
    return cdiv(npix, ppb), ppb


def loss_blocks(kind, npix, C):
    """Blocks of the fixed-order losses: 'l2', 'l1' over npix * C values, 'cosine' one warp per pixel, 'gan' over npix."""
    n, per = {"l2": (npix * C, TPB * 4), "l1": (npix * C, TPB * 4), "cosine": (npix * 32, TPB), "gan": (npix, TPB * 4)}[kind]
    return max(1, min(cdiv(n, per), DET_LOSS_BLOCKS))


def loss_bytes(npix, C):
    return 4 * max(loss_blocks("l2", npix, C), loss_blocks("l1", npix, C), loss_blocks("cosine", npix, C),
                   5 * loss_blocks("gan", npix, C))


def warp_bytes(N, H, W):
    P = N * H * W
    return 4 * (6 * P + cdiv(P, WD_SCAN))
