"""Case tables of tests/test_gpu_resample_exact.py, their seeded inputs, and a host restatement of which edges of the
resampling kernels (csrc/resample.cu) each case reaches.

The inputs sit on coarse dyadic grids so that every fp32 intermediate of the kernels is exact (the GPU test asserts
that per case before it compares).  `keys(family, name)` classifies a case from its inputs, as the kernel would see
them: for the warp, which class alpha_raw = q - clamp(floor(q), 0, size-2) falls in on each axis; for max-pool, which
window positions tie for the maximum; for the bf16 ×2 resize, which fp32 blends are exact bf16 rounding midpoints and
which way round-to-nearest-even takes them; for bicubic_four, which kernel the entry point dispatches to (the RGB
fast path needs C == 3 and a 16-byte-aligned output); and whether the launch is larger than one grid-stride pass.
tests/test_host_logic.py checks that the tables reach every key in REQUIRED.

A launch covers at most 32 blocks of 256 threads per SM (`grid_for`); above that each thread takes more than one
grid-stride step.  The table is classified at 132 SMs (H100 SXM); the GPU test recomputes the cap from the device.
"""
import zlib
from collections import namedtuple

import numpy as np

TPB, BLOCKS_PER_SM = 256, 32


def cap(sms=132):
    """Threads of one grid-stride pass."""
    return BLOCKS_PER_SM * sms * TPB


def rng(name):
    return np.random.RandomState(zlib.crc32(name.encode()) & 0x7FFFFFFF)


def grid(a, e):
    """float32 values of a rounded to the 2^-e grid."""
    return (np.round(np.asarray(a, np.float64) * 2.0 ** e) / 2.0 ** e).astype(np.float32)


def uniform(r, shape, e, lo=-1.0, hi=1.0):
    return grid(r.uniform(lo, hi, shape), e)


# ----------------------------------------------------------------------------------------------------------- warp
# name: N, H, W, C, outlier probability, which frames have zero flow ("mid": every third frame from the second, the
# middle frame of each Dt triplet, lib/Teco.py:186)
Warp = namedtuple("Warp", "N H W C p_far zero")
WARP = {
    "5x7_c3": Warp(2, 5, 7, 3, 0.08, ()),
    "h2_c1": Warp(2, 2, 9, 1, 0.08, ()),
    "w2_c5": Warp(2, 6, 2, 5, 0.08, ()),
    "h2w2_c3": Warp(3, 2, 2, 3, 0.08, ()),
    "zero_flow_c3": Warp(1, 8, 8, 3, 0.0, "all"),
    "dt_72x128x128": Warp(72, 128, 128, 3, 0.002, "mid"),
}


def warp_inputs(name):
    """img on the 2^-7 grid in [-1, 1], dout on 2^-4, flow = integer shift in [-2, 2] + a 2^-6 fraction that is zero
    on 40 % of the pixels (integer queries: alpha_raw = 0 inside the frame, 1 at q = size-1); a fraction p_far of
    the pixels points 1-20 pixels beyond the frame."""
    c, r = WARP[name], rng("warp " + name)
    sh = (c.N, c.H, c.W)
    img = uniform(r, sh + (c.C,), 7)
    dout = uniform(r, sh + (c.C,), 4)
    frac = np.where(r.rand(*sh, 2) < 0.4, 0.0, r.randint(1, 64, sh + (2,)) / 64.0)
    flow = r.randint(-2, 3, sh + (2,)) + frac
    size = np.array([c.H, c.W], np.float64)
    far = r.rand(*sh, 2) < c.p_far
    far_v = np.where(r.rand(*sh, 2) < 0.5, -1.0, 1.0) * (size + r.randint(1, 21, sh + (2,)))
    flow = grid(np.where(far, far_v, flow), 6)
    if c.zero == "all":
        flow[:] = 0
    elif c.zero == "mid":
        flow[1::3] = 0
    return img, flow, dout


def alpha_classes(q, size, axis):
    fl = np.clip(np.floor(q), 0, size - 2)
    a = q - fl
    out = set()
    for k, m in (("alpha<=-1", a <= -1), ("alpha in (-1,0)", (a > -1) & (a < 0)), ("alpha=0 at q=0", (a == 0) & (q == 0)),
                 ("alpha=0 interior", (a == 0) & (q > 0)), ("alpha in (0,1)", (a > 0) & (a < 1)),
                 ("alpha=1 at q=size-1", (a == 1) & (q == size - 1)), ("alpha>1", a > 1)):
        if m.any():
            out.add("%s %s" % (axis, k))
    return out


def _warp_keys(name, sms):
    c = WARP[name]
    _, flow, _ = warp_inputs(name)
    qy = np.arange(c.H, dtype=np.float32)[None, :, None] - flow[..., 0]
    qx = np.arange(c.W, dtype=np.float32)[None, None, :] - flow[..., 1]
    k = alpha_classes(qy, c.H, "y") | alpha_classes(qx, c.W, "x") | {"C=%d" % c.C}
    k |= {"H=2"} if c.H == 2 else set()
    k |= {"W=2"} if c.W == 2 else set()
    k |= {"zero flow"} if (flow.reshape(c.N, -1) == 0).all(1).any() else set()
    k |= {"above cap"} if c.N * c.H * c.W > cap(sms) else set()
    return k


# -------------------------------------------------------------------------------------------- legacy bilinear resize
# name: N, h, w, C, oh, ow.  x2 is FNet's decoder in fp32, x4 is upscale_four and lib/Teco.py:183 (9 channels)
Resize = namedtuple("Resize", "N h w C oh ow")
RESIZE = {
    "x2_fnet": Resize(2, 4, 5, 8, 8, 10),
    "x4_upscale": Resize(2, 6, 7, 2, 24, 28),
    "x1_odd": Resize(1, 5, 7, 3, 5, 7),
    "x2_odd": Resize(2, 9, 7, 5, 18, 14),
    "x4_odd_1px": Resize(1, 1, 3, 2, 4, 12),
    "x4_teco183": Resize(24, 32, 32, 9, 128, 128),
    "5to7_up": Resize(2, 5, 5, 3, 7, 7),
    "7to5_down": Resize(2, 7, 7, 3, 5, 5),
}


def resize_dyadic(c):
    return all((o / i) in (1, 2, 4) for i, o in ((c.h, c.oh), (c.w, c.ow)))


def resize_inputs(name):
    """x on the 2^-7 grid in [-1, 1] and the incoming gradient on 2^-7."""
    c, r = RESIZE[name], rng("resize " + name)
    return uniform(r, (c.N, c.h, c.w, c.C), 7), uniform(r, (c.N, c.oh, c.ow, c.C), 7)


def _resize_keys(name, sms):
    c = RESIZE[name]
    k = set()
    for i, o in ((c.h, c.oh), (c.w, c.ow)):
        k.add("x%d" % (o // i) if o % i == 0 else ("non-dyadic up" if o > i else "non-dyadic down"))
    k |= {"odd h"} if c.h % 2 else set()
    k |= {"odd w"} if c.w % 2 else set()
    k |= {"above cap"} if c.N * c.oh * c.ow * c.C > cap(sms) else set()
    return k


# ---------------------------------------------------------------------------------------------------- max-pool fp32
Pool = namedtuple("Pool", "N H W C relu")
MAXPOOL = {
    "c1_odd_h": Pool(2, 7, 8, 1, False),
    "c3_odd_w": Pool(2, 6, 9, 3, True),
    "c64_odd_hw": Pool(1, 9, 7, 64, True),
    "c64_even": Pool(2, 8, 10, 64, False),
    "above_cap_c64": Pool(3, 160, 161, 64, True),
}
POS = ("TL", "TR", "BL", "BR")


def maxpool_inputs(name):
    """Values in {-2, ..., 3} / 8 (ReLU'd to [0, 3/8] where `relu`): many ties, and all-zero windows after the ReLU."""
    c, r = MAXPOOL[name], rng("maxpool " + name)
    x = r.randint(-2, 4, (c.N, c.H, c.W, c.C)) / 8.0
    if c.relu:
        x = np.maximum(x, 0.0)
    return x.astype(np.float32), uniform(r, (c.N, c.H // 2, c.W // 2, c.C), 7)


def windows(x):
    """[N, H/2, W/2, 4, C]: the 2x2 windows in TL, TR, BL, BR order (the dropped odd row / column excluded)."""
    N, H, W, C = x.shape
    oh, ow = H // 2, W // 2
    return x[:, :2 * oh, :2 * ow].reshape(N, oh, 2, ow, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, oh, ow, 4, C)


def _maxpool_keys(name, sms):
    c = MAXPOOL[name]
    win = windows(maxpool_inputs(name)[0])
    eq = win == win.max(3, keepdims=True)
    k = {"C=%d" % c.C}
    k |= {"all equal"} if eq.all(3).any() else set()
    for a in range(4):
        for b in range(a + 1, 4):
            if (eq[:, :, :, a] & eq[:, :, :, b]).any():
                k.add("tie %s/%s" % (POS[a], POS[b]))
    k |= {"odd H"} if c.H % 2 else set()
    k |= {"odd W"} if c.W % 2 else set()
    k |= {"above cap"} if c.N * (c.H // 2) * (c.W // 2) * c.C > cap(sms) else set()
    return k


# ----------------------------------------------------------------------------------------------------- bicubic_four
# name: N, h, w, C, in_cpitch, byte offset of the output from a 16-byte boundary
Bicubic = namedtuple("Bicubic", "N h w C cpitch out_off")
BICUBIC = {
    "rgb_3x5": Bicubic(2, 3, 5, 3, 3, 0),
    "rgb_1x2_pitch51": Bicubic(2, 1, 2, 3, 51, 0),
    "rgb_offset4_2x3": Bicubic(2, 2, 3, 3, 3, 4),
    "c1_1x1": Bicubic(2, 1, 1, 1, 1, 0),
    "c2_3x2_pitch51": Bicubic(1, 3, 2, 2, 51, 0),
    "c4_2x3": Bicubic(2, 2, 3, 4, 4, 0),
    "rgb_above_cap": Bicubic(4, 264, 264, 3, 3, 0),
    "c1_above_cap": Bicubic(2, 192, 192, 1, 1, 0),
}


def bicubic_rgb_path(c):
    return c.C == 3 and c.out_off % 16 == 0


def bicubic_threads(c):
    return c.N * c.h * 4 * c.w * (1 if bicubic_rgb_path(c) else 4 * c.C)


def bicubic_inputs(name):
    """x [N, h, w, cpitch] on the 2^-6 grid in [-1, 1]; channels from C on hold 2^20, which no output can absorb."""
    c, r = BICUBIC[name], rng("bicubic " + name)
    x = np.full((c.N, c.h, c.w, c.cpitch), 2.0 ** 20, np.float32)
    x[..., :c.C] = uniform(r, (c.N, c.h, c.w, c.C), 6)
    return x


def _bicubic_keys(name, sms):
    c = BICUBIC[name]
    k = {"rgb path" if bicubic_rgb_path(c) else "generic path", "C=%d" % c.C, "h=%d" % c.h, "w=%d" % c.w}
    k |= {"C=3 generic (unaligned output)"} if c.C == 3 and not bicubic_rgb_path(c) else set()
    k |= {"in_cpitch>C"} if c.cpitch > c.C else set()
    if bicubic_threads(c) > cap(sms):
        k.add("above cap " + ("rgb" if bicubic_rgb_path(c) else "generic"))
    return k


# ------------------------------------------------------------------------------------------------------ upscale_four
Up = namedtuple("Up", "N h w C scale")
UPSCALE = {
    "h1_c2_s4": Up(2, 1, 5, 2, 4.0),
    "w1_c3": Up(2, 4, 1, 3, 1.0),
    "3x4_c3_s4": Up(1, 3, 4, 3, 4.0),
    "above_cap_c2_s4": Up(4, 96, 96, 2, 4.0),
}


def upscale_inputs(name):
    c, r = UPSCALE[name], rng("upscale " + name)
    return uniform(r, (c.N, c.h, c.w, c.C), 7)


def _upscale_keys(name, sms):
    c = UPSCALE[name]
    k = {"C=%d" % c.C, "scale %g" % c.scale}
    k |= {"h=1"} if c.h == 1 else set()
    k |= {"w=1"} if c.w == 1 else set()
    k |= {"above cap"} if c.N * 16 * c.h * c.w * c.C > cap(sms) else set()
    return k


# ------------------------------------------------------------------------------------- space-to-depth / depth-to-space
S2d = namedtuple("S2d", "N h w C pitch ch_off")
S2D = {
    "c3_dense": S2d(2, 3, 5, 3, 48, 0),
    "c3_pitch51_off3": S2d(2, 2, 3, 3, 51, 3),
    "c1_pitch40_off17": S2d(1, 3, 2, 1, 40, 17),
    "c5_pitch96_off8": S2d(2, 1, 2, 5, 96, 8),
    "above_cap_c3_pitch64_off8": S2d(4, 80, 80, 3, 64, 8),
}


def s2d_inputs(name):
    """Arbitrary float32 bit patterns (no NaN), with +-0.0, +-inf and subnormals among them."""
    c, r = S2D[name], rng("s2d " + name)
    n = c.N * 16 * c.h * c.w * c.C
    bits = r.randint(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32).copy()
    x[np.isnan(x)] = 1.5
    x[:8] = np.float32([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1.0, -1.0])[:min(8, n)]
    return x.reshape(c.N, 4 * c.h, 4 * c.w, c.C)


def _s2d_keys(name, sms):
    c = S2D[name]
    x = s2d_inputs(name)
    k = set()
    k |= {"pitch>16C"} if c.pitch > 16 * c.C else set()
    k |= {"ch_off>0"} if c.ch_off > 0 else set()
    k |= {"-0.0"} if (np.signbit(x) & (x == 0)).any() else set()
    k |= {"above cap"} if c.N * 16 * c.h * c.w * c.C > cap(sms) else set()
    return k


# ------------------------------------------------------------------------------------------------ Gaussian LR synthesis
Gauss = namedtuple("Gauss", "N H W C")
GAUSS = {
    "loader_crop32": Gauss(2, 4 * 32 + 8, 4 * 32 + 8, 3),     # HRClipLoader's 4 crop + 8: the last 3 rows unused
    "h9_w9": Gauss(2, 9, 9, 3),
    "h13_w17": Gauss(1, 13, 17, 2),                          # H, W = 1 (mod 4): every row and column used
    "above_cap_crop152": Gauss(16, 4 * 152 + 8, 4 * 152 + 8, 3),
}


def gauss_inputs(name):
    c, r = GAUSS[name], rng("gauss " + name)
    return r.rand(c.N, c.H, c.W, c.C).astype(np.float32)


def _gauss_keys(name, sms):
    c = GAUSS[name]
    k = set()
    k |= {"H=4crop+8"} if c.H % 4 == 0 and c.H > 8 else set()
    k |= {"H=9"} if c.H == 9 else set()
    k |= {"H=1 mod 4"} if c.H % 4 == 1 and c.H > 9 else set()
    oh, ow = (c.H - 9) // 4 + 1, (c.W - 9) // 4 + 1
    k |= {"above cap"} if c.N * oh * ow * c.C > cap(sms) else set()
    return k


# -------------------------------------------------------------------------------------------- FNet bf16 glue kernels
# name: N, H, W, C.  FNet's maxpool inputs at 32x32 are 32, 16, 8 (C 64, 64, 128); at 36x45: 36x45, 18x22, 9x11.  Its
# resize inputs are 4x4, 8x8, 16x16 (C 256, 128, 64) and 4x5, 8x10, 16x20
Bf = namedtuple("Bf", "N H W C")
MAXPOOL_BF16 = {
    "fnet32_l0": Bf(2, 32, 32, 64), "fnet32_l1": Bf(2, 16, 16, 64), "fnet32_l2": Bf(2, 8, 8, 128),
    "fnet36x45_l0": Bf(1, 36, 45, 64), "fnet36x45_l1": Bf(1, 18, 22, 64), "fnet36x45_l2": Bf(1, 9, 11, 128),
    "c8_odd": Bf(2, 5, 7, 8), "c256_odd": Bf(1, 3, 5, 256),
    "above_cap_c256": Bf(34, 64, 64, 256),
}
RESIZE_BF16 = {
    "fnet32_l3": Bf(2, 4, 4, 256), "fnet32_l4": Bf(2, 8, 8, 128), "fnet32_l5": Bf(2, 16, 16, 64),
    "fnet36x45_l3": Bf(1, 4, 5, 256), "fnet36x45_l4": Bf(1, 8, 10, 128), "fnet36x45_l5": Bf(1, 16, 20, 64),
    "c8_1x3": Bf(2, 1, 3, 8), "c8_odd": Bf(2, 5, 7, 8),
    "above_cap_c256": Bf(9, 32, 32, 256),
}


def bf16_values(r, shape):
    """bf16-exact values +-m 2^(e-7), m in [128, 255], e in [-3, 1]: every blend of up to four of them is exact in fp32
    (spread of 5 binades + 8 significant bits + 2 bits of the quarter weights)."""
    m = r.randint(128, 256, shape).astype(np.float64)
    e = r.randint(-3, 2, shape)
    s = np.where(r.rand(*shape) < 0.5, -1.0, 1.0)
    return (s * m * 2.0 ** (e - 7)).astype(np.float32)


def maxpool_bf16_inputs(name):
    c = MAXPOOL_BF16[name]
    return bf16_values(rng("maxpool_bf16 " + name), (c.N, c.H, c.W, c.C))


def resize_bf16_inputs(name):
    c = RESIZE_BF16[name]
    return bf16_values(rng("resize_bf16 " + name), (c.N, c.H, c.W, c.C))


def resize2x_blend(x):
    """float64 of resize2x's fp32 blend on [N, h, w, C]: out[2i] = x[i], out[2i+1] = (x[i] + x[min(i+1, n-1)]) / 2 on
    both axes, x first (exact: see bf16_values)."""
    N, h, w, C = x.shape
    x = x.astype(np.float64)
    iy, ix = np.arange(2 * h), np.arange(2 * w)
    y0, x0 = iy >> 1, ix >> 1
    y1 = np.where(iy & 1, np.minimum(y0 + 1, h - 1), y0)
    x1 = np.where(ix & 1, np.minimum(x0 + 1, w - 1), x0)
    wy = np.where(iy & 1, 0.5, 0.0)[None, :, None, None]
    wx = np.where(ix & 1, 0.5, 0.0)[None, None, :, None]
    a, b = x[:, y0], x[:, y1]
    top = a[:, :, x0] + (a[:, :, x1] - a[:, :, x0]) * wx
    bot = b[:, :, x0] + (b[:, :, x1] - b[:, :, x0]) * wx
    return top + (bot - top) * wy


def bf16_rne_bits(v32):
    """uint16 bits of float32 values rounded to bf16 with round-to-nearest-even (no NaN among them)."""
    b = np.asarray(v32, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _pool_bf16_keys(name, sms):
    c = MAXPOOL_BF16[name]
    k = {"C=%d" % c.C}
    k |= {"odd H"} if c.H % 2 else set()
    k |= {"odd W"} if c.W % 2 else set()
    k |= {"above cap"} if c.N * (c.H // 2) * (c.W // 2) * (c.C // 8) > cap(sms) else set()
    return k


def _resize_bf16_keys(name, sms):
    c = RESIZE_BF16[name]
    v = resize2x_blend(resize_bf16_inputs(name)).astype(np.float32).view(np.uint32)
    low, odd = v & 0xFFFF, (v >> 16) & 1
    k = {"C=%d" % c.C}
    k |= {"midpoint to even (down)"} if ((low == 0x8000) & (odd == 0)).any() else set()
    k |= {"midpoint to even (up)"} if ((low == 0x8000) & (odd == 1)).any() else set()
    k |= {"odd h"} if c.H % 2 else set()
    k |= {"odd w"} if c.W % 2 else set()
    k |= {"above cap"} if c.N * 4 * c.H * c.W * (c.C // 8) > cap(sms) else set()
    return k


FAMILIES = {
    "warp": (WARP, _warp_keys),
    "resize": (RESIZE, _resize_keys),
    "maxpool": (MAXPOOL, _maxpool_keys),
    "bicubic": (BICUBIC, _bicubic_keys),
    "upscale": (UPSCALE, _upscale_keys),
    "s2d": (S2D, _s2d_keys),
    "gauss": (GAUSS, _gauss_keys),
    "maxpool_bf16": (MAXPOOL_BF16, _pool_bf16_keys),
    "resize_bf16": (RESIZE_BF16, _resize_bf16_keys),
}

REQUIRED = {
    "warp": {"%s %s" % (a, k) for a in "yx" for k in ("alpha<=-1", "alpha in (-1,0)", "alpha=0 at q=0", "alpha=0 interior",
                                                       "alpha in (0,1)", "alpha=1 at q=size-1", "alpha>1")}
    | {"H=2", "W=2", "C=1", "C=3", "C=5", "zero flow", "above cap"},
    "resize": {"x1", "x2", "x4", "non-dyadic up", "non-dyadic down", "odd h", "odd w", "above cap"},
    "maxpool": {"all equal", "odd H", "odd W", "C=1", "C=3", "C=64", "above cap"}
    | {"tie %s/%s" % (POS[a], POS[b]) for a in range(4) for b in range(a + 1, 4)},
    "bicubic": {"rgb path", "generic path", "C=1", "C=2", "C=3", "C=4", "C=3 generic (unaligned output)", "in_cpitch>C",
                "h=1", "h=2", "h=3", "w=1", "w=2", "w=3", "above cap rgb", "above cap generic"},
    "upscale": {"h=1", "w=1", "C=2", "C=3", "scale 4", "above cap"},
    "s2d": {"pitch>16C", "ch_off>0", "-0.0", "above cap"},
    "gauss": {"H=4crop+8", "H=9", "H=1 mod 4", "above cap"},
    "maxpool_bf16": {"odd H", "odd W", "C=8", "C=64", "C=256", "above cap"},
    "resize_bf16": {"midpoint to even (down)", "midpoint to even (up)", "odd h", "odd w", "C=8", "C=64", "C=256",
                    "above cap"},
}


def keys(family, name, sms=132):
    return FAMILIES[family][1](name, sms)
