"""The resampling kernels of csrc/resample.cu and their gradients, called through the C ABI, against a float64 numpy
restatement of each operation as the kernel states it -- bit for bit wherever the inputs make that possible.

Why equality can be required: the inputs (tests/resample_cases.py) sit on coarse dyadic grids.  Pixels are multiples of
2^-7 (2^-6 for bicubic_four), incoming gradients of 2^-4 or 2^-7, flows of 2^-6.  Bilinear weights are then multiples of
2^-6 (warp) or 2^-2 (x2, x4 resizes, upscale_four), and the x4 Keys weights multiples of 2^-8 (for t = 1/4: -27, 225, 67,
-9 over 256).  Every product and partial sum is a multiple of a known power of two and, as `_exact` asserts per case
before comparing, smaller than 2^24 of those units; it is therefore exact in fp32 whatever FMA contraction the compiler
chose and whatever order the atomics of the gradients land in.  For the accumulated gradients the guard bounds every
partial sum by the sum of the absolute values of the terms.  bf16 outputs are compared with round-to-nearest-even of the
exact fp32 value, restated on the bits.

Two operations cannot be made exact and are held to a stated rounding bound instead: the legacy resize at a non-dyadic
ratio (5 -> 7, 7 -> 5) and the Gaussian LR synthesis, whose weights are not dyadic.

Every output is prefilled with a sentinel and followed by a guard region that must stay untouched; pitched outputs also
keep the sentinel in the channels outside the written range.  Each family has a case above one grid-stride pass (32
blocks of 256 threads per SM); those are compared on sampled frames, which always include the last one.
"""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests import resample_cases as R

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
GUARD = 4096
U = 2.0 ** -24                       # unit roundoff of fp32


def _cap():
    return R.cap(torch.cuda.get_device_properties(0).multi_processor_count)


def _assert_multi_pass(threads, name):
    if threads > R.cap():
        assert threads > _cap(), (name, threads, _cap())


def _frames(N, extra=()):
    """Frames a large case is checked on: all of a small batch, else the first and the last (which holds the threads of
    the last grid-stride pass)."""
    return list(range(N)) if N <= 3 else sorted({0, N - 1, *extra})


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _buf(n, dtype=torch.float32, fill=SENTINEL, offset=0):
    """n elements (filled with `fill`) at `offset` elements into a buffer whose other elements hold the sentinel."""
    b = torch.full((offset + n + GUARD,), SENTINEL, dtype=dtype, device="cuda")
    b[offset:offset + n] = fill
    return b, b[offset:offset + n]


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _guard_untouched(b, n, offset, what):
    s = _bits(torch.full((1,), SENTINEL, dtype=b.dtype, device=b.device))
    rest = torch.cat((_bits(b[:offset]), _bits(b[offset + n:])))
    assert (rest == s).all(), "%s: wrote %d elements outside its output" % (what, int((rest != s).sum()))


def _host(t, shape):
    return t.cpu().numpy().reshape(shape)


def _exact(a, e, what):
    """Every value of `a` is a multiple of 2^-e and smaller than 2^24 of those units: representable in fp32."""
    s = np.asarray(a, np.float64) * 2.0 ** e
    assert np.array_equal(s, np.round(s)), "%s: off the 2^-%d grid" % (what, e)
    assert np.abs(s).max(initial=0) < 2 ** 24, "%s: %g units of 2^-%d do not fit 24 bits" % (what, np.abs(s).max(), e)


def _assert_equal(got, exp, what):
    bad = got.astype(np.float64) != exp
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError("%s: %d / %d elements differ, first at %s: got %r, expected %r"
                             % (what, int(bad.sum()), bad.size, i, float(got[i]), float(exp[i])))


def _assert_within(got, exp, tol, what):
    err = np.abs(got.astype(np.float64) - exp)
    bad = err > tol
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError("%s: %d / %d elements beyond the bound, first at %s: err %.3e, bound %.3e"
                             % (what, int(bad.sum()), bad.size, i, err[i], np.broadcast_to(tol, err.shape)[i]))


def _call(name, *args):
    from tecogan_b200._ffi import call, stream_ptr
    call(name, *args, stream_ptr())
    torch.cuda.synchronize()


def _p(t):
    from tecogan_b200._ffi import ptr
    return ptr(t)


# ------------------------------------------------------------------------------------------------------------- warp
def _warp_ref(img, flow, dout):
    """dense_image_warp and both gradients (teco_warp_f32 / teco_warp_bwd_f32): query (y - f0, x - f1), floor clamped to
    [0, size-2], alpha to [0, 1]; top = ax (tr - tl) + tl, bot = ax (br - bl) + bl, out = ay (bot - top) + top.  dimg
    gets the four bilinear weights of the clamped alphas; dflow = -sum_c d out / d query, but only on an axis where
    0 < alpha_raw <= 1 (TF's minimum(maximum(0, a), 1))."""
    img, flow, g = img.astype(np.float64), flow.astype(np.float64), dout.astype(np.float64)
    N, H, W, C = img.shape
    qy = np.arange(H, dtype=np.float64)[None, :, None] - flow[..., 0]
    qx = np.arange(W, dtype=np.float64)[None, None, :] - flow[..., 1]
    _exact(qy, 6, "query y"), _exact(qx, 6, "query x")
    fy, fx = np.clip(np.floor(qy), 0, H - 2), np.clip(np.floor(qx), 0, W - 2)
    ary, arx = qy - fy, qx - fx
    ay, ax = np.clip(ary, 0, 1)[..., None], np.clip(arx, 0, 1)[..., None]
    n, y0, x0 = np.arange(N)[:, None, None], fy.astype(np.int64), fx.astype(np.int64)
    tl, tr, bl, br = img[n, y0, x0], img[n, y0, x0 + 1], img[n, y0 + 1, x0], img[n, y0 + 1, x0 + 1]
    top, bot = ax * (tr - tl) + tl, ax * (br - bl) + bl
    out = ay * (bot - top) + top
    _exact(top, 13, "top"), _exact(bot, 13, "bot"), _exact(out, 19, "out")
    ty = g * (bot - top)
    sx = (1 - ay) * (tr - tl) + ay * (br - bl)
    tx = g * sx
    _exact(sx, 13, "d out / d ax")
    for t, what in ((ty, "dflow y"), (tx, "dflow x")):
        _exact(t, 17, what + " terms"), _exact(np.abs(t).sum(-1), 17, what + " partial sums")
    dflow = np.stack((np.where((ary > 0) & (ary <= 1), -ty.sum(-1), 0.0),
                      np.where((arx > 0) & (arx <= 1), -tx.sum(-1), 0.0)), -1)
    base = ((n * H + y0) * W + x0)[..., None] * C + np.arange(C)
    size = N * H * W * C
    dimg, absum = np.zeros(size), np.zeros(size)
    for off, t in ((0, g * (1 - ay) * (1 - ax)), (C, g * (1 - ay) * ax), (W * C, g * ay * (1 - ax)), (W * C + C, g * ay * ax)):
        _exact(t, 16, "dimg terms")
        dimg += np.bincount((base + off).ravel(), t.ravel(), size)
        absum += np.bincount((base + off).ravel(), np.abs(t).ravel(), size)
    _exact(absum, 16, "dimg partial sums")
    return out, dimg.reshape(N, H, W, C), dflow


@pytest.mark.parametrize("name", list(R.WARP))
def test_warp_and_both_gradients_bit_exact(name):
    """teco_warp_f32 and teco_warp_bwd_f32 with dimg and dflow, dimg alone and dflow alone.  The cases reach every class
    of alpha_raw on both axes (tests/resample_cases.py), H = 2 and W = 2, C in {1, 3, 5}, zero flow, and the 72 x 128 x
    128 x 3 warp of the discriminator's input triplets (lib/Teco.py:186), whose middle frames have zero flow and which
    takes more than one grid-stride pass."""
    c = R.WARP[name]
    img, flow, dout = R.warp_inputs(name)
    N, H, W, C = img.shape
    _assert_multi_pass(N * H * W, name)
    fr = _frames(N, extra=(1,))
    out_r, dimg_r, dflow_r = _warp_ref(img[fr], flow[fr], dout[fr])
    d_img, d_flow, d_dout = _dev(img), _dev(flow), _dev(dout)
    n = N * H * W * C
    b, out = _buf(n)
    _call("teco_warp_f32", _p(d_img), _p(d_flow), _p(out), N, H, W, C)
    _guard_untouched(b, n, 0, name + " warp")
    _assert_equal(_host(out, img.shape)[fr], out_r, name + " warp")
    for with_dimg, with_dflow in ((True, True), (False, True), (True, False)):
        what = "%s bwd%s%s" % (name, " dimg" if with_dimg else "", " dflow" if with_dflow else "")
        bi, dimg = _buf(n, fill=0.0) if with_dimg else (None, None)
        bf, dflow = _buf(N * H * W * 2) if with_dflow else (None, None)
        _call("teco_warp_bwd_f32", _p(d_img), _p(d_flow), _p(d_dout), _p(dimg), _p(dflow), N, H, W, C)
        if with_dimg:
            _guard_untouched(bi, n, 0, what)
            _assert_equal(_host(dimg, img.shape)[fr], dimg_r, what + ": dimg")
        if with_dflow:
            _guard_untouched(bf, N * H * W * 2, 0, what)
            _assert_equal(_host(dflow, flow.shape)[fr], dflow_r, what + ": dflow")


# --------------------------------------------------------------------------------------------- legacy bilinear resize
def _resize_axis(n_in, n_out):
    """Legacy coordinates as the kernel computes them: s = (float)n_in / (float)n_out, f = Y * s in fp32."""
    f = (np.arange(n_out, dtype=np.float32) * (np.float32(n_in) / np.float32(n_out))).astype(np.float64)
    i0 = np.floor(f).astype(np.int64)
    return i0, np.minimum(i0 + 1, n_in - 1), f - i0


def _resize_ref(x, g, oh, ow):
    """Forward (top / bot lerp in x, then y) and the scattered gradient; with Σ|term| and the term count per element."""
    x, g = x.astype(np.float64), g.astype(np.float64)
    N, h, w, C = x.shape
    y0, y1, wy = _resize_axis(h, oh)
    x0, x1, wx = _resize_axis(w, ow)
    a, b = x[:, y0], x[:, y1]
    wx_, wy_ = wx[None, None, :, None], wy[None, :, None, None]
    top = a[:, :, x0] + (a[:, :, x1] - a[:, :, x0]) * wx_
    bot = b[:, :, x0] + (b[:, :, x1] - b[:, :, x0]) * wx_
    out = top + (bot - top) * wy_
    n = np.arange(N)[:, None, None, None]
    cc = np.arange(C)[None, None, None, :]
    size = N * h * w * C
    dx, sg, cnt = np.zeros(size), np.zeros(size), np.zeros(size)
    for yy, xx, t in ((y0, x0, (1 - wy_) * (1 - wx_)), (y0, x1, (1 - wy_) * wx_), (y1, x0, wy_ * (1 - wx_)), (y1, x1, wy_ * wx_)):
        idx = (((n * h + yy[None, :, None, None]) * w + xx[None, None, :, None]) * C + cc).ravel()
        term = np.broadcast_to(g * t, g.shape)
        dx += np.bincount(idx, term.ravel(), size)
        sg += np.bincount(idx, np.abs(g).ravel(), size)
        cnt += np.bincount(idx, None, size)
    return out, top, bot, dx.reshape(x.shape), sg.reshape(x.shape), cnt.reshape(x.shape)


@pytest.mark.parametrize("name", list(R.RESIZE))
def test_resize_bilinear_and_gradient(name):
    """teco_resize_bilinear_f32 and its gradient (memset + atomics).  Dyadic ratios (x1, x2, x4: FNet's decoder,
    upscale_four, lib/Teco.py:183 on 9 channels, which takes more than one grid-stride pass) are exact.

    The non-dyadic ratios (5 -> 7, 7 -> 5) are held to a bound.  The reference uses the kernel's fp32 coordinates; the
    kernel may still contract f - floor(f) with the product Y * s, which moves a weight by at most half an ulp of f <= 7,
    2^-22.  Forward: values in [-1, 1], so every intermediate is below 2 in magnitude and each of at most 8 roundings is
    within 2^-23; the weights' shift moves the convex blends by at most 2 x 2 x 2^-22.  Together below 2^-19.
    Gradient: a term g (1 - wy)(1 - wx) is off by at most |g| (2 (2^-22 + 2^-24) + 2 x 2^-24) < 2^-20 |g|, and each of
    the k atomic adds into an element rounds by at most 2^-23 S, S = sum of |g| over its terms: bound (2^-19 + k 2^-23) S."""
    c = R.RESIZE[name]
    x, g = R.resize_inputs(name)
    _assert_multi_pass(c.N * c.oh * c.ow * c.C, name)
    fr = _frames(c.N)
    out_r, top, bot, dx_r, sg, cnt = _resize_ref(x[fr], g[fr], c.oh, c.ow)
    exact = R.resize_dyadic(c)
    if exact:
        _exact(top, 9, "top"), _exact(bot, 9, "bot"), _exact(out_r, 11, "out")
        _exact(dx_r, 11, "dx")                                   # terms are multiples of 2^-11 and |partials| <= sum |g|
        _exact(sg, 11, "dx partial sums")
    n_out, n_in = c.N * c.oh * c.ow * c.C, c.N * c.h * c.w * c.C
    b, y = _buf(n_out)
    _call("teco_resize_bilinear_f32", _p(_dev(x)), _p(y), c.N, c.h, c.w, c.C, c.oh, c.ow)
    _guard_untouched(b, n_out, 0, name)
    got = _host(y, (c.N, c.oh, c.ow, c.C))[fr]
    if exact:
        _assert_equal(got, out_r, name)
    else:
        _assert_within(got, out_r, 2.0 ** -19, name)
    b, dx = _buf(n_in)
    _call("teco_resize_bilinear_bwd_f32", _p(_dev(g)), _p(dx), c.N, c.h, c.w, c.C, c.oh, c.ow)
    _guard_untouched(b, n_in, 0, name + " bwd")
    got = _host(dx, x.shape)[fr]
    if exact:
        _assert_equal(got, dx_r, name + " bwd")
    else:
        _assert_within(got, dx_r, (2.0 ** -19 + cnt * 2.0 ** -23) * sg, name + " bwd")


# ----------------------------------------------------------------------------------------------------- max-pool fp32
@pytest.mark.parametrize("name", list(R.MAXPOOL))
def test_maxpool2_and_gradient_send_ties_to_the_first_maximum(name):
    """teco_maxpool2_f32 and its gradient: the max of each 2x2 window; the gradient goes to the first maximum in TL, TR,
    BL, BR order (torch's max_pool2d) and every other element, the dropped odd row and column included, gets 0.  The
    inputs tie at every pair of positions and hold all-zero windows (after a ReLU)."""
    c = R.MAXPOOL[name]
    x, g = R.maxpool_inputs(name)
    oh, ow = c.H // 2, c.W // 2
    _assert_multi_pass(c.N * oh * ow * c.C, name)
    win = R.windows(x.astype(np.float64))
    y_r = win.max(3)
    best = win.argmax(3)                                     # first occurrence
    dwin = np.where(np.arange(4)[None, None, None, :, None] == best[:, :, :, None], g[:, :, :, None].astype(np.float64), 0.0)
    dx_r = np.zeros(x.shape)
    dx_r[:, :2 * oh, :2 * ow] = dwin.reshape(c.N, oh, ow, 2, 2, c.C).transpose(0, 1, 3, 2, 4, 5).reshape(c.N, 2 * oh, 2 * ow, c.C)
    d_x = _dev(x)
    b, y = _buf(g.size)
    _call("teco_maxpool2_f32", _p(d_x), _p(y), c.N, c.H, c.W, c.C)
    _guard_untouched(b, g.size, 0, name)
    _assert_equal(_host(y, g.shape), y_r, name)
    b, dx = _buf(x.size)
    _call("teco_maxpool2_bwd_f32", _p(d_x), _p(_dev(g)), _p(dx), c.N, c.H, c.W, c.C)
    _guard_untouched(b, x.size, 0, name + " bwd")
    _assert_equal(_host(dx, x.shape), dx_r, name + " bwd")


# ----------------------------------------------------------------------------------------------------- bicubic_four
def _keys_weights(k):
    """Keys A = -0.75 at t = k/4 as the kernel writes them (exact in float64 and in fp32)."""
    r, t = 0.75, 0.25 * k
    return [-r * t + 2 * r * t * t - r * t ** 3, 1 + (r - 3) * t * t + (2 - r) * t ** 3,
            r * t + (3 - 2 * r) * t * t + (r - 2) * t ** 3, -r * t * t + r * t ** 3]


WT = np.array([_keys_weights(k) for k in range(4)])


def _bicubic_ref(x, C):
    """bicubic_four: edge-replicated taps ly - 1 .. ly + 2, vertical taps first, then horizontal."""
    x = x[..., :C].astype(np.float64)
    N, h, w, _ = x.shape
    Y, X = np.arange(4 * h), np.arange(4 * w)
    yy = np.clip((Y >> 2)[:, None] - 1 + np.arange(4), 0, h - 1)
    xx = np.clip((X >> 2)[:, None] - 1 + np.arange(4), 0, w - 1)
    wy, wx = WT[Y & 3], WT[X & 3]
    col = sum(wy[None, :, b, None, None] * x[:, yy[:, b]] for b in range(4))
    cola = sum(np.abs(wy[None, :, b, None, None]) * np.abs(x[:, yy[:, b]]) for b in range(4))
    out = sum(wx[None, None, :, b, None] * col[:, :, xx[:, b]] for b in range(4))
    outa = sum(np.abs(wx[None, None, :, b, None]) * cola[:, :, xx[:, b]] for b in range(4))
    _exact(col, 14, "column sums"), _exact(cola, 14, "column partial sums")
    _exact(out, 22, "bicubic"), _exact(outa, 22, "bicubic partial sums")
    return out


@pytest.mark.parametrize("name", list(R.BICUBIC))
def test_bicubic4_bit_exact_on_both_kernels(name):
    """teco_bicubic4_f32 on the RGB fast path (C == 3, 16-byte-aligned output) and the generic kernel (C in {1, 2, 4},
    and C == 3 with an output 4 bytes off alignment), in_cpitch = C and 51 (unread channels hold 2^20), frames of 1, 2
    and 3 pixels a side, and both kernels above one grid-stride pass."""
    c = R.BICUBIC[name]
    _exact(WT, 8, "Keys weights")
    x = R.bicubic_inputs(name)
    _assert_multi_pass(R.bicubic_threads(c), name)
    fr = _frames(c.N)
    ref = _bicubic_ref(x[fr], c.C)
    n, off = c.N * 16 * c.h * c.w * c.C, c.out_off // 4
    b, y = _buf(n, offset=off)
    assert y.data_ptr() % 16 == c.out_off
    _call("teco_bicubic4_f32", _p(_dev(x)), _p(y), c.N, c.h, c.w, c.C, c.cpitch)
    _guard_untouched(b, n, off, name)
    _assert_equal(_host(y, (c.N, 4 * c.h, 4 * c.w, c.C))[fr], ref, name)


@pytest.mark.parametrize("N,h,w,cpitch", [(2, 37, 29, 3), (1, 64, 48, 51)])
def test_bicubic4_rgb_fast_path_equals_generic_kernel_on_continuous_inputs(N, h, w, cpitch):
    """resample.cu states the RGB fast path's results are identical to the generic kernel's (same association order).  On
    torch.rand frames, the aligned output (fast path) and an output 4 bytes off (generic kernel) agree bit for bit."""
    x = torch.rand(N, h, w, cpitch, device="cuda", generator=torch.Generator(device="cuda").manual_seed(h))
    n = N * 16 * h * w * 3
    _, fast = _buf(n)
    _, gen = _buf(n, offset=1)
    assert fast.data_ptr() % 16 == 0 and gen.data_ptr() % 16 == 4
    _call("teco_bicubic4_f32", _p(x), _p(fast), N, h, w, 3, cpitch)
    _call("teco_bicubic4_f32", _p(x), _p(gen), N, h, w, 3, cpitch)
    assert torch.equal(_bits(fast), _bits(gen))
    assert not (fast == SENTINEL).any()


# ------------------------------------------------------------------------------------------------------ upscale_four
@pytest.mark.parametrize("name", list(R.UPSCALE))
def test_upscale4_bit_exact(name):
    """teco_upscale4_f32: the four corners (bottom / right neighbours replicated) scaled by `scale` first, then blended
    with the 1/4-step weights tl wy0 wx0 + tr wy0 wx1 + bl wy1 wx0 + br wy1 wx1."""
    c = R.UPSCALE[name]
    x = R.upscale_inputs(name)
    _assert_multi_pass(c.N * 16 * c.h * c.w * c.C, name)
    fr = _frames(c.N)
    xs = x[fr].astype(np.float64) * c.scale
    Y, X = np.arange(4 * c.h), np.arange(4 * c.w)
    ly, lx = Y >> 2, X >> 2
    i1, j1 = np.minimum(ly + 1, c.h - 1), np.minimum(lx + 1, c.w - 1)
    wy1, wx1 = (0.25 * (Y & 3))[None, :, None, None], (0.25 * (X & 3))[None, None, :, None]
    wy0, wx0 = 1 - wy1, 1 - wx1
    a, b = xs[:, ly], xs[:, i1]
    terms = (a[:, :, lx] * wy0 * wx0, a[:, :, j1] * wy0 * wx1, b[:, :, lx] * wy1 * wx0, b[:, :, j1] * wy1 * wx1)
    ref = sum(terms)
    _exact(xs, 7, "scaled corners"), _exact(sum(np.abs(t) for t in terms), 11, "upscale partial sums")
    n = c.N * 16 * c.h * c.w * c.C
    buf, y = _buf(n)
    _call("teco_upscale4_f32", _p(_dev(x)), _p(y), c.N, c.h, c.w, c.C, c.scale)
    _guard_untouched(buf, n, 0, name)
    _assert_equal(_host(y, (c.N, 4 * c.h, 4 * c.w, c.C))[fr], ref, name)


# ------------------------------------------------------------------------------------- space-to-depth / depth-to-space
@pytest.mark.parametrize("name", list(R.S2D))
def test_space_to_depth_and_back_copy_every_bit(name):
    """teco_space_to_depth4_f32 writes HR pixel (4 ly + dy, 4 lx + dx, c) to channel ch_off + (dy 4 + dx) C + c of LR
    pixel (ly, lx) in a pitch of out_cpitch channels, leaving every other channel alone; teco_depth_to_space4_f32 reads
    it back.  Compared as bits (-0.0, infinities and subnormals included)."""
    c = R.S2D[name]
    x = R.s2d_inputs(name)
    _assert_multi_pass(x.size, name)
    exp = np.full((c.N, c.h, c.w, c.pitch), SENTINEL, np.float32)
    exp[..., c.ch_off:c.ch_off + 16 * c.C] = x.reshape(c.N, c.h, 4, c.w, 4, c.C).transpose(0, 1, 3, 2, 4, 5).reshape(
        c.N, c.h, c.w, 16 * c.C)
    n = exp.size
    b, y = _buf(n)
    _call("teco_space_to_depth4_f32", _p(_dev(x)), _p(y), c.N, c.h, c.w, c.C, c.pitch, c.ch_off)
    _guard_untouched(b, n, 0, name)
    got = _host(y, exp.shape)
    bad = got.view(np.int32) != exp.view(np.int32)
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[0])
    b2, x2 = _buf(x.size)
    _call("teco_depth_to_space4_f32", _p(y), _p(x2), c.N, c.h, c.w, c.C, c.pitch, c.ch_off)
    _guard_untouched(b2, x.size, 0, name + " d2s")
    assert np.array_equal(_host(x2, x.shape).view(np.int32), x.view(np.int32)), name + " round trip"


# ------------------------------------------------------------------------------------------------ Gaussian LR synthesis
@pytest.mark.parametrize("name", list(R.GAUSS))
def test_gauss_down4_within_its_rounding_bound(name):
    """teco_gauss_down4_f32: 9x9 Gaussian, sigma 1.5, stride 4, VALID, against float64 of the reference's 2-D kernel in
    float32 (O.gaussian_2dkernel, as tf_data_gaussDownby4 feeds it to conv2d).

    Error model, with u = 2^-24 and S = sum_k k |x| over the window: the kernel holds the normalised 1-D factor g in fp32
    (|g32 - g| <= u g), so its 2-D weights g32[ky] g32[kx] are within (2u + u^2) k of the exact k, and the float32 kernel
    within u k: the weights alone account for 3.01 u S.  Each row sum of 9 products (with or without FMA) is within
    gamma_9 = 9u / (1 - 9u) of sum g |x|, and the outer sum of 9 weighted rows adds gamma_9 again, on rows already
    carrying their own error: together 18.01 u S.  Bound: 22 u S."""
    c = R.GAUSS[name]
    hr = R.gauss_inputs(name)
    oh, ow = (c.H - 9) // 4 + 1, (c.W - 9) // 4 + 1
    _assert_multi_pass(c.N * oh * ow * c.C, name)
    fr = _frames(c.N)
    k32 = np.float32(O.gaussian_2dkernel(9, 1.5)).astype(np.float64)
    x = hr[fr].astype(np.float64)
    ref, S = 0.0, 0.0
    for ky in range(9):
        for kx in range(9):
            p = x[:, ky:ky + 4 * (oh - 1) + 1:4, kx:kx + 4 * (ow - 1) + 1:4]
            ref, S = ref + k32[ky, kx] * p, S + k32[ky, kx] * np.abs(p)
    n = c.N * oh * ow * c.C
    b, lr = _buf(n)
    _call("teco_gauss_down4_f32", _p(_dev(hr)), _p(lr), c.N, c.H, c.W, c.C)
    _guard_untouched(b, n, 0, name)
    _assert_within(_host(lr, (c.N, oh, ow, c.C))[fr], ref, 22 * U * S, name)


# -------------------------------------------------------------------------------------------- FNet bf16 glue kernels
def _bf16_dev(x):
    t = _dev(x).to(torch.bfloat16)
    assert torch.equal(t.float().cpu(), torch.from_numpy(x)), "input not bf16-exact"
    return t


@pytest.mark.parametrize("name", list(R.MAXPOOL_BF16))
def test_maxpool2_bf16_bit_exact(name):
    """teco_maxpool2_bf16 (FNet's encoder): the max of each 2x2 window, the odd row and column dropped, at FNet's level
    sizes for 32 x 32 and 36 x 45 frames, C in {8, 64, 128, 256}, and above one grid-stride pass."""
    c = R.MAXPOOL_BF16[name]
    x = R.maxpool_bf16_inputs(name)
    oh, ow = c.H // 2, c.W // 2
    _assert_multi_pass(c.N * oh * ow * (c.C // 8), name)
    fr = _frames(c.N)
    ref = R.bf16_rne_bits(R.windows(x[fr]).max(3))            # bf16-exact: the rounding is the identity
    n = c.N * oh * ow * c.C
    b, y = _buf(n, dtype=torch.bfloat16)
    _call("teco_maxpool2_bf16", _p(_bf16_dev(x)), _p(y), c.N, c.H, c.W, c.C)
    _guard_untouched(b, n, 0, name)
    got = _host(_bits(y), (c.N, oh, ow, c.C))[fr]
    assert np.array_equal(got, ref.view(np.int16)), (name, int((got != ref.view(np.int16)).sum()))


@pytest.mark.parametrize("name", list(R.RESIZE_BF16))
def test_resize2x_bf16_rounds_to_nearest_even(name):
    """teco_resize2x_bf16 (FNet's decoder): the legacy x2 blend in fp32 (exact on these inputs), then one bf16
    round-to-nearest-even.  Each case must hit exact rounding midpoints; the odd output index at the right / bottom edge
    repeats the last pixel (min(i + 1, n - 1))."""
    c = R.RESIZE_BF16[name]
    x = R.resize_bf16_inputs(name)
    _assert_multi_pass(c.N * 4 * c.H * c.W * (c.C // 8), name)
    assert {"midpoint to even (down)", "midpoint to even (up)"} & R.keys("resize_bf16", name), name + ": no midpoint"
    fr = _frames(c.N)
    blend = R.resize2x_blend(x[fr])
    _exact(blend, 12, "bf16 blend")                          # inputs m 2^(e-7), e >= -3; quarter weights
    assert np.array_equal(blend.astype(np.float32).astype(np.float64), blend)
    ref = R.bf16_rne_bits(blend.astype(np.float32)).view(np.int16)
    n = c.N * 4 * c.H * c.W * c.C
    b, y = _buf(n, dtype=torch.bfloat16)
    _call("teco_resize2x_bf16", _p(_bf16_dev(x)), _p(y), c.N, c.H, c.W, c.C)
    _guard_untouched(b, n, 0, name)
    got = _host(_bits(y), (c.N, 2 * c.H, 2 * c.W, c.C))[fr]
    bad = got != ref
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[0])
