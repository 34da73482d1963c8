"""The rest of the training step -- batch-norm, the four fused losses, Adam, the activations, channel L2 norm, the bias
gradient and the fp32 / bf16 / uint8 conversions (csrc/eltwise.cu, bias_grad_kernel of csrc/conv_simt.cu) -- called
through the C ABI against the float64 restatements of tests/train_kernel_cases.py, at the shapes training runs and at
the edges of each kernel's launch geometry.  u = 2^-24 is the unit roundoff of fp32 throughout.

Which comparisons are bit for bit, and why:
  * Reductions on dyadic inputs (batch-norm mean and variance, its dbeta without LeakyReLU, the L2 / L1 scalars whose
    divisor is a power of two, the bias gradient): the case module's guards show that the sum of |terms| fits 24 bits
    of the grid unit, so every partial sum is an fp32 number in any order of loops, trees and atomics, and with or
    without FMA contraction.  The batch-norm inputs are built so that the mean is a grid number at any pixel count; the
    variance is then one correctly rounded fp32 division of two integers below 2^24, which float64 division followed
    by rounding to fp32 reproduces (53 >= 2 x 24 + 2 bits).
  * Elementwise gradients that are a fixed chain of IEEE fp32 multiplies and divisions with no multiply-add to contract
    (L2 da, L1 da / db, the three GAN gradients, the ReLU / LeakyReLU / sigmoid derivatives): restated in numpy float32 in
    the kernel's order and compared as bits on arbitrary inputs.  The library is built without fast-math.
  * Conversions: bf16 round-to-nearest-even restated on the bits; uint8 quantisation in numpy float32.
Where a bound is used instead, the test's docstring derives it from the operation count: rsqrtf, tanhf and expf are
2 ulp (4u relative) and logf 1 ulp in the CUDA math library, sqrtf and division are correctly rounded, and a sum of
terms whose longest chain has k additions is within k u sum|terms|.

Every output is prefilled with a sentinel and followed by a guard region that must stay untouched; pitched outputs
keep the sentinel in the channels outside the written range.  Each family has one case above a grid-stride pass or
above its block cap.  A failure names the count of wrong elements, the worst one and the block / pass it belongs to.
"""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests import train_kernel_cases as T

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
GUARD = 4096
U = T.U
TINY = 2.0 ** -149                   # one subnormal quantum


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """The large cases leave a few GB in torch's caching allocator; hand them back so that the tests after this module, and
    the training subprocesses some of them start, find the device as they would without it."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _same_class(family, name, must):
    """A key the table claims at 132 SMs is also reached on this device."""
    at132, here = T.keys(family, name), T.keys(family, name, _sms())
    for k in must:
        assert (k not in at132) or (k in here), "%s %s: '%s' is not reached with %d SMs" % (family, name, k, _sms())


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _buf(n, dtype=torch.float32, fill=SENTINEL):
    """n elements (filled with `fill`) followed by a guard region holding the sentinel."""
    b = torch.full((n + GUARD,), SENTINEL, dtype=dtype, device="cuda")
    b[:n] = fill
    return b, b[:n]


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _guard_untouched(b, n, what):
    s = _bits(torch.full((1,), SENTINEL, dtype=b.dtype, device=b.device))
    rest = _bits(b[n:])
    assert (rest == s).all(), "%s: wrote %d elements past its output" % (what, int((rest != s).sum()))


def _host(t, shape=None):
    a = t.cpu().numpy()
    return a if shape is None else a.reshape(shape)


def _elt_where(n, per_block=T.TPB):
    blocks, _ = T.elt_launch(n, _sms(), per_block)
    return lambda i: "grid-stride pass %d, block %d" % (i // (blocks * T.TPB), i % (blocks * T.TPB) // T.TPB)


def _report(bad, err, what, where, detail):
    flat = np.flatnonzero(bad.ravel())
    w = int(flat[np.argmax(err.ravel()[flat])])
    idx = tuple(int(v) for v in np.unravel_index(w, bad.shape))
    raise AssertionError("%s: %d / %d elements wrong, worst at %s%s: %s" % (
        what, flat.size, bad.size, idx, " (%s)" % where(w) if where else "", detail(idx)))


def _assert_equal(got, exp, what, where=None):
    """Values equal (exp is float64 holding fp32 numbers; +0 and -0 compare equal)."""
    got, exp = np.asarray(got), np.asarray(exp, np.float64)
    bad = ~(got.astype(np.float64) == exp)
    if bad.any():
        _report(bad, np.abs(got.astype(np.float64) - exp), what, where, lambda i: "got %r, expected %r" % (float(got[i]), float(exp[i])))


def _assert_bits(got, exp, what, where=None):
    """Same bit patterns (exp is the numpy float32 restatement)."""
    got, exp = np.asarray(got), np.asarray(exp, got.dtype)
    v = {1: np.uint8, 2: np.int16, 4: np.int32}[got.dtype.itemsize]
    bad = got.view(v) != exp.view(v)
    if bad.any():
        _report(bad, np.abs(got.astype(np.float64) - exp.astype(np.float64)) + 1, what, where,
                lambda i: "got %r, expected %r" % (got[i].item(), exp[i].item()))


def _assert_within(got, exp, tol, what, where=None):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    tol = np.broadcast_to(tol, exp.shape)
    err = np.abs(got - exp)
    bad = ~(err <= tol)
    if bad.any():
        _report(bad, np.where(bad, err / np.maximum(tol, 1e-300), 0), what, where,
                lambda i: "got %r, expected %r, error %.3e, bound %.3e" % (float(got[i]), float(exp[i]), err[i], tol[i]))


def _call(name, *args):
    from tecogan_b200._ffi import call, stream_ptr
    call(name, *args, stream_ptr())
    torch.cuda.synchronize()


def _p(t):
    """Device pointer of a tensor the caller keeps alive until the call has run."""
    from tecogan_b200._ffi import ptr
    return ptr(t)


def _unchanged(t, a, what):
    assert np.array_equal(_host(_bits(t)).ravel(), np.ascontiguousarray(a).view(_host(_bits(t)).dtype).ravel()), what + ": input modified"


# ------------------------------------------------------------------------------------------------------- batch norm
@pytest.mark.parametrize("name", list(T.BN))
def test_batchnorm_forward_and_backward(name):
    """teco_bn_train_f32 / teco_bn_train_bwd_f32 at C in {1, 3, 48, 64, 100, 128, 256}, one block, several, a short last
    block, the block cap, and the discriminator's four layers.

    Statistics: exact on the dyadic cases (module docstring), mean 100 included, where a one-pass variance could not be.
    On continuous inputs, with k the additions of the longest chain (T.split_steps): |mean - ref| <= k u sum|x| / npix,
    and against float64 of sum (x - mean_kernel)^2 / npix the variance is within (k + 4) u of it (subtraction, square and
    division add 4 roundings to a sum of non-negative terms).
    y is judged from the kernel's own stats: x - mean (u), var + eps (u / 2 after the root), rsqrtf (4u), the product or
    FMA (u), together under 8 u |xhat|; the add of beta and the 0.2 of LeakyReLU round the result, 2 u |xhat + beta|.
    Where x == mean and beta == 0, y must be +0 so that the backward mask y < 0 agrees with the forward's v >= 0.
    dbeta = sum g is exact without LeakyReLU; with it g = 0.2f dy is rounded once: (k + 1) u sum|g|.
    dx = rstd (g - m1 - xhat m2), m1 = sum g / npix, m2 = sum g xhat / npix: the sums are within (k + 2) u sum|g| and
    (k + 10) u sum|g xhat| (each g xhat term carries xhat's 8 u), and the remaining roundings (1 / npix, three products,
    two subtractions, rstd's 4 u) stay under 16 u (|g| + |m1| + |xhat m2|).
    stats is 4C floats (mean, variance, two scratch rows) and dbeta 2C: nothing past them is written."""
    c, sms = T.BN[name], _sms()
    _same_class("bn", name, ("bn: blocks capped", "bn: multi block", "bn: last block short", "bn: apply >1 grid-stride pass"))
    x, beta, dy = T.bn_inputs(name)
    n, C = c.npix * c.C, c.C
    blocks, ppb, _ = T.bn_launch(c.npix, sms)
    k = T.split_steps(blocks, ppb, C)
    where = lambda i: "pixel %d, statistics block %d of %d" % (i // C, i // C // ppb, blocks)
    d_x, d_beta, d_dy = _dev(x), _dev(beta), _dev(dy)
    by, y = _buf(n)
    bs, stats = _buf(4 * C)
    _call("teco_bn_train_f32", _p(d_x), _p(d_beta), _p(y), _p(stats), c.npix, C, 1e-3, c.lrelu)
    _guard_untouched(by, n, name + " y"), _guard_untouched(bs, 4 * C, name + " stats")
    _unchanged(d_x, x, name)
    st = _host(stats).astype(np.float64)
    mean_k, var_k = st[:C], st[C:2 * C]
    x64 = x.astype(np.float64)
    if c.kind != "cont":
        T.bn_guard(name)
        mean_r, var_r = T.bn_stats_ref(x)
        _assert_equal(st[:C], mean_r, name + " mean")
        _assert_equal(st[C:2 * C], np.float32(var_r), name + " variance")
    else:
        _assert_within(mean_k, x64.mean(0), k * U * np.abs(x64).sum(0) / c.npix, name + " mean")
        var_r = ((x64 - mean_k) ** 2).mean(0)
        _assert_within(var_k, var_r, (k + 4) * U * var_r, name + " variance")
    y_r, xhat = T.bn_apply_ref(x, beta, mean_k, var_k, c.lrelu)
    got_y = _host(y, x.shape)
    _assert_within(got_y, y_r, U * (8 * np.abs(xhat) + 2 * np.abs(xhat + beta)), name + " y", where)
    if c.kind != "cont":
        zero = (x64 == mean_k) & (beta == 0)
        if "bn: y==0" in T.keys("bn", name):
            assert zero.any()
        assert (got_y[zero].view(np.int32) == 0).all(), name + ": y is not +0 where x == mean and beta == 0"

    bd, dx = _buf(n)
    bb, dbeta = _buf(2 * C)
    _call("teco_bn_train_bwd_f32", _p(d_x), _p(y), _p(d_dy), _p(stats), _p(dx), _p(dbeta), c.npix, C, 1e-3, c.lrelu)
    _guard_untouched(bd, n, name + " dx"), _guard_untouched(bb, 2 * C, name + " dbeta")
    dx_r, dbeta_r, sg, sgx, g, xhat = T.bn_bwd_ref(x, got_y, dy, mean_k, var_k, c.lrelu)
    got_db = _host(dbeta)[:C]
    if c.kind != "cont" and not c.lrelu:
        _assert_equal(got_db, dbeta_r, name + " dbeta")
    else:
        _assert_within(got_db, dbeta_r, (k + 1) * U * sg, name + " dbeta")
    rstd = 1.0 / np.sqrt(var_k + T.BN_EPS)
    m1, m2 = g.sum(0) / c.npix, (g * xhat).sum(0) / c.npix
    tol = rstd * (16 * U * (np.abs(g) + np.abs(m1) + np.abs(xhat * m2))
                  + (k + 2) * U * sg / c.npix + np.abs(xhat) * (k + 10) * U * sgx / c.npix)
    _assert_within(_host(dx, x.shape), dx_r, tol, name + " dx", where)


def test_batchnorm_rejects_unsupported_channel_counts():
    t = torch.zeros(4 * 257, device="cuda")
    for C in (0, 257):
        with pytest.raises(ValueError):
            _call("teco_bn_train_f32", _p(t), _p(t), _p(t), _p(t), 1, C, 1e-3, 0)
        with pytest.raises(ValueError):
            _call("teco_bn_train_bwd_f32", _p(t), _p(t), _p(t), _p(t), _p(t), _p(t), 1, C, 1e-3, 0)


# --------------------------------------------------------------------------------------------------- L2 / L1 losses
def _scalar(out_buf, out, what):
    _guard_untouched(out_buf, 1, what)
    return float(_host(out)[0])


@pytest.mark.parametrize("name", list(T.L2))
def test_loss_l2(name):
    """teco_loss_l2_f32: the scalar is exact on the dyadic cases (npix a power of two, the 64 x 128 x 128 x 3 content-loss
    size with capped blocks included); on continuous inputs at npix = 1001 within k u sum d^2 / npix, k = T.reduce_steps
    + 3 (subtraction, square, and the accumulate).  da = 2 d inv_npix gscale equals the numpy float32 chain bit for
    bit.  da == NULL leaves the value unchanged."""
    c = T.L2[name]
    _same_class("l2", name, ("eltwise: >1 grid-stride pass", "l2: blocks capped"))
    a, b = T.loss_inputs(T.L2, name)
    n = a.size
    val, _, s = T.l2_ref(a, b, c.gscale)
    d_a, d_b = _dev(a), _dev(b)
    for with_da in (True, False):
        what = name + (" with da" if with_da else " value only")
        bo, out = _buf(1)
        bd, da = _buf(n) if with_da else (None, None)
        _call("teco_loss_l2_f32", _p(d_a), _p(d_b), _p(out), _p(da), c.npix, c.C, c.gscale)
        got = _scalar(bo, out, what)
        if T.loss_scalar_exact(c):
            T.loss_guard(T.L2, name)
            assert got == val, "%s: got %r, expected %r" % (what, got, val)
        else:
            assert abs(got - val) <= (T.reduce_steps(n, _sms()) + 3) * U * s / c.npix, (what, got, val)
        if with_da:
            _guard_untouched(bd, n, what)
            _assert_bits(_host(da, a.shape), T.l2_da_f32(a, b, c.gscale), what + " da", _elt_where(n, 1024))
    _unchanged(d_a, a, name), _unchanged(d_b, b, name)


@pytest.mark.parametrize("name", list(T.L1))
def test_loss_l1(name):
    """teco_loss_l1_f32 over all elements and per pixel: exact scalar where the divisor is a power of two, else within
    k u sum|d| / den with k = T.reduce_steps + 2.  da = sign(d) inv_den gscale and db = -da equal the numpy float32 chain bit
    for bit, +0 / -0 at d = +-0 included; da and db may each be NULL."""
    c = T.L1[name]
    _same_class("l1", name, ("eltwise: >1 grid-stride pass",))
    a, b = T.loss_inputs(T.L1, name)
    n = a.size
    val, _, s = T.l1_ref(a, b, c.gscale, c.per_pixel)
    g32 = T.l1_da_f32(a, b, c.gscale, c.per_pixel)
    d_a, d_b = _dev(a), _dev(b)
    for with_da, with_db in ((True, True), (True, False), (False, True), (False, False)):
        what = "%s%s%s" % (name, " da" if with_da else "", " db" if with_db else "")
        bo, out = _buf(1)
        ba, da = _buf(n) if with_da else (None, None)
        bb, db = _buf(n) if with_db else (None, None)
        _call("teco_loss_l1_f32", _p(d_a), _p(d_b), _p(out), _p(da), _p(db), c.npix, c.C, c.per_pixel, c.gscale)
        got = _scalar(bo, out, what)
        if T.loss_scalar_exact(c):
            T.loss_guard(T.L1, name)
            assert got == val, "%s: got %r, expected %r" % (what, got, val)
        else:
            assert abs(got - val) <= (T.reduce_steps(n, _sms()) + 2) * U * s / T.loss_den(c), (what, got, val)
        if with_da:
            _guard_untouched(ba, n, what)
            _assert_bits(_host(da, a.shape), g32, what + ": da", _elt_where(n, 1024))
        if with_db:
            _guard_untouched(bb, n, what)
            _assert_bits(_host(db, a.shape), -g32, what + ": db", _elt_where(n, 1024))


# ---------------------------------------------------------------------------------------- cosine loss / channel L2 norm
@pytest.mark.parametrize("name", list(T.COS))
def test_loss_cosine(name):
    """teco_loss_cosine_f32 at C in {3, 48, 64, 128, 256, 512}, with pixels whose f, g or both are all zero (the 1e-12
    under the root then decides value and gradient), more pixels than warps, df NULL and gscale != 1.

    With c = ceil(C / 32): a squared norm or dot product is a lane's c serial products and a 5-level tree, (c + 5) u of
    sum|terms|; + eps and the root leave (c + 5) / 2 + 1.5 on a norm; nf ng and the division give cos an absolute error
    under (2c + 14) u A, A = sum|f g| / (nf ng) <= 1.  The value sums cos over a warp's pixels, the block tree, one
    atomic per block, scales by 1 / npix and adds 1 (result <= 2): (2c + 26 + pixels per warp + blocks) u mean(A) + 2u.
    The gradient k1 g + k2 f has k1 within (c + 12) u and k2 within (2c + 14 + c + 12) u of A gscale / (npix nf^2),
    plus two roundings of the multiply-add: (3c + 28) u (|k1 g| + A gscale |f| / (npix nf^2)) per element.
    Called twice on the same `out`, the second value obeys the same bound: the kernel clears it first."""
    c, sms = T.COS[name], _sms()
    _same_class("cos", name, ("cos: >1 pixel per warp",))
    f, g = T.cos_inputs(T.COS, name)
    val, df_r, A, mag = T.cos_ref(f, g, c.gscale)
    cc = -(-c.C // 32)
    warps, ppw = T.warp_launch(c.npix, sms)
    tol = (2 * cc + 26 + ppw + warps // 8) * U * A + 2 * U
    d_f, d_g = _dev(f), _dev(g)
    bo, out = _buf(1)
    bd, df = (None, None) if c.df_null else _buf(f.size)
    for turn in ("first", "second"):
        _call("teco_loss_cosine_f32", _p(d_f), _p(d_g), _p(out), _p(df), c.npix, c.C, c.gscale)
        got = _scalar(bo, out, name)
        assert abs(got - val) <= tol, "%s %s call: got %r, expected %r, bound %.3e" % (name, turn, got, val, tol)
    if not c.df_null:
        _guard_untouched(bd, f.size, name + " df")
        where = lambda i: "pixel %d, grid-stride pass %d of its warp" % (i // c.C, i // c.C // warps)
        _assert_within(_host(df, f.shape), df_r, (3 * cc + 28) * U * mag, name + " df", where)
    _unchanged(d_f, f, name), _unchanged(d_g, g, name)


@pytest.mark.parametrize("name", list(T.L2NORM))
def test_l2norm_channels(name):
    """teco_l2norm_channels_f32: y = f (1 / sqrt(sum f^2 + 1e-12)).  With c = ceil(C / 32) the sum is within (c + 5) u, the
    root halves that and adds eps' and its own rounding, the reciprocal and the product one each: (c / 2 + 6) u |y|.  An
    all-zero pixel gives exactly 0, not NaN; the input is left alone."""
    c = T.L2NORM[name]
    _same_class("l2norm", name, ("l2norm: >1 pixel per warp",))
    f, _ = T.cos_inputs(T.L2NORM, name)
    ref = T.l2norm_ref(f)
    d_f = _dev(f)
    b, y = _buf(f.size)
    _call("teco_l2norm_channels_f32", _p(d_f), _p(y), c.npix, c.C)
    _guard_untouched(b, f.size, name)
    got = _host(y, f.shape)
    warps = T.warp_launch(c.npix, _sms())[0]
    where = lambda i: "pixel %d, grid-stride pass %d of its warp" % (i // c.C, i // c.C // warps)
    _assert_within(got, ref, (-(-c.C // 32) / 2 + 6) * U * np.abs(ref), name, where)
    assert (got[(f == 0).all(1)].view(np.int32) == 0).all(), name + ": zero pixel"
    _unchanged(d_f, f, name)


# --------------------------------------------------------------------------------------------------------- GAN loss
@pytest.mark.parametrize("name", list(T.GAN))
def test_loss_gan(name):
    """teco_loss_gan_f32 with eps = 1e-12 on inputs that include 0, 1 and their 2^-24 neighbours, on the discriminator's
    24 x 8 x 8 x 1 output, at n = 1 and above one pass, with each gradient pointer NULL.

    The five means are compared with float64 of the fp32 arguments f + eps, (1 - f) + eps, r + eps: logf is 1 ulp (2u
    relative), the sum is within k u sum|terms| with k = T.reduce_steps, and out[1] adds two logarithms per element: (k + 4)
    u mean|terms| for every scalar.  The three gradients equal the numpy float32 chain bit for bit (saturated inputs
    give finite values of order 1e12 / n)."""
    c = T.GAN[name]
    _same_class("gan", name, ("eltwise: >1 grid-stride pass",))
    f, r = T.gan_inputs(name)
    val, mag = T.gan_ref(f, r)
    exp = dict(zip(("adv", "dis_f", "dis_r"), T.gan_grads_f32(f, r, c.s_adv, c.s_dis)))
    bo, out = _buf(5)
    bufs = {k: (None, None) if k in c.null else _buf(c.n) for k in exp}
    d_f, d_r = _dev(f), _dev(r)
    _call("teco_loss_gan_f32", _p(d_f), _p(d_r), _p(out), _p(bufs["adv"][1]), _p(bufs["dis_f"][1]),
          _p(bufs["dis_r"][1]), c.n, 1e-12, c.s_adv, c.s_dis)
    _guard_untouched(bo, 5, name)
    _assert_within(_host(out), val, (T.reduce_steps(c.n, _sms()) + 4) * U * mag, name + " scalars")
    for k, (b, t) in bufs.items():
        if t is not None:
            _guard_untouched(b, c.n, name + " g_" + k)
            assert np.isfinite(exp[k]).all()
            _assert_bits(_host(t), exp[k], name + " g_" + k, _elt_where(c.n, 1024))


# ------------------------------------------------------------------------------------------------------------- Adam
@pytest.mark.parametrize("name", list(T.ADAM))
def test_adam_one_step(name):
    """teco_adam_f32, one step in place, n in {1, 255, 257, 1000, above one grid-stride pass, the generator's flat size},
    gscale in {1, 1/4, 1/3}, |g| from 1e-8 to 1 so that sqrt(v') runs from far below eps to far above it.

    Against float64 on the fp32 inputs and constants (1.f - b1 and 1.f - b2 are exact subtractions): m' = t0 + t1 with
    t0 = b1 m, t1 = (1 - b1) (g s): g s, each product and the sum round once, |m' - ref| <= u (2 |t0| + 3 |t1|) with or
    without FMA.  v' likewise with one more product: u (2 |t0| + 5 |t1|).  p' is judged from the kernel's own m', v':
    lr_t m', sqrtf, + eps and the division round once each, and so does the subtraction: u (|p| + 6 |step|).
    Elements with g = m = v = 0 keep p's bits and stay 0 (0 / eps, no NaN); g is not modified."""
    c = T.ADAM[name]
    _same_class("adam", name, ("eltwise: >1 grid-stride pass",))
    p, m, v, g = T.adam_inputs(name)
    bufs = [_buf(c.n) for _ in range(3)]
    for (_, t), a in zip(bufs, (p, m, v)):
        t.copy_(_dev(a))
    d_g = _dev(g)
    _call("teco_adam_f32", _p(bufs[0][1]), _p(bufs[1][1]), _p(bufs[2][1]), _p(d_g), c.n, T.ADAM_LR_T, T.ADAM_B1, T.ADAM_B2,
          T.ADAM_EPS, c.gscale)
    for (b, _), w in zip(bufs, "pmv"):
        _guard_untouched(b, c.n, name + " " + w)
    _unchanged(d_g, g, name)
    p1, m1, v1 = (_host(t) for _, t in bufs)
    m_r, v_r, mt, vt, step = T.adam_ref(p, m, v, g, c.gscale)
    where = _elt_where(c.n)
    _assert_within(m1, m_r, U * (2 * np.abs(mt[0]) + 3 * np.abs(mt[1])), name + " m", where)
    _assert_within(v1, v_r, U * (2 * np.abs(vt[0]) + 5 * np.abs(vt[1])), name + " v", where)
    s = step(m1, v1)
    _assert_within(p1, p.astype(np.float64) - s, U * (np.abs(p) + 6 * np.abs(s)), name + " p", where)
    still = (g == 0) & (m == 0) & (v == 0)
    assert np.array_equal(p1[still].view(np.int32), p[still].view(np.int32)) and not m1[still].any() and not v1[still].any()
    assert np.isfinite(p1).all() and np.isfinite(m1).all() and np.isfinite(v1).all()


def test_adam_three_steps_match_tf_adam_with_a_gradient_scale():
    """Three chained steps with gscale = 1/4 on gradients four times as large against O.TFAdam (1e-7, as the unscaled test of
    tests/test_gpu_kernels.py)."""
    r = T.rng("adam chain")
    p, g = r.uniform(-1, 1, 1000).astype(np.float32), r.uniform(-1, 1, 1000).astype(np.float32)
    P = {"a": torch.from_numpy(p.copy())}
    opt = O.TFAdam(["a"], P, lr=5e-5)
    dp, m, v = _dev(p), torch.zeros(1000, device="cuda"), torch.zeros(1000, device="cuda")
    for t in range(1, 4):
        opt.apply(P, {"a": torch.from_numpy(g * t)})
        lr_t = 5e-5 * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
        d_g = _dev(g * (4 * t))
        _call("teco_adam_f32", _p(dp), _p(m), _p(v), _p(d_g), 1000, lr_t, 0.9, 0.999, 1e-8, 0.25)
    assert float((dp.cpu() - P["a"]).abs().max()) <= 1e-7


# ------------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("size", list(T.ACT_SIZES))
def test_affine_act_forward(size):
    """teco_affine_act_f32 with a = 1, b = 0 (the pre-activation is then x itself, fused or not) on a table holding +-0,
    +-subnormal, +-tiny, inputs that saturate tanh and +-100 for the sigmoid.  none / ReLU are exact, LeakyReLU is one
    rounding of 0.2f x (exact against float64 of that product rounded to fp32).  tanh24: tanhf is 2 ulp and the product with
    24 rounds once, 5 u |y| (+ one subnormal quantum); saturated inputs give exactly +-24.  sigmoid 1 / (1 + expf(-x)): expf's
    4u on e, the sum's u and the division's u give y^2 (4u e + u (1 + e)) + u y <= 6 u y; below x = -88.7 expf overflows and
    the result is 0 where float64 has a number under 2^-126, which is the floor of the bound."""
    n = T.ACT_SIZES[size]
    _same_class("act", size, ("eltwise: >1 grid-stride pass",))
    x = T.act_x(size)
    d_x = _dev(x)
    for act, an in T.ACT_NAMES.items():
        what = "%s %s" % (size, an)
        b, y = _buf(n)
        _call("teco_affine_act_f32", _p(d_x), _p(y), n, 1.0, 0.0, act)
        _guard_untouched(b, n, what)
        got, ref = _host(y), T.act_ref(x, act)
        if act in (T.ACT_NONE, T.ACT_RELU):
            _assert_equal(got, ref, what, _elt_where(n))
        elif act == T.ACT_LRELU02:
            _assert_equal(got, ref.astype(np.float32), what, _elt_where(n))
        elif act == T.ACT_TANH24:
            _assert_within(got, ref, 5 * U * np.abs(ref) + TINY, what, _elt_where(n))
            assert (got[np.abs(x) >= 20] == 24 * np.sign(x[np.abs(x) >= 20])).all(), what + ": saturation"
        else:
            _assert_within(got, ref, 6 * U * ref + 2.0 ** -126, what, _elt_where(n))
            assert (got[x == 100] == 1).all() and (got[x == -100] == 0).all(), what + ": saturation"
        # the in-place call kernels._AffineAct.backward makes
        z = d_x.clone()
        _call("teco_affine_act_f32", _p(z), _p(z), n, 1.0, 0.0, act)
        assert torch.equal(_bits(z), _bits(y)), what + ": in place differs"


def test_affine_act_scale_and_shift():
    """y = a x + b: preprocess (2, -1) and deprocess (0.5, 0.5) on 2^-7-grid inputs are exact fused or not.  At a = 1/3,
    b = 0.1 the unfused form rounds twice, u (|a x| + |a x + b|), and the fused one less; LeakyReLU rounds once more and may take
    the other branch within that error of 0: 2 u (|a x| + |a x + b|)."""
    x = T.uniform(T.rng("affine"), (1000,), 7)
    d_x = _dev(x)
    for a, b_ in ((2.0, -1.0), (0.5, 0.5)):
        b, y = _buf(x.size)
        _call("teco_affine_act_f32", _p(d_x), _p(y), x.size, a, b_, T.ACT_NONE)
        _guard_untouched(b, x.size, "affine")
        _assert_equal(_host(y), a * x.astype(np.float64) + b_, "affine %g %g" % (a, b_))
    a, b_ = float(np.float32(1.0 / 3.0)), float(np.float32(0.1))
    x = T.rng("affine cont").uniform(-2, 2, 1000).astype(np.float32)
    b, y = _buf(x.size)
    d_x = _dev(x)
    _call("teco_affine_act_f32", _p(d_x), _p(y), x.size, a, b_, T.ACT_LRELU02)
    pre = a * x.astype(np.float64) + b_
    ref = np.where(pre >= 0, pre, T.F02 * pre)
    _assert_within(_host(y), ref, 2 * U * (np.abs(a * x) + np.abs(pre)), "affine 1/3 0.1 lrelu")


@pytest.mark.parametrize("size", list(T.ACT_SIZES))
def test_act_bwd_on_saved_outputs(size):
    """teco_act_bwd_f32 on saved outputs that hold +0 and -0 (ReLU passes the gradient for y > 0, LeakyReLU for y >= 0),
    +-subnormal, tanh at |y| = 24 and sigmoid at 0 and 1.  none / ReLU / LeakyReLU / sigmoid equal the numpy float32 chain
    bit for bit.  tanh24 is g 24 (1 - t t), t = y (1 / 24): t rounds once, 1 - t t is fused (one rounding) or not (two),
    the two outer products round once each: 4 u |24 g| (t^2 + |1 - t^2|)."""
    n = T.ACT_SIZES[size]
    for act, an in T.ACT_NAMES.items():
        what = "%s %s bwd" % (size, an)
        y, dy = T.act_bwd_inputs(size, act)
        b, dx = _buf(n)
        d_y, d_dy = _dev(y), _dev(dy)
        _call("teco_act_bwd_f32", _p(d_y), _p(d_dy), _p(dx), n, act)
        _guard_untouched(b, n, what)
        if act != T.ACT_TANH24:
            _assert_bits(_host(dx), T.act_bwd_f32(y, dy, act), what, _elt_where(n))
        else:
            t = y.astype(np.float64) * T.INV24
            _assert_within(_host(dx), T.act_bwd_ref(y, dy, act), 4 * U * np.abs(24.0 * dy) * (t * t + np.abs(1 - t * t)) + TINY,
                           what, _elt_where(n))


# ---------------------------------------------------------------------------------------------------- bias gradient
@pytest.mark.parametrize("name", list(T.BIAS))
def test_bias_grad(name):
    """teco_bias_grad_f32 on dyadic dy: exact at C in {1, 2, 3, 4, 64, 100, 256}, npix in {1, 7, 8 ppar +- 1, above the
    block cap}, with cpitch > C (the pad channels hold 2^20 and must not be summed), overwriting a db that holds 1e30 and
    accumulating onto one that holds dyadic values."""
    c = T.BIAS[name]
    _same_class("bias", name, ("bias: capped", "bias: multi block", "bias: last block short"))
    T.bias_guard(name)
    dy, db0 = T.bias_inputs(name)
    ref, _ = T.bias_ref(dy, db0, c.C, c.accumulate)
    d_dy = _dev(dy)
    b, db = _buf(c.C)
    db.copy_(_dev(db0))
    _call("teco_bias_grad_f32", _p(d_dy), _p(db), c.npix, c.C, c.cpitch, c.accumulate)
    _guard_untouched(b, c.C, name)
    _assert_equal(_host(db), ref, name + " %s" % (T.bias_launch(c.npix, c.C, _sms()),))
    _unchanged(d_dy, dy, name)


def test_bias_grad_rejects_bad_channel_arguments():
    t = torch.zeros(1024, device="cuda")
    for C, cpitch in ((257, 257), (0, 4), (4, 3)):
        with pytest.raises(ValueError):
            _call("teco_bias_grad_f32", _p(t), _p(t), 2, C, cpitch, 0)


@pytest.mark.parametrize("cout,accumulate", [(3, 0), (64, 0), (100, 1)])
def test_wgrad_bias_gradient_on_a_strided_output_map(cout, accumulate):
    """teco_conv2d_wgrad_f32's db when the output map is one phase of a transposed convolution (out_sy = out_sx = 2):
    bias_grad_kernel's strided branch sums dy[:, a::2, b::2] only.  Exact on dyadic dy; the other phases hold 2^20."""
    from tecogan_b200 import kernels as K
    r = T.rng("wgrad bias %d" % cout)
    N, H, W, cin = 3, 5, 7, 4
    x = _dev(T.uniform(r, (N, H, W, cin), 4))
    db0 = (r.randint(-40, 41, cout) / 4.0).astype(np.float32) if accumulate else np.full(cout, 1e30, np.float32)
    for a, b_ in ((0, 0), (1, 0), (0, 1), (1, 1)):
        dy = np.full((N, 2 * H, 2 * W, cout), T.BIAS_PAD, np.float32)
        dy[:, a::2, b_::2] = T.uniform(r, (N, H, W, cout), 2)
        T.exact(np.abs(dy[:, a::2, b_::2]).sum((0, 1, 2)) + np.abs(db0) * accumulate, 2, "sum |dy|")
        ref = dy[:, a::2, b_::2].astype(np.float64).sum((0, 1, 2)) + (db0 if accumulate else 0)
        dw = torch.zeros(1, 1, cin, cout, device="cuda")
        b, db = _buf(cout)
        db.copy_(_dev(db0))
        K.conv2d_wgrad_raw(x, _dev(dy), dw, db, stride=1, pad_t=0, pad_l=0, OH=H, OW=W, out_map=(2, a, 2, b_),
                           accumulate=bool(accumulate))
        torch.cuda.synchronize()
        _guard_untouched(b, cout, "wgrad db")
        _assert_equal(_host(db), ref, "wgrad db phase (%d, %d)" % (a, b_))


# ------------------------------------------------------------------------------------------------------ conversions
@pytest.mark.parametrize("name", list(T.ROWPAD))
def test_f32_to_bf16_rowpad_rounds_to_nearest_even_and_zero_fills(name):
    """teco_f32_to_bf16_rowpad: channels below C are round-to-nearest-even of the source (a quarter of the inputs are exact
    midpoints, both parities), channels from C to dst_cpitch are +0, source channels beyond C are not read into the row."""
    c = T.ROWPAD[name]
    _same_class("rowpad", name, ("rows: >1 grid-stride pass",))
    src = T.rows_inputs(T.ROWPAD, name)
    exp = np.zeros((c.npix, c.dst_cpitch), np.uint16)
    exp[:, :c.C] = T.bf16_rne_bits(src[:, :c.C])
    n = exp.size
    b, dst = _buf(n, dtype=torch.bfloat16)
    d_src = _dev(src)
    _call("teco_f32_to_bf16_rowpad", _p(d_src), _p(dst), c.npix, c.C, c.src_cpitch, c.dst_cpitch)
    _guard_untouched(b, n, name)
    _assert_bits(_host(_bits(dst), exp.shape), exp.view(np.int16), name, _elt_where(n))


@pytest.mark.parametrize("name", list(T.FROM_BF16))
def test_bf16_to_f32_with_and_without_add(name):
    """teco_bf16_to_f32_add with add (one fp32 addition, restated in numpy float32) and with add == NULL, and
    teco_bf16_to_f32: channels below C of each row are written, the rest of a pitched row keeps the sentinel."""
    c = T.FROM_BF16[name]
    _same_class("from_bf16", name, ("rows: >1 grid-stride pass",))
    src, add = T.rows_inputs(T.FROM_BF16, name)
    d_src = _dev(src).to(torch.bfloat16)
    assert torch.equal(_bits(d_src.float().cpu()), _bits(torch.from_numpy(src)))
    n = c.npix * c.dst_cpitch
    for fn, with_add in (("teco_bf16_to_f32_add", True), ("teco_bf16_to_f32_add", False), ("teco_bf16_to_f32", False)):
        what = "%s %s%s" % (name, fn, " add" if with_add else "")
        exp = np.full((c.npix, c.dst_cpitch), SENTINEL, np.float32)
        with np.errstate(over="ignore"):
            exp[:, :c.C] = src[:, :c.C] + add[:, :c.C] if with_add else src[:, :c.C]
        b, dst = _buf(n)
        d_add = _dev(add) if with_add else None
        args = (_p(d_src), _p(d_add), _p(dst)) if fn.endswith("add") else (_p(d_src), _p(dst))
        _call(fn, *args, c.npix, c.C, c.src_cpitch, c.dst_cpitch)
        _guard_untouched(b, n, what)
        _assert_bits(_host(dst, exp.shape), exp, what)


def test_f32_to_bf16_pad_above_one_pass_and_to_u8():
    """teco_f32_to_bf16_pad writes channels [c_off, c_off + C) of each pitched row and nothing else, here above one
    grid-stride pass with scale 1, shift 0 (x 1 + 0 is x fused or not) and, on 2^-7-grid inputs, with the deprocess pair
    0.5, 0.5 (exact before the rounding).  teco_to_u8 is clip(x 255, 0, 255) truncated: k / 255 and both fp32 neighbours for
    every k, negatives, -0 and values above 1, against numpy float32."""
    r = T.rng("pad")
    npix, C, sp, dp, off = (16 * 132 * 256) // 48 + 11, 48, 51, 64, 8
    assert T.elt_launch(npix * C, _sms())[1] > 1
    for scale, shift, src in ((1.0, 0.0, T.bf16_midpoint_values(r, (npix, sp))), (0.5, 0.5, T.uniform(r, (npix, sp), 7))):
        exp = np.full((npix, dp), SENTINEL, np.float32)
        exp = T.bf16_rne_bits(exp)
        exp[:, off:off + C] = T.bf16_rne_bits((src[:, :C].astype(np.float64) * scale + shift).astype(np.float32))
        b, dst = _buf(npix * dp, dtype=torch.bfloat16)
        d_src = _dev(src)
        _call("teco_f32_to_bf16_pad", _p(d_src), _p(dst), npix, C, sp, dp, off, scale, shift)
        _guard_untouched(b, npix * dp, "f32_to_bf16_pad")
        _assert_bits(_host(_bits(dst), exp.shape), exp.view(np.int16), "f32_to_bf16_pad scale %g" % scale)
    x = T.u8_inputs()
    b = torch.full((x.size + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    q = b[:x.size]
    d_x = _dev(x)
    _call("teco_to_u8", _p(d_x), _p(q), x.size)
    assert (b[x.size:] == 0xA5).all(), "to_u8 wrote past its output"
    _assert_bits(_host(q), T.u8_ref(x), "to_u8")


# --------------------------------------------------------------------------------------------------- autograd wrappers
def test_loss_wrappers_route_gradients_as_documented():
    """kernels._LossL2 / _LossL1 give the second argument the negated gradient and None to an input that needs none;
    _LossCos gives its target no gradient; _LossGAN.backward combines out[0] and out[1] into d_fake, out[1] and out[2] into
    d_real, and out[3] / out[4] (mean D_real / D_fake) are report-only: they contribute no gradient."""
    from tecogan_b200 import kernels as K
    a, b = T.loss_inputs(T.L2, "4x16x16_c3_gs")
    for fn in (K.loss_l2, lambda u, v: K.loss_l1(u, v, False), lambda u, v: K.loss_l1(u, v, True)):
        ta, tb = _dev(a).requires_grad_(True), _dev(b).requires_grad_(True)
        ga, gb = torch.autograd.grad(fn(ta, tb) * 1.5, [ta, tb])
        assert torch.equal(_bits(gb), _bits(-ga)) and bool(ga.abs().sum() > 0)
        tb2 = _dev(b).requires_grad_(True)
        loss = fn(_dev(a), tb2)
        assert torch.equal(_bits(torch.autograd.grad(loss * 1.5, tb2)[0]), _bits(gb))
        assert not fn(_dev(a), _dev(b)).requires_grad
    f, g = T.cos_inputs(T.COS, "5px_c48_gs")
    tf, tg = _dev(f).requires_grad_(True), _dev(g).requires_grad_(True)
    loss = K.loss_cosine(tf, tg)
    gf, gg = torch.autograd.grad(loss, [tf, tg], allow_unused=True)
    assert gg is None and bool(gf.abs().sum() > 0)
    fk, rl = T.gan_inputs("disc_24x8x8x1")
    e_adv, e_f, e_r = (torch.from_numpy(t).cuda() for t in T.gan_grads_f32(fk, rl, 1.0, 1.0))
    for w in ((1.0, 0.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0, 0.0), (0.0, 0.0, 1.0, 0.0, 0.0), (0.25, 0.5, 2.0, 0.0, 0.0),
              (0.25, 0.5, 2.0, 3.0, 5.0)):
        tf, tr = _dev(fk).requires_grad_(True), _dev(rl).requires_grad_(True)
        out = K.loss_gan(tf, tr, 1e-12)
        gfk, grl = torch.autograd.grad((out * torch.tensor(w, device="cuda")).sum(), [tf, tr])
        assert torch.equal(gfk, e_adv * w[0] + e_f * w[1]), w
        assert torch.equal(grl, e_r * w[1] - e_r * w[2]), w


def test_batchnorm_wrapper_accepts_a_strided_beta():
    """kernels.batchnorm_train makes beta contiguous like its other inputs: a strided view gives what its copy gives (y
    and, on these dyadic inputs, dbeta bit for bit; dx up to the order of the atomics)."""
    from tecogan_b200 import kernels as K
    x, beta, dy = T.bn_inputs("192px_c64")
    wide = torch.zeros(2 * beta.size, device="cuda")
    wide[::2] = _dev(beta)
    outs = []
    for bt in (wide[::2], _dev(beta)):
        tx, tb = _dev(x.reshape(3, 8, 8, 64)).requires_grad_(True), bt.detach().requires_grad_(True)
        assert tb.is_contiguous() == (len(outs) == 1)
        y = K.batchnorm_train(tx, tb, False)
        outs.append((y,) + torch.autograd.grad(y, [tx, tb], _dev(dy.reshape(3, 8, 8, 64))))
    (y0, dx0, db0), (y1, dx1, db1) = outs
    assert torch.equal(y0, y1) and torch.equal(db0, db1) and float((dx0 - dx1).abs().max()) <= 1e-6
