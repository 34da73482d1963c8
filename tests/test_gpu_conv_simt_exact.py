"""The fp32 direct convolution teco_conv2d_f32, its weight gradient teco_conv2d_wgrad_f32 (csrc/conv_simt.cu) and the
3 x 3 / 2 max-pool of LPIPS, called through the C ABI against the float64 restatements of tests/conv_simt_cases.py, bit
for bit: at every launch the networks and LPIPS make (with a census test that keeps that table honest) and at the edges
of the kernels' load paths and launch geometry.  The exactness argument, the epilogue candidates and the bound for tanh
and the sigmoid are in that module's docstring; the guard is asserted per case before any comparison.

Every output is prefilled with a sentinel and followed by a guard region.  Pitched outputs keep the sentinel in the
channels from Cout on, and a phase-mapped output keeps it at the other three phases.  Pitched inputs and the unread
elements of residuals and of dy hold NaN, so a read outside the restated operands shows in the result.  A failure
names the count of wrong elements, the worst one and the pixel tile / Cout tile (forward) or the tap, ci tile, co tile
and split count (weight gradient) it belongs to."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests import conv_simt_cases as T

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
GUARD = 4096


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
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


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _buf(n, fill=None):
    """n floats (the sentinel, or `fill`) followed by a guard region holding the sentinel."""
    b = torch.full((n + GUARD,), SENTINEL, dtype=torch.float32, device="cuda")
    if fill is not None:
        b[:n] = torch.from_numpy(np.ascontiguousarray(fill, np.float32).ravel()).cuda()
    return b, b[:n]


def _guard_untouched(b, n, what):
    rest = b[n:].view(torch.int32)
    s = torch.tensor([SENTINEL], dtype=torch.float32).view(torch.int32).item()
    assert bool((rest == s).all()), "%s: wrote %d elements past its output" % (what, int((rest != s).sum()))


def _desc(c):
    from tecogan_b200._ffi import ConvDesc
    act, post = getattr(c, "act", 0), getattr(c, "post", (1.0, 0.0))
    return ConvDesc(N=c.N, H=c.H, W=c.W, Cin=c.Cin, OH=c.OH, OW=c.OW, Cout=c.Cout, KH=c.KH, KW=c.KW, stride=c.stride,
                    pad_t=c.pad_t, pad_l=c.pad_l, out_H=c.out_H, out_W=c.out_W, out_sy=c.out_map[0], out_oy=c.out_map[1],
                    out_sx=c.out_map[2], out_ox=c.out_map[3], in_cpitch=c.in_cp, out_cpitch=c.out_cp, act=act,
                    post_scale=post[0], post_shift=post[1])


def _call(name, *args):
    from tecogan_b200._ffi import call, stream_ptr
    call(name, *args, stream_ptr())
    torch.cuda.synchronize()


def _p(t):
    from tecogan_b200._ffi import ptr
    return ptr(t)


def _report(bad, err, what, where, detail):
    flat = np.flatnonzero(bad.ravel())
    w = int(flat[np.argmax(err.ravel()[flat])])
    idx = tuple(int(v) for v in np.unravel_index(w, bad.shape))
    raise AssertionError("%s: %d / %d elements wrong, worst at %s (%s): %s" % (
        what, flat.size, bad.size, idx, where(idx), detail(idx)))


def _i32(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _fwd_where(c):
    def f(idx):
        n, oy, ox, co = idx
        m = (n * c.OH + oy) * c.OW + ox
        return "pixel tile %d of %d, Cout tile %d" % (m // T.BM, T.fwd_launch(c)["tiles"], co // T.BN)
    return f


def _check_sentinel(got, mask, what):
    s = np.float32(SENTINEL).view(np.int32)
    bad = (_i32(got) != s) & ~mask
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError("%s: %d elements outside the written range changed, first at %s (%r)" % (
            what, int(bad.sum()), i, float(got[i])))


def _check_fwd(c, got_full, exp, what):
    """got_full: the whole output buffer [N,out_H,out_W,out_cp]; exp: candidate list or (value, bound)."""
    _check_sentinel(got_full, T.out_mask(c), what)
    got = T._mapped(c, got_full)
    if isinstance(exp, tuple):
        ref, bound = exp
        err = np.abs(got.astype(np.float64) - ref)
        bad = ~(err <= bound)
        if bad.any():
            _report(bad, err / np.maximum(bound, 1e-300), what, _fwd_where(c),
                    lambda i: "got %r, expected %r +- %.3g" % (float(got[i]), float(ref[i]), bound[i]))
        return
    ok = np.zeros(got.shape, bool)
    for a in exp:
        ok |= _i32(got) == _i32(a)
    if not ok.all():
        e = exp[0]
        _report(~ok, np.abs(got.astype(np.float64) - e) + 1, what, _fwd_where(c),
                lambda i: "got %r, expected %r" % (float(got[i]), float(e[i])))


def _run_fwd(c, x, w, b, res):
    n = c.N * c.out_H * c.out_W * c.out_cp
    buf, y = _buf(n)
    xd, wd, bd, rd = _dev(x), _dev(w), _dev(b), _dev(res)
    _call("teco_conv2d_f32", _desc(c), _p(xd), _p(wd), _p(bd), _p(rd), _p(y))
    _guard_untouched(buf, n, "y")
    return y.cpu().numpy().reshape(c.N, c.out_H, c.out_W, c.out_cp)


@pytest.mark.parametrize("name", list(T.FWD_CASES))
def test_conv2d_f32_bit_for_bit(name):
    c = T.FWD_CASES[name]
    x, w, b, res = T.fwd_inputs(name)
    z, mag = T.fwd_ref(c, x, w, b, res)
    T.guard(mag, T.G, name)
    got = _run_fwd(c, x, w, b, res)
    _check_fwd(c, got, T.epilogue(c, z, res), name)


def _wgrad_where(c):
    L = T.wgrad_launch(c, _sms())

    def f(idx):
        ky, kx, ci, co = idx
        return "tap %d, ci tile %d of %d, co tile %d of %d, %d splits of %d pixels" % (
            ky * c.KW + kx, ci // T.BM, L["ci_tiles"], co // T.BN, L["co_tiles"], L["splits"], L["pps"])
    return f


def _assert_equal(got, exp, what, where):
    bad = _i32(got) != _i32(exp.astype(np.float32))
    if bad.any():
        _report(bad, np.abs(got.astype(np.float64) - exp) + 1, what, where,
                lambda i: "got %r, expected %r" % (float(got[i]), float(exp[i])))


@pytest.mark.parametrize("name", list(T.WGRAD_CASES))
def test_conv2d_wgrad_f32_bit_for_bit(name):
    c = T.WGRAD_CASES[name]
    _same_class("wgrad", name, T.REQUIRED["wgrad"])
    x, dy, dw0, db0 = T.wgrad_inputs(name)
    dw_ref, mag, db_ref, dbm = T.wgrad_ref(c, x, dy, dw0, db0)
    T.guard(mag, T.G, name + " dw")
    T.guard(dbm, T.G_DB, name + " db")
    nw = dw0.size
    bw, dw = _buf(nw, dw0)
    bb, db = _buf(c.Cout, db0) if c.db else (None, None)
    xd, dyd = _dev(x), _dev(dy)
    _call("teco_conv2d_wgrad_f32", _desc(c), _p(xd), _p(dyd), _p(dw), _p(db), int(c.accumulate))
    _guard_untouched(bw, nw, name + " dw")
    _assert_equal(dw.cpu().numpy().reshape(dw0.shape), dw_ref, name + " dw", _wgrad_where(c))
    if c.db:
        _guard_untouched(bb, c.Cout, name + " db")
        _assert_equal(db.cpu().numpy(), db_ref, name + " db", lambda i: "channel %d" % i[0])


# ----------------------------------------------------------------------------------- validation order of the ABI
def test_rejected_wgrad_call_leaves_its_outputs_alone():
    """Cout = 320 with a bias gradient is rejected (bias_grad_kernel takes Cout <= 256) before anything is written; the
    same call without db runs and is exact."""
    c = T.wg(1, 6, 5, 1, 1, 8, 320, db=False)
    r = np.random.RandomState(3)
    x = (r.randint(-16, 17, (1, 6, 5, 8)) / 16).astype(np.float32)
    dy = (r.randint(-16, 17, (1, 6, 5, 320)) / 128).astype(np.float32)
    nw = 8 * 320
    bw, dw = _buf(nw)
    bb, db = _buf(320)
    xd, dyd = _dev(x), _dev(dy)
    with pytest.raises(ValueError, match="Cout <= 256"):
        _call("teco_conv2d_wgrad_f32", _desc(c), _p(xd), _p(dyd), _p(dw), _p(db), 0)
    _guard_untouched(bw, 0, "rejected call: dw")
    _guard_untouched(bb, 0, "rejected call: db")
    _call("teco_conv2d_wgrad_f32", _desc(c), _p(xd), _p(dyd), _p(dw), _p(None), 0)
    _guard_untouched(bw, nw, "dw")
    dw_ref = T.wgrad_ref(c, x, dy, None, None)[0]
    _assert_equal(dw.cpu().numpy().reshape(dw_ref.shape), dw_ref, "Cout 320 dw", _wgrad_where(c))


# ------------------------------------------------------------------------------------ the wrappers' autograd paths
def _g(r, shape, den, kmax=16):
    return r.randint(-kmax, kmax + 1, shape) / den


def _abs_grads(x, w, b, dy, stride, transpose=False):
    """Sum of |terms| of y, dx and dw (float64): the same linear maps on the magnitudes."""
    xa, wa = torch.from_numpy(np.abs(x)).requires_grad_(True), torch.from_numpy(np.abs(w)).requires_grad_(True)
    op = (lambda p, q: O.conv2d_transpose(p, q)) if transpose else (lambda p, q: O.conv2d(p, q, None, stride))
    y = op(xa, wa) + (0 if b is None else torch.from_numpy(np.abs(b)))
    gx, gw = torch.autograd.grad(op(xa, wa), (xa, wa), torch.from_numpy(np.abs(dy)))
    return y.detach().numpy(), gx.numpy(), gw.numpy()


def _bits_equal(got, exp, what):
    got = got.detach().cpu().numpy()
    exp = np.asarray(exp, np.float64)
    assert np.array_equal(got.astype(np.float64), exp) and np.array_equal(_i32(got), _i32(exp.astype(np.float32))), (
        "%s: %d / %d elements differ" % (what, int((got != exp).sum()), got.size))


# K, stride, (N, H, W), Cin, Cout, act, bias, residual: the dense layer (1 x 1, Cout 1), a 3 x 3 layer with each fused
# epilogue the networks use, the discriminator's 4 x 4 stride-2 blocks.  LeakyReLU and tanh are checked forward only:
# their derivatives leave the grid the exact comparison of the input and weight gradients needs.
WRAP = [(1, 1, (2, 3, 5), 256, 1, T.NONE, True, False), (3, 1, (2, 9, 11), 27, 64, T.LRELU, True, False),
        (3, 1, (2, 7, 6), 64, 64, T.RELU, True, False), (3, 1, (2, 8, 5), 64, 3, T.NONE, True, True),
        (3, 1, (1, 9, 7), 32, 2, T.TANH24, True, False), (4, 2, (2, 10, 12), 64, 128, T.NONE, False, False),
        (4, 2, (2, 8, 8), 128, 256, T.NONE, False, False)]


@pytest.mark.parametrize("K,stride,nhw,Cin,Cout,act,bias,res", WRAP)
def test_kernels_conv2d_forward_and_gradients_bit_for_bit(K, stride, nhw, Cin, Cout, act, bias, res):
    from tecogan_b200 import kernels as K_
    r = np.random.RandomState(K * 100 + Cin + Cout)
    x, w = _g(r, nhw + (Cin,), 16), _g(r, (K, K, Cin, Cout), 128)
    b = _g(r, (Cout,), 2048, 2048) if bias else None
    y64 = O.conv2d(torch.from_numpy(x), torch.from_numpy(w), None if b is None else torch.from_numpy(b), stride).numpy()
    rs = _g(r, y64.shape, 2048, 2048) if res else None
    dy = _g(r, y64.shape, 128)
    ya, gxa, gwa = _abs_grads(x, w, b, dy, stride)
    T.guard(ya + (0 if rs is None else np.abs(rs)), T.G, "y")
    T.guard(gxa, 2.0 ** -14, "dx")
    T.guard(gwa, T.G, "dw")
    T.guard(np.abs(dy).sum((0, 1, 2)), T.G_DB, "db")

    xg, wg = _dev(x).requires_grad_(True), _dev(w).requires_grad_(True)
    bg = _dev(b).requires_grad_(True) if bias else None
    y = K_.conv2d(xg, wg, bg, stride, act, _dev(rs))
    c = T.fwd(nhw[0], nhw[1], nhw[2], K, K, Cin, Cout, stride=stride, act=act, bias=bias, res=res)
    resf = None if rs is None else rs.astype(np.float32)
    exp = T.epilogue(c, y64, resf)
    _check_fwd(c, y.detach().cpu().numpy(), exp, "conv2d forward")
    if act in (T.LRELU, T.TANH24):
        return
    z = y64 if act == T.NONE else np.maximum(y64, 0)
    dz = dy if act == T.NONE else np.where(z > 0, dy, 0.0)
    xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
    gx, gw = torch.autograd.grad(O.conv2d(xt, wt, None, stride), (xt, wt), torch.from_numpy(dz))
    grads = torch.autograd.grad(y, [t for t in (xg, wg, bg) if t is not None], _dev(dy))
    _bits_equal(grads[0], gx.numpy(), "conv2d dx")
    _bits_equal(grads[1], gw.numpy(), "conv2d dw")
    if bias:
        _bits_equal(grads[2], dz.sum((0, 1, 2)), "conv2d db")


@pytest.mark.parametrize("nhw,Cin,Cout,act", [((2, 5, 7), 64, 64, T.RELU), ((1, 1, 3), 16, 12, T.NONE),
                                              ((2, 4, 4), 20, 8, T.RELU)])
def test_kernels_conv2d_transpose_forward_and_gradients_bit_for_bit(nhw, Cin, Cout, act):
    from tecogan_b200 import kernels as K_
    r = np.random.RandomState(Cin + Cout + nhw[1])
    x, w, b = _g(r, nhw + (Cin,), 16), _g(r, (3, 3, Cout, Cin), 128), _g(r, (Cout,), 2048, 2048)
    y64 = O.conv2d_transpose(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b)).numpy()
    dy = _g(r, y64.shape, 128)
    ya, gxa, gwa = _abs_grads(x, w, b, dy, 2, transpose=True)
    T.guard(ya, T.G, "y")
    T.guard(gxa, 2.0 ** -14, "dx")
    T.guard(gwa, T.G, "dw")
    xg, wg, bg = (_dev(a).requires_grad_(True) for a in (x, w, b))
    y = K_.conv2d_transpose(xg, wg, bg, act)
    z = y64 if act == T.NONE else np.maximum(y64, 0)
    _bits_equal(y, z, "conv2d_transpose forward")
    dz = dy if act == T.NONE else np.where(z > 0, dy, 0.0)
    xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
    gx, gw = torch.autograd.grad(O.conv2d_transpose(xt, wt), (xt, wt), torch.from_numpy(dz))
    dx, dw, db = torch.autograd.grad(y, (xg, wg, bg), _dev(dy))
    _bits_equal(dx, gx.numpy(), "conv2d_transpose dx")
    _bits_equal(dw, gw.numpy(), "conv2d_transpose dw")
    _bits_equal(db, dz.sum((0, 1, 2)), "conv2d_transpose db")


# ------------------------------------------------------------------------------------------------------ census
def census():
    """run -> set of launch keys of every teco_conv2d_f32 / teco_conv2d_wgrad_f32 call the run makes (kernels.call
    wrapped, each call passed through unchanged)."""
    from tecogan_b200 import config, kernels as K_
    from tecogan_b200.lib.frvsr import fnet, generator_F
    from tecogan_b200.lib.Teco import FRVSR, TecoGAN
    from tecogan_b200.variables import variable_scope
    from tests.golden import lpips_oracle as LO
    from tests.test_gpu_train import Flags, _case, _fresh_store, _load
    from tecogan_b200.lpips import LPIPS

    rec = set()
    orig = K_.call

    def spy(name, *args):
        if name == "teco_conv2d_f32":
            rec.add(T.desc_key("fwd", args[0], bias=args[3].value is not None, res=args[4].value is not None))
        elif name == "teco_conv2d_wgrad_f32":
            rec.add(T.desc_key("wgrad", args[0], accumulate=args[5], db=args[4].value is not None))
        return orig(name, *args)

    def step(case, precision):
        g, FL, P = _case(case)
        _fresh_store(P)
        config.set_train_precision(precision)
        ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
        net = TecoGAN(ri, rt, FL) if bool(g["gan"]) else FRVSR(ri, rt, FL)
        net.train()

    def inference():
        config.set_precision("fp32")
        _fresh_store({**O.init_generator(seed=5, num_resblock=2, bias_std=0.05), **O.init_fnet(seed=6, bias_std=0.05)})
        gen = torch.rand(2, 12, 16, 51, generator=torch.Generator().manual_seed(1)).cuda()
        fin = torch.rand(2, 16, 24, 6, generator=torch.Generator().manual_seed(2)).cuda()
        with torch.no_grad():
            with variable_scope('generator'):
                generator_F(gen, 3, reuse=False, FLAGS=Flags(num_resblock=2))
            with variable_scope('fnet'):
                fnet(fin, reuse=False)

    def lpips():
        g = _load("lpips")
        lin = {"lin%d.model.1.weight" % l: torch.from_numpy(g["lin%d" % l]).reshape(1, -1, 1, 1) for l in range(5)}
        model = LPIPS(LO.lpips_test_weights(int(g["alex_seed"])), lin)
        model.features(torch.from_numpy(g["tgt0"]).cuda(), tuple(int(v) for v in g["crop0"]))

    runs = {"fp32 FRVSR step": lambda: step("frvsr", "fp32"), "fp32 TecoGAN step": lambda: step("teco_pp", "fp32"),
            "bf16 TecoGAN step": lambda: step("teco_pp", "bf16"), "fp32 inference": inference,
            "LPIPS.features": lpips}
    out = {}
    prec, tprec = config.precision(), config.train_precision()
    K_.call = spy
    try:
        for run, f in runs.items():
            rec.clear()
            f()
            torch.cuda.synchronize()
            out[run] = set(rec)
    finally:
        K_.call = orig
        config.set_precision(prec)
        config.set_train_precision(tprec)
    return out


def test_census_of_network_launches_equals_the_layer_table(monkeypatch):
    """The keys of every fp32 convolution launch of an fp32 FRVSR and TecoGAN training step, a bf16 TecoGAN step, fp32
    inference of generator_F and fnet, and LPIPS.features are the layer table's, run by run: a layer that changes shape
    or kernel shows here, and so does a table entry no network launches."""
    from tecogan_b200 import kernels as K_
    monkeypatch.setattr(K_, "call", K_.call)        # restored even if census() is interrupted
    got = census()
    msgs = []
    for run, want in T.LAYERS.items():
        if got[run] != want:
            msgs.append("%s: launched but not in the table %s; in the table but not launched %s" % (
                run, sorted(got[run] - want), sorted(want - got[run])))
    assert not msgs, "\n".join(msgs)


# ---------------------------------------------------------------------------------------------- 3x3 / 2 max-pool
def _pool_input(shape, seed):
    r = np.random.RandomState(seed)
    x = r.randint(-3, 4, shape).astype(np.float32)           # few values: many tied maxima
    z = x == 0
    x[z & (r.rand(*shape) < 0.5)] = -0.0                     # +-0 mixed where the window maximum is zero
    return x


@pytest.mark.parametrize("shape", [(2, 7, 8, 5), (1, 3, 3, 4), (3, 3, 9, 2), (2, 10, 3, 3), (1, 6, 6, 1),
                                   (2, 31, 33, 64)])
def test_maxpool3s2_bit_for_bit(shape):
    x = _pool_input(shape, sum(shape))
    allneg = x.copy()
    allneg[0, :3, :3, 0] = [[-0.0, 0.0, -0.0], [0.0, -1.0, -0.0], [-2.0, 0.0, -0.0]]   # first max is -0: it stays
    nan = allneg.copy()
    nan[-1, 2, 2, -1] = np.nan                               # shared by up to four windows: NaN wins there
    for a, what in ((x, "ties"), (allneg, "+-0"), (nan, "NaN")):
        N, H, W, C = a.shape
        exp = T.maxpool3s2_ref(a)
        n = exp.size
        buf, y = _buf(n)
        xd = _dev(a)
        _call("teco_maxpool3s2_f32", _p(xd), _p(y), N, H, W, C)
        _guard_untouched(buf, n, what)
        got = y.cpu().numpy().reshape(exp.shape)
        bad = _i32(got) != _i32(exp)
        if bad.any():
            _report(bad, bad.astype(float), "maxpool3s2 %s %s" % (shape, what), lambda i: "window %s" % (i,),
                    lambda i: "got %r, expected %r" % (float(got[i]), float(exp[i])))
    assert np.isnan(T.maxpool3s2_ref(nan)[-1, 0, 0, -1])
    assert np.signbit(T.maxpool3s2_ref(allneg)[0, 0, 0, 0])
