"""GPU: the fixed-order (*_det) entry points sum in their declared order.  Where every operation of a kernel is a
correctly rounded fp32 operation, the result equals a host restatement of the order bit for bit, on continuous random
operands: bias gradient, batch-norm sums and variance, the beta gradient, L2 / L1 losses, the warp and resize scatter
gradients and the sum over ranks.  Where a kernel computes its partials with operations the host cannot restate (wgmma,
FMA main loops, log, rsqrt), the workspace it leaves holds the per-split partials and the result equals their fixed-order
sum.  Also: two calls agree bit for bit, grid operands are exact against float64, bad arguments (a short workspace
included) raise ValueError, and nothing outside the outputs is written."""
import ctypes

import numpy as np
import pytest
import torch

from tests import det_plans as DP

pytestmark = pytest.mark.gpu

f32 = np.float32


def _K():
    from tecogan_b200 import kernels as K
    return K


def _call(name, *args):
    from tecogan_b200._ffi import call
    call(name, *args)


def _p(t):
    from tecogan_b200._ffi import ptr
    return ptr(t)


def _s():
    from tecogan_b200._ffi import stream_ptr
    return stream_ptr()


def _ws(name, *plan):
    nb = _K().plan_bytes(name, *plan)
    return torch.full((nb // 4 + 64,), float("nan"), device="cuda", dtype=torch.float32), nb


def _guarded(n, fill=0.0, guard=64):
    """A device buffer with `guard` NaN-marked floats each side; returns (whole, view)."""
    whole = torch.full((n + 2 * guard,), float("nan"), device="cuda", dtype=torch.float32)
    v = whole[guard:guard + n]
    v.fill_(fill)
    return whole, v


def _guards_intact(whole, guard=64):
    return bool(torch.isnan(whole[:guard]).all()) and bool(torch.isnan(whole[-guard:]).all())


def _eq(a, b):
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _ordered(parts, prev=None):
    """parts[0] + parts[1] + ... in order, in float32; then prev + that when accumulating."""
    t = parts[0].astype(f32)
    for p in parts[1:]:
        t = (t + p).astype(f32)
    return t if prev is None else (prev + t).astype(f32)


# ------------------------------------------------------------------------------------------ bias gradient
def _bias_host(dy, C, prev=None):
    M = dy.shape[0]
    blocks, ppb = DP.bias(M, C)
    ppar = 256 // C
    parts = []
    for b in range(blocks):
        p0, p1 = b * ppb, min(M, (b + 1) * ppb)
        lanes = []
        for ps in range(ppar):
            s = np.zeros(C, f32)
            for p in range(p0 + ps, p1, ppar):
                s = (s + dy[p, :C]).astype(f32)
            lanes.append(s)
        parts.append(_ordered(lanes))
    return _ordered(parts, prev)


@pytest.mark.parametrize("npix,C,cpitch", [(1, 1, 1), (37, 3, 3), (1000, 64, 64), (5003, 100, 128), (2049, 256, 256),
                                           (40000, 1, 4)])
@pytest.mark.parametrize("acc", [0, 1])
def test_bias_grad_det_is_its_declared_order(npix, C, cpitch, acc):
    rng = np.random.default_rng(npix + C)
    dy = rng.standard_normal((npix, cpitch)).astype(f32)
    prev = rng.standard_normal(C).astype(f32)
    whole, db = _guarded(C)
    db.copy_(torch.from_numpy(prev))
    ws, nb = _ws("teco_bias_grad_f32_det", npix, C)
    _call("teco_bias_grad_f32_det", _p(torch.from_numpy(dy).cuda()), _p(db), npix, C, cpitch, acc, _p(ws), nb, _s())
    torch.cuda.synchronize()
    assert _eq(db.cpu().numpy(), _bias_host(dy, C, prev if acc else None))
    assert _guards_intact(whole)


# ------------------------------------------------------------------------------------------ batch norm
def _bn_sums_host(x, npix, C):
    blocks, ppb = DP.bn(npix)
    ppar = 256 // C

    def reduce(f):
        parts = []
        for b in range(blocks):
            p0, p1 = b * ppb, min(npix, (b + 1) * ppb)
            lanes = []
            for ps in range(ppar):
                s = np.zeros(C, f32)
                for p in range(p0 + ps, p1, ppar):
                    s = (s + f(p)).astype(f32)
                lanes.append(s)
            parts.append(_ordered(lanes))
        return _ordered(parts)
    s = reduce(lambda p: x[p])
    mean = (s / f32(npix)).astype(f32)
    q = reduce(lambda p: ((x[p] - mean).astype(f32) * (x[p] - mean).astype(f32)).astype(f32))
    return s, q


@pytest.mark.parametrize("npix,C", [(1, 1), (5, 3), (1500, 64), (3000, 256), (2100, 100), (300000, 1)])
def test_bn_det_statistics_and_beta_gradient(npix, C):
    rng = np.random.default_rng(npix * 7 + C)
    x = (rng.standard_normal((npix, C)) * 2 + 0.5).astype(f32)
    dy = rng.standard_normal((npix, C)).astype(f32)
    beta = rng.standard_normal(C).astype(f32)
    xd, dyd, bd = (torch.from_numpy(a).cuda() for a in (x, dy, beta))
    y = torch.empty_like(xd)
    sw, stats = _guarded(4 * C)
    ws, nb = _ws("teco_bn_det", npix, C)
    _call("teco_bn_train_f32_det", _p(xd), _p(bd), _p(y), _p(stats), npix, C, ctypes.c_float(1e-3), 1, _p(ws), nb, _s())
    torch.cuda.synchronize()
    s, q = _bn_sums_host(x, npix, C)
    st = stats.cpu().numpy()
    assert _eq(st[2 * C:3 * C], s) and _eq(st[3 * C:], q)
    assert _eq(st[:C], (s / f32(npix)).astype(f32)) and _eq(st[C:2 * C], (q / f32(npix)).astype(f32))
    assert _guards_intact(sw)
    # backward: dbeta = sum of g in the declared order (restated); the sum of g * xhat is the ordered sum of its partials
    dx = torch.empty_like(xd)
    dw_, dbeta = _guarded(2 * C)
    _call("teco_bn_train_bwd_f32_det", _p(xd), _p(y), _p(dyd), _p(stats), _p(dx), _p(dbeta), npix, C, ctypes.c_float(1e-3),
          1, _p(ws), nb, _s())
    torch.cuda.synchronize()
    g = np.where(y.cpu().numpy() < 0, (dy * f32(0.2)).astype(f32), dy)
    blocks, _ = DP.bn(npix)
    gsum, _ = _bn_sums_host(g, npix, C)
    db = dbeta.cpu().numpy()
    assert _eq(db[:C], gsum)
    parts = ws[:blocks * 2 * C].cpu().numpy().reshape(blocks, 2 * C)
    assert _eq(db, _ordered(list(parts)))
    assert _guards_intact(dw_)
    # the default kernels agree to rounding
    stats2 = torch.empty(4 * C, device="cuda")
    _call("teco_bn_train_f32", _p(xd), _p(bd), _p(torch.empty_like(xd)), _p(stats2), npix, C, ctypes.c_float(1e-3), 1, _s())
    torch.testing.assert_close(stats2[:2 * C], stats[:2 * C], rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------ losses
def _block_values_host(vals, blocks):
    """Per-thread grid-stride sums of `vals` (already rounded per element), then block_sum's warp butterflies, for a grid
    of `blocks` x 256 threads: the value thread 0 of each block holds."""
    T = blocks * 256
    n = vals.shape[0]
    pad = np.zeros(DP.cdiv(n, T) * T, f32)
    pad[:n] = vals
    s = np.zeros(T, f32)
    for row in pad.reshape(-1, T):
        s = (s + row).astype(f32)
    v = s.reshape(blocks, 8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, :, lanes ^ o]).astype(f32)
    w = np.zeros((blocks, 32), f32)
    w[:, :8] = v[:, :, 0]
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, lanes ^ o]).astype(f32)
    return w[:, 0]


@pytest.mark.parametrize("npix,C", [(1, 1), (333, 3), (4096, 64), (70001, 3), (3_000_000, 3)])
def test_l2_l1_losses_det_are_their_declared_order(npix, C):
    rng = np.random.default_rng(npix + 11 * C)
    a = rng.standard_normal(npix * C).astype(f32)
    b = rng.standard_normal(npix * C).astype(f32)
    ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    d = (a - b).astype(f32)
    ws, nb = _ws("teco_loss_det", npix, C)
    out = torch.empty(1, device="cuda")
    _call("teco_loss_l2_f32_det", _p(ad), _p(bd), _p(out), _p(None), npix, C, ctypes.c_float(1.0), _p(ws), nb, _s())
    blocks = DP.loss_blocks("l2", npix, C)
    inv = f32(1.0) / f32(npix)
    want = _ordered(list((_block_values_host((d * d).astype(f32), blocks) * inv).astype(f32)))
    assert _eq(out.cpu().numpy()[0], want)
    for per_pixel in (0, 1):
        _call("teco_loss_l1_f32_det", _p(ad), _p(bd), _p(out), _p(None), _p(None), npix, C, per_pixel, ctypes.c_float(1.0),
              _p(ws), nb, _s())
        inv = f32(1.0) / f32(npix) if per_pixel else f32(1.0) / (f32(npix) * f32(C))
        want = _ordered(list((_block_values_host(np.abs(d), blocks) * inv).astype(f32)))
        assert _eq(out.cpu().numpy()[0], want)


@pytest.mark.parametrize("npix,C", [(1, 64), (500, 64), (20000, 256)])
def test_cosine_and_gan_losses_det_sum_their_partials_in_order(npix, C):
    rng = np.random.default_rng(npix)
    f = torch.from_numpy(rng.standard_normal(npix * C).astype(f32)).cuda()
    g = torch.from_numpy(rng.standard_normal(npix * C).astype(f32)).cuda()
    ws, nb = _ws("teco_loss_det", npix, C)
    out = torch.empty(1, device="cuda")
    outs = []
    for _ in range(2):
        _call("teco_loss_cosine_f32_det", _p(f), _p(g), _p(out), _p(None), npix, C, ctypes.c_float(1.0), _p(ws), nb, _s())
        outs.append(out.clone())
    blocks = DP.loss_blocks("cosine", npix, C)
    assert torch.equal(outs[0], outs[1])
    assert _eq(out.cpu().numpy()[0], (_ordered(list(ws[:blocks].cpu().numpy())) + f32(1.0)).astype(f32))
    ref = torch.empty(1, device="cuda")
    _call("teco_loss_cosine_f32", _p(f), _p(g), _p(ref), _p(None), npix, C, ctypes.c_float(1.0), _s())
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-6)
    n = npix * 3
    pf = torch.from_numpy(rng.uniform(0.01, 0.99, n).astype(f32)).cuda()
    pr = torch.from_numpy(rng.uniform(0.01, 0.99, n).astype(f32)).cuda()
    ws, nb = _ws("teco_loss_det", n, 1)
    o5 = torch.empty(5, device="cuda")
    _call("teco_loss_gan_f32_det", _p(pf), _p(pr), _p(o5), _p(None), _p(None), _p(None), n, ctypes.c_float(1e-12),
          ctypes.c_float(1.0), ctypes.c_float(1.0), _p(ws), nb, _s())
    blocks = DP.loss_blocks("gan", n, 1)
    assert _eq(o5.cpu().numpy(), _ordered(list(ws[:blocks * 5].cpu().numpy().reshape(blocks, 5))))
    r5 = torch.empty(5, device="cuda")
    _call("teco_loss_gan_f32", _p(pf), _p(pr), _p(r5), _p(None), _p(None), _p(None), n, ctypes.c_float(1e-12),
          ctypes.c_float(1.0), ctypes.c_float(1.0), _s())
    torch.testing.assert_close(o5, r5, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------ scatter gradients
def _ordered_scatter(targets, keys, values, n):
    """out[t] = sum of values[j] with targets[j] == t, in ascending keys[j], starting from 0, in float32."""
    out = np.zeros((n,) + values.shape[1:], f32)
    for j in np.lexsort((keys, targets)):
        out[targets[j]] = (out[targets[j]] + values[j]).astype(f32)
    return out


def _warp_dimg_host(flow, dout, N, H, W, C):
    P = N * H * W
    i = np.arange(P)
    x, y, n = i % W, (i // W) % H, i // (W * H)
    fl = flow.reshape(P, 2)
    qy = (y.astype(f32) - fl[:, 0]).astype(f32)
    qx = (x.astype(f32) - fl[:, 1]).astype(f32)
    fy = np.clip(np.floor(qy), f32(0), f32(H - 2)).astype(f32)
    fx = np.clip(np.floor(qx), f32(0), f32(W - 2)).astype(f32)
    ay = np.clip((qy - fy).astype(f32), f32(0), f32(1))
    ax = np.clip((qx - fx).astype(f32), f32(0), f32(1))
    y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
    g = dout.reshape(P, C)
    tg, ks, vs = [], [], []
    for k in range(4):
        wy = ay if k >> 1 else (f32(1) - ay).astype(f32)
        wx = ax if k & 1 else (f32(1) - ax).astype(f32)
        tg.append((n * H + y0 + (k >> 1)) * W + x0 + (k & 1))
        ks.append(4 * i + k)
        vs.append(((g * wy[:, None]).astype(f32) * wx[:, None]).astype(f32))
    return _ordered_scatter(np.concatenate(tg), np.concatenate(ks), np.concatenate(vs), P).reshape(N, H, W, C)


def _flows(kind, N, H, W, rng):
    if kind == "random":
        return (rng.standard_normal((N, H, W, 2)) * 2.5).astype(f32)
    yy, xx = np.meshgrid(np.arange(H, dtype=f32), np.arange(W, dtype=f32), indexing="ij")
    if kind == "converge":      # every source of an image reads around pixel (H/2 + 0.3, W/3 + 0.6)
        f = np.stack([yy - (H // 2 + f32(0.3)), xx - (W // 3 + f32(0.6))], -1)
        return np.broadcast_to(f, (N, H, W, 2)).astype(f32)
    f = (rng.standard_normal((N, H, W, 2)) * 3 * max(H, W)).astype(f32)   # "clamp": most queries leave the image
    return f


@pytest.mark.parametrize("N,H,W,C", [(1, 2, 2, 1), (2, 17, 23, 3), (3, 32, 32, 3), (1, 40, 9, 5)])
@pytest.mark.parametrize("kind", ["random", "converge", "clamp"])
def test_warp_bwd_det_is_ascending_source_order(N, H, W, C, kind):
    rng = np.random.default_rng(N * H * W + C)
    flow = _flows(kind, N, H, W, rng)
    img = rng.standard_normal((N, H, W, C)).astype(f32)
    dout = rng.standard_normal((N, H, W, C)).astype(f32)
    imgd, flowd, doutd = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (img, flow, dout))
    wd, dimg = _guarded(N * H * W * C, fill=123.0)
    dflow = torch.empty_like(flowd)
    ws, nb = _ws("teco_warp_bwd_f32_det", N, H, W)
    _call("teco_warp_bwd_f32_det", _p(imgd), _p(flowd), _p(doutd), _p(dimg), _p(dflow), N, H, W, C, _p(ws), nb, _s())
    torch.cuda.synchronize()
    assert _eq(dimg.cpu().numpy().reshape(N, H, W, C), _warp_dimg_host(flow, dout, N, H, W, C))
    assert _guards_intact(wd)
    ref_dimg, ref_dflow = torch.zeros_like(imgd), torch.empty_like(flowd)
    _call("teco_warp_bwd_f32", _p(imgd), _p(flowd), _p(doutd), _p(ref_dimg), _p(ref_dflow), N, H, W, C, _s())
    assert torch.equal(dflow, ref_dflow)            # dflow is the same gather on both paths
    torch.testing.assert_close(dimg.view(N, H, W, C), ref_dimg, rtol=1e-5, atol=1e-5)


def _resize_host(dy, N, h, w, C, oh, ow):
    sy, sx = f32(h) / f32(oh), f32(w) / f32(ow)
    Y, X = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    fy = (Y.astype(f32) * sy).astype(f32)
    fx = (X.astype(f32) * sx).astype(f32)
    y0, x0 = np.floor(fy).astype(np.int64), np.floor(fx).astype(np.int64)
    y1, x1 = np.minimum(y0 + 1, h - 1), np.minimum(x0 + 1, w - 1)
    wy, wx = (fy - y0.astype(f32)).astype(f32), (fx - x0.astype(f32)).astype(f32)
    out = np.zeros((N, h, w, C), f32)
    key = (Y * ow + X).ravel()
    for n in range(N):
        g = dy[n].reshape(oh * ow, C)
        tg, ks, vs = [], [], []
        for k, (yy, xx, a, b) in enumerate([(y0, x0, f32(1) - wy, f32(1) - wx), (y0, x1, f32(1) - wy, wx),
                                            (y1, x0, wy, f32(1) - wx), (y1, x1, wy, wx)]):
            a, b = np.asarray(a, f32).ravel(), np.asarray(b, f32).ravel()
            tg.append((yy * w + xx).ravel())
            ks.append(4 * key + k)
            vs.append(((g * a[:, None]).astype(f32) * b[:, None]).astype(f32))
        out[n] = _ordered_scatter(np.concatenate(tg), np.concatenate(ks), np.concatenate(vs), h * w).reshape(h, w, C)
    return out


@pytest.mark.parametrize("N,h,w,C,oh,ow", [(1, 1, 1, 1, 3, 2), (2, 4, 4, 32, 8, 8), (3, 8, 12, 3, 32, 48),
                                           (1, 5, 7, 2, 11, 13), (2, 9, 6, 3, 5, 4)])
def test_resize_bilinear_bwd_det_is_its_gather_order(N, h, w, C, oh, ow):
    rng = np.random.default_rng(h * w + oh)
    dy = rng.standard_normal((N, oh, ow, C)).astype(f32)
    dyd = torch.from_numpy(dy).cuda()
    wd, dx = _guarded(N * h * w * C, fill=7.0)
    _call("teco_resize_bilinear_bwd_f32_det", _p(dyd), _p(dx), N, h, w, C, oh, ow, _s())
    torch.cuda.synchronize()
    assert _eq(dx.cpu().numpy().reshape(N, h, w, C), _resize_host(dy, N, h, w, C, oh, ow))
    assert _guards_intact(wd)


# ------------------------------------------------------------------------------------------ weight gradients
def _bf16_rows(a, cpad):
    N, H, W, C = a.shape
    t = torch.zeros((N, H, W, cpad), dtype=torch.bfloat16)
    t[..., :C] = torch.from_numpy(a).to(torch.bfloat16)
    return t.cuda()


@pytest.mark.parametrize("N,H,W,cin,cout", [(1, 8, 16, 64, 64), (3, 13, 29, 64, 4), (40, 16, 16, 64, 64),
                                            (2, 9, 21, 256, 64), (2, 8, 8, 512, 256)])
@pytest.mark.parametrize("acc", [0, 1])
def test_wgrad_tc_det_sums_its_splits_in_order(N, H, W, cin, cout, acc):
    rng = np.random.default_rng(N * H + cin + cout)
    x = _bf16_rows(rng.standard_normal((N, H, W, cin)).astype(f32), DP.cdiv(cin, 64) * 64)
    dz = _bf16_rows(rng.standard_normal((N, H, W, cout)).astype(f32), DP.cdiv(cout, 64) * 64)
    prev = rng.standard_normal(9 * cin * cout).astype(f32)
    wd, dw = _guarded(9 * cin * cout)
    dw.copy_(torch.from_numpy(prev))
    ws, nb = _ws("teco_conv3x3_wgrad_tc_det", N, H, W, cin, cout)
    args = (N, H, W, x.shape[-1], dz.shape[-1], cin, cout, _p(x), _p(dz), _p(dw), acc, _p(ws), nb, _s())
    _call("teco_conv3x3_wgrad_tc_det", *args)
    torch.cuda.synchronize()
    splits, _ = DP.wgrad_tc(N, H, W, cin, cout)
    parts = ws[:splits * 9 * cin * cout].cpu().numpy().reshape(splits, -1)
    first = dw.cpu().numpy()
    assert _eq(first, _ordered(list(parts), prev if acc else None))
    assert _guards_intact(wd)
    dw.copy_(torch.from_numpy(prev))
    _call("teco_conv3x3_wgrad_tc_det", *args)
    assert _eq(dw.cpu().numpy(), first)
    ref = torch.from_numpy(prev).cuda() if acc else torch.empty(9 * cin * cout, device="cuda")
    _call("teco_conv3x3_wgrad_tc", N, H, W, x.shape[-1], dz.shape[-1], cin, cout, _p(x), _p(dz), _p(ref), acc, _s())
    torch.testing.assert_close(dw, ref, rtol=1e-4, atol=1e-3)


def test_wgrad_tc_det_exact_on_grid_operands():
    """Small integers in bf16, products and sums exact in fp32: the result equals float64 whatever the order."""
    N, H, W, cin, cout = 5, 19, 35, 64, 64
    rng = np.random.default_rng(5)
    xa = rng.integers(-3, 4, (N, H, W, cin)).astype(f32)
    za = rng.integers(-3, 4, (N, H, W, cout)).astype(f32)
    x, dz = _bf16_rows(xa, 64), _bf16_rows(za, 64)
    dw = torch.empty(9 * cin * cout, device="cuda")
    ws, nb = _ws("teco_conv3x3_wgrad_tc_det", N, H, W, cin, cout)
    _call("teco_conv3x3_wgrad_tc_det", N, H, W, 64, 64, cin, cout, _p(x), _p(dz), _p(dw), 0, _p(ws), nb, _s())
    xp = np.pad(xa.astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
    want = np.zeros((3, 3, cin, cout))
    for ky in range(3):
        for kx in range(3):
            want[ky, kx] = np.einsum("nhwc,nhwd->cd", xp[:, ky:ky + H, kx:kx + W], za.astype(np.float64))
    assert np.array_equal(dw.cpu().numpy().reshape(3, 3, cin, cout).astype(np.float64), want)


def _desc(N, H, W, Cin, Cout, K, stride):
    from tecogan_b200._ffi import ConvDesc
    from tecogan_b200.kernels import same_pad
    pt, OH = same_pad(H, K, stride)
    pl, OW = same_pad(W, K, stride)
    return ConvDesc(N=N, H=H, W=W, Cin=Cin, OH=OH, OW=OW, Cout=Cout, KH=K, KW=K, stride=stride, pad_t=pt, pad_l=pl,
                    out_H=OH, out_W=OW, out_sy=1, out_oy=0, out_sx=1, out_ox=0, in_cpitch=Cin, out_cpitch=Cout, act=0,
                    post_scale=1.0, post_shift=0.0)


@pytest.mark.parametrize("N,H,W,Cin,Cout,K,stride", [(1, 5, 7, 3, 64, 3, 1), (4, 32, 32, 64, 64, 3, 1),
                                                     (2, 33, 17, 20, 3, 3, 1), (2, 32, 32, 64, 128, 4, 2)])
@pytest.mark.parametrize("acc", [0, 1])
def test_wgrad_f32_det_sums_its_splits_in_order(N, H, W, Cin, Cout, K, stride, acc):
    d = _desc(N, H, W, Cin, Cout, K, stride)
    rng = np.random.default_rng(N + H + Cin + Cout)
    x = torch.from_numpy(rng.standard_normal((N, H, W, Cin)).astype(f32)).cuda()
    dy_np = rng.standard_normal((N, d.OH, d.OW, Cout)).astype(f32)
    dy = torch.from_numpy(dy_np).cuda()
    E = K * K * Cin * Cout
    prev_w = rng.standard_normal(E).astype(f32)
    prev_b = rng.standard_normal(Cout).astype(f32)
    wd, dw = _guarded(E)
    bd, db = _guarded(Cout)
    dw.copy_(torch.from_numpy(prev_w))
    db.copy_(torch.from_numpy(prev_b))
    ws, nb = _ws("teco_conv2d_wgrad_f32_det", d, 1)
    _call("teco_conv2d_wgrad_f32_det", d, _p(x), _p(dy), _p(dw), _p(db), acc, _p(ws), nb, _s())
    torch.cuda.synchronize()
    M = N * d.OH * d.OW
    splits, _ = DP.wgrad_f32(M, K, K, Cin, Cout)
    parts = ws[:splits * E].cpu().numpy().reshape(splits, E)
    assert _eq(dw.cpu().numpy(), _ordered(list(parts), prev_w if acc else None))
    assert _eq(db.cpu().numpy(), _bias_host(dy_np.reshape(M, Cout), Cout, prev_b if acc else None))
    assert _guards_intact(wd) and _guards_intact(bd)
    rw = torch.from_numpy(prev_w).cuda() if acc else torch.empty(E, device="cuda")
    rb = torch.from_numpy(prev_b).cuda() if acc else torch.empty(Cout, device="cuda")
    _call("teco_conv2d_wgrad_f32", d, _p(x), _p(dy), _p(rw), _p(rb), acc, _s())
    torch.testing.assert_close(dw, rw, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(db, rb, rtol=1e-4, atol=1e-4)


def test_sum_ranks_is_rank_order():
    rng = np.random.default_rng(3)
    src = rng.standard_normal((5, 10007)).astype(f32)
    out = _K().sum_ranks(torch.from_numpy(src).cuda())
    assert _eq(out.cpu().numpy(), _ordered(list(src)))


def test_det_entry_points_reject_bad_arguments():
    x = torch.zeros(4096, device="cuda")
    ws, nb = _ws("teco_bias_grad_f32_det", 100, 8)
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_bias_grad_f32_det", _p(x), _p(x), 100, 8, 8, 0, _p(ws), nb - 4, _s())
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_bias_grad_f32_det", _p(x), _p(x), 100, 8, 8, 0, _p(None), nb, _s())
    with pytest.raises(ValueError):
        _call("teco_bias_grad_f32_det", _p(x), _p(x), 100, 300, 300, 0, _p(ws), nb, _s())
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_bn_train_f32_det", _p(x), _p(x), _p(x), _p(x), 100, 4, ctypes.c_float(1e-3), 0, _p(ws), 4, _s())
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_loss_l2_f32_det", _p(x), _p(x), _p(x), _p(None), 100, 4, ctypes.c_float(1.0), _p(ws), 0, _s())
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_warp_bwd_f32_det", _p(x), _p(x), _p(x), _p(x), _p(None), 1, 8, 8, 3, _p(ws), 8, _s())
    with pytest.raises(ValueError):
        _call("teco_warp_bwd_f32_det", _p(x), _p(x), _p(x), _p(x), _p(None), 1, 1, 8, 3, _p(ws), nb, _s())
    xb = torch.zeros(8 * 16 * 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_conv3x3_wgrad_tc_det", 1, 8, 16, 64, 64, 64, 64, _p(xb), _p(xb), _p(x), 0, _p(ws), 16, _s())
    with pytest.raises(ValueError):
        _call("teco_conv3x3_wgrad_tc_det", 1, 8, 16, 64, 64, 64, 6, _p(xb), _p(xb), _p(x), 0, _p(ws), nb, _s())
    with pytest.raises(ValueError):
        _call("teco_sum_ranks_f32", _p(x), 0, 10, _p(x), _s())
    d = _desc(1, 8, 8, 4, 4, 3, 1)
    with pytest.raises(ValueError, match="workspace"):
        _call("teco_conv2d_wgrad_f32_det", d, _p(x), _p(x), _p(x), _p(x), 0, _p(ws), 4, _s())
