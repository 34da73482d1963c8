"""GPU parity: every libteco.so kernel (through the C ABI) against the CPU oracle on the same seeded inputs.
fp32 kernels: tight tolerances (accumulation-order noise only).  bf16 tensor-core kernel: compared with the
oracle evaluated on the SAME bf16-rounded operands, so only fp32 accumulation order and the final bf16
rounding (2^-9 relative) remain."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O

pytestmark = pytest.mark.gpu


def dev(t):
    return t.cuda().contiguous()


def rnd(seed, *shape, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape, generator=g) * (hi - lo) + lo


def assert_close(got, ref, atol, rtol=0.0, what=""):
    got = got.detach().float().cpu()
    ref = ref.detach().float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    assert not bad.any(), "%s: max err %.3e (tol %.1e) at %d/%d elements; ref scale %.3e" % (
        what, err.max().item(), atol, int(bad.sum()), bad.numel(), ref.abs().max().item())


# ------------------------------------------------------------------------------------ fp32 convolutions
@pytest.mark.parametrize("n,h,w,cin,cout,k,s", [
    (2, 13, 17, 3, 64, 3, 1), (1, 32, 32, 51, 64, 3, 1), (2, 16, 20, 64, 64, 3, 1), (1, 9, 11, 64, 3, 3, 1),
    (1, 8, 8, 32, 2, 3, 1), (2, 32, 32, 27, 64, 3, 1), (2, 32, 32, 64, 64, 4, 2), (1, 16, 16, 128, 256, 4, 2),
    (1, 6, 10, 256, 1, 1, 1), (1, 24, 16, 6, 32, 3, 1), (1, 14, 18, 128, 128, 3, 1),
])
def test_conv2d_f32_matches_oracle(n, h, w, cin, cout, k, s):
    from tecogan_b200 import kernels as K
    x, wt, b = rnd(1, n, h, w, cin), rnd(2, k, k, cin, cout) * 0.2, rnd(3, cout)
    ref = O.conv2d(x, wt, b, s)
    got = K.conv2d(dev(x), dev(wt), dev(b), s)
    assert_close(got, ref, 2e-5 * max(1.0, ref.abs().max().item()), what="conv2d")
    for act, fn in ((K.ACT_RELU, torch.relu), (K.ACT_LRELU02, O.lrelu), (K.ACT_TANH24, lambda v: torch.tanh(v) * 24),
                    (K.ACT_SIGMOID, torch.sigmoid)):
        got = K.conv2d(dev(x), dev(wt), dev(b), s, act)
        assert_close(got, fn(ref), 5e-5 * max(1.0, ref.abs().max().item()), what="conv2d+act%d" % act)
    res = rnd(4, *ref.shape)
    got = K.conv2d(dev(x), dev(wt), None, s, K.ACT_NONE, dev(res))
    assert_close(got, O.conv2d(x, wt, None, s) + res, 2e-5 * max(1.0, ref.abs().max().item()), what="conv2d+res")


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 8, 8, 64, 64), (2, 5, 7, 16, 8), (1, 16, 12, 64, 64)])
def test_conv2d_transpose_f32_matches_oracle(n, h, w, cin, cout):
    from tecogan_b200 import kernels as K
    x, wt, b = rnd(5, n, h, w, cin), rnd(6, 3, 3, cout, cin) * 0.2, rnd(7, cout)
    ref = O.conv2d_transpose(x, wt, b)
    got = K.conv2d_transpose(dev(x), dev(wt), dev(b))
    assert_close(got, ref, 2e-5 * max(1.0, ref.abs().max().item()), what="conv2d_transpose")
    got = K.conv2d_transpose(dev(x), dev(wt), dev(b), K.ACT_RELU)
    assert_close(got, torch.relu(ref), 2e-5 * max(1.0, ref.abs().max().item()), what="conv2d_transpose+relu")


def _grads(fn_ref, fn_got, tensors, seed=11):
    """Compare autograd gradients of sum(out * r) between oracle (CPU) and kernels (GPU)."""
    cpu = [t.clone().requires_grad_(True) for t in tensors]
    gpu = [dev(t).requires_grad_(True) for t in tensors]
    o_ref, o_got = fn_ref(*cpu), fn_got(*gpu)
    r = rnd(seed, *o_ref.shape)
    g_ref = torch.autograd.grad((o_ref * r).sum(), cpu)
    g_got = torch.autograd.grad((o_got * dev(r)).sum(), gpu)
    return o_ref, o_got, g_ref, g_got


@pytest.mark.parametrize("n,h,w,cin,cout,k,s,act", [
    (2, 12, 10, 16, 24, 3, 1, 0), (1, 16, 16, 51, 64, 3, 1, 1), (2, 16, 16, 27, 64, 4, 2, 2), (1, 8, 8, 64, 2, 3, 1, 3),
    (1, 8, 8, 256, 1, 1, 1, 4), (1, 32, 32, 64, 128, 4, 2, 0),
])
def test_conv2d_backward_matches_oracle_autograd(n, h, w, cin, cout, k, s, act):
    from tecogan_b200 import kernels as K
    acts = {0: lambda v: v, 1: torch.relu, 2: O.lrelu, 3: lambda v: torch.tanh(v) * 24, 4: torch.sigmoid}
    x, wt, b = rnd(1, n, h, w, cin), rnd(2, k, k, cin, cout) * 0.1, rnd(3, cout) * 0.1
    o_ref, o_got, g_ref, g_got = _grads(lambda a, c, d: acts[act](O.conv2d(a, c, d, s)),
                                        lambda a, c, d: K.conv2d(a, c, d, s, act), [x, wt, b])
    for name, gr, gg in zip(("dx", "dw", "db"), g_ref, g_got):
        assert_close(gg, gr, 1e-4 * max(1.0, gr.abs().max().item()), what="conv2d bwd " + name)


def test_conv2d_transpose_backward_matches_oracle_autograd():
    from tecogan_b200 import kernels as K
    x, wt, b = rnd(1, 2, 6, 5, 16), rnd(2, 3, 3, 24, 16) * 0.1, rnd(3, 24) * 0.1
    _, _, g_ref, g_got = _grads(lambda a, c, d: torch.relu(O.conv2d_transpose(a, c, d)),
                                lambda a, c, d: K.conv2d_transpose(a, c, d, K.ACT_RELU), [x, wt, b])
    for name, gr, gg in zip(("dx", "dw", "db"), g_ref, g_got):
        assert_close(gg, gr, 1e-4 * max(1.0, gr.abs().max().item()), what="tconv bwd " + name)


# ------------------------------------------------------------------------------------ resampling family
def test_warp_and_gradients_match_oracle():
    from tecogan_b200 import kernels as K
    img, flow = rnd(1, 2, 20, 24, 3), rnd(2, 2, 20, 24, 2, lo=-5, hi=5)
    flow[0, 0, 0] = torch.tensor([30.0, -30.0])  # far out of range: clamped
    ref = O.dense_image_warp(img, flow)
    assert_close(K.dense_image_warp(dev(img), dev(flow)), ref, 1e-5, what="warp")
    _, _, g_ref, g_got = _grads(O.dense_image_warp, K.dense_image_warp, [img, flow])
    assert_close(g_got[0], g_ref[0], 1e-5, what="warp dimg")
    assert_close(g_got[1], g_ref[1], 1e-4, what="warp dflow")


def test_in_tree_resamplers_match_golden_and_oracle():
    import os
    from tecogan_b200 import kernels as K
    from tests.conftest import GOLDEN
    g = np.load(os.path.join(GOLDEN, "ops.npz"))
    x, f, hr = torch.from_numpy(g["x"]), torch.from_numpy(g["f"]), torch.from_numpy(g["hr"])
    assert_close(K.bicubic4(dev(x)), torch.from_numpy(g["bicubic_four"]), 1e-5, what="bicubic_four")
    assert_close(K.upscale4(dev(f)), torch.from_numpy(g["upscale_four"]), 1e-5, what="upscale_four")
    assert_close(K.resize_bilinear(dev(f), f.shape[1] * 4, f.shape[2] * 4), torch.from_numpy(g["upscale_four"]), 1e-5)
    assert_close(K.gauss_down4(dev(hr)), torch.from_numpy(g["gauss_down"]), 1e-5, what="gauss_down")
    y = rnd(3, 2, 9, 7, 5)
    assert_close(K.resize_bilinear(dev(y), 18, 14), O.resize_bilinear_legacy(y, 18, 14), 1e-6, what="resize x2")
    assert_close(K.maxpool2(dev(y)), O.maxpool(y), 0.0, what="maxpool")
    assert_close(K.space_to_depth4(dev(rnd(4, 2, 8, 12, 3))), O.space_to_depth4(rnd(4, 2, 8, 12, 3)), 0.0, what="s2d")
    u = rnd(5, 3, 4, 5, lo=-0.2, hi=1.2)
    assert np.array_equal(K.to_u8(dev(u)).cpu().numpy(), O.save_img_u8(u))


def test_resample_gradients_match_oracle_autograd():
    from tecogan_b200 import kernels as K
    y = rnd(3, 2, 8, 6, 4)
    for ref_fn, got_fn, name in ((lambda t: O.resize_bilinear_legacy(t, 16, 12), lambda t: K.resize_bilinear(t, 16, 12), "resize"),
                                 (O.maxpool, K.maxpool2, "maxpool"), (O.space_to_depth4, K.space_to_depth4, "s2d"),
                                 (lambda t: O.resize_bilinear_legacy(t, 32, 24), lambda t: K.resize_bilinear(t, 32, 24), "x4")):
        _, _, g_ref, g_got = _grads(ref_fn, got_fn, [rnd(3, 2, 8, 8, 4) if name == "s2d" else y])
        assert_close(g_got[0], g_ref[0], 1e-5, what=name + " grad")


def test_batchnorm_and_gradients_match_oracle():
    from tecogan_b200 import kernels as K
    x, beta = rnd(1, 3, 8, 8, 64) * 3 + 1, rnd(2, 64)
    ref_fn = lambda a, b: O.lrelu(O.batchnorm_train(a, b))
    got_fn = lambda a, b: K.batchnorm_train(a, b, True)
    o_ref, o_got, g_ref, g_got = _grads(ref_fn, got_fn, [x, beta])
    assert_close(o_got, o_ref, 2e-5, what="bn")
    assert_close(g_got[0], g_ref[0], 2e-5, what="bn dx")
    assert_close(g_got[1], g_ref[1], 2e-4, what="bn dbeta")


def test_losses_and_gradients_match_oracle():
    from tecogan_b200 import kernels as K
    a, b = rnd(1, 4, 16, 16, 3), rnd(2, 4, 16, 16, 3)
    cases = [
        (lambda u, v: ((u - v) ** 2).sum(dim=3).mean(), K.loss_l2, "l2"),
        (lambda u, v: (u - v).abs().mean(), lambda u, v: K.loss_l1(u, v, False), "l1"),
        (lambda u, v: (u - v).abs().sum(dim=3).mean(), lambda u, v: K.loss_l1(u, v, True), "l1pp"),
    ]
    for ref_fn, got_fn, name in cases:
        ca, cb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        ga, gb = dev(a).requires_grad_(True), dev(b).requires_grad_(True)
        lr, lg = ref_fn(ca, cb), got_fn(ga, gb)
        assert abs(float(lr) - float(lg)) < 1e-5 * max(1.0, abs(float(lr))), name
        gr = torch.autograd.grad(lr * 1.7, [ca, cb])
        gg = torch.autograd.grad(lg * 1.7, [ga, gb])
        assert_close(gg[0], gr[0], 1e-7, 1e-4, what=name + " da")
        assert_close(gg[1], gr[1], 1e-7, 1e-4, what=name + " db")
    f, g = rnd(3, 2, 8, 8, 128, lo=0, hi=2), rnd(4, 2, 8, 8, 128, lo=0, hi=2)

    def cos_ref(u, v):
        un = u / torch.sqrt((u * u).sum(dim=3, keepdim=True) + 1e-12)
        vn = v / torch.sqrt((v * v).sum(dim=3, keepdim=True) + 1e-12)
        return 1.0 - (un * vn).sum(dim=3).mean()
    cf = f.clone().requires_grad_(True)
    gf = dev(f).requires_grad_(True)
    lr, lg = cos_ref(cf, g), K.loss_cosine(gf, dev(g))
    assert abs(float(lr) - float(lg)) < 1e-5
    assert_close(torch.autograd.grad(lg, gf)[0], torch.autograd.grad(lr, cf)[0], 1e-8, 1e-3, what="cosine df")
    df_, dr_ = rnd(5, 24, 8, 8, 1, lo=0.05, hi=0.95), rnd(6, 24, 8, 8, 1, lo=0.05, hi=0.95)
    cdf, cdr = df_.clone().requires_grad_(True), dr_.clone().requires_grad_(True)
    gdf, gdr = dev(df_).requires_grad_(True), dev(dr_).requires_grad_(True)
    out = K.loss_gan(gdf, gdr, 1e-12)
    adv = (-torch.log(cdf + 1e-12)).mean()
    dis = (-(torch.log(1 - cdf + 1e-12) + torch.log(cdr + 1e-12))).mean()
    ref = [adv, dis, torch.log(cdr + 1e-12).mean(), cdr.mean(), cdf.mean()]
    for i in range(5):
        assert abs(float(out[i]) - float(ref[i])) < 1e-5, i
    gr = torch.autograd.grad(0.3 * adv + 0.7 * dis, [cdf, cdr])
    gg = torch.autograd.grad(0.3 * out[0] + 0.7 * out[1], [gdf, gdr])
    assert_close(gg[0], gr[0], 1e-8, 1e-4, what="gan d_fake")
    assert_close(gg[1], gr[1], 1e-8, 1e-4, what="gan d_real")


def test_adam_matches_tf_formulation():
    from tecogan_b200 import kernels as K
    p, g = rnd(1, 1000), rnd(2, 1000)
    P = {"a": p.clone()}
    opt = O.TFAdam(["a"], P, lr=5e-5)
    dp, m, v = dev(p), torch.zeros(1000, device="cuda"), torch.zeros(1000, device="cuda")
    for t in range(1, 4):
        opt.apply(P, {"a": g * t})
        lr_t = 5e-5 * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
        K.adam_step(dp, m, v, dev(g * t), lr_t, 0.9, 0.999, 1e-8)
    assert_close(dp, P["a"], 1e-7, what="adam")


# ------------------------------------------------------------------------------------ wgmma kernel
def _bf(t):
    return t.to(torch.bfloat16).to(torch.float32)


def _p64(c):
    return (c + 63) // 64 * 64


def _xpad(x):
    """NHWC fp32 -> bf16 CUDA tensor with the channel count zero-padded to a multiple of 64 (the kernel's layout)."""
    n, h, w, c = x.shape
    out = torch.zeros(n, h, w, _p64(c), dtype=torch.bfloat16, device="cuda")
    out[..., :c] = x.cuda().to(torch.bfloat16)
    return out


# Error model of the float64 references of the bf16 training convolutions.  The products of bf16 operands are exact in fp32;
# each tensor-core K-step (16 products into the fp32 accumulator) and each later fp32 add (bias, residual, one atomicAdd of
# a tile's partial dW) is off by at most one fp32 ulp of the running sum -- 2^-23 of sum|terms|, twice the round-to-nearest
# bound, because the tensor cores' adder may truncate.  An fp32 result of S such steps is therefore within
# S * 2^-23 * sum|terms| of the exact value, where sum|terms| is the same operation evaluated on |operands|.  A result
# rounded to bf16 may in addition land on the neighbouring bf16 value: one bf16 ulp, at most 2^-7 of its magnitude.
_STEP = 2.0 ** -23
_BF_ULP = 2.0 ** -7


def _act64(act, z):
    return {0: lambda v: v, 1: torch.relu, 2: O.lrelu, 3: lambda v: torch.tanh(v) * 24}[act](z)


def _act_grad64(act, y):
    """act'(.) from the saved output y, as the backward pass computes it (LeakyReLU: y >= 0, like the forward's z >= 0)."""
    if act == 1:
        return (y > 0).double()
    if act == 2:
        return torch.where(y >= 0, torch.ones_like(y), torch.full_like(y, 0.2))
    if act == 3:
        return 24.0 * (1.0 - (y / 24.0) ** 2)
    return torch.ones_like(y)


def _bf_tie_ulp(v):
    """One bf16 ulp where v (float64) lies within 2^-20 |v| of a bf16 rounding midpoint, else 0: there the fp32 arithmetic
    of the kernel (a few fp32 roundings away from float64) may round v to either neighbour.  Zero for every element of a
    bf16-valued dy times 1 or 0.2, so it only matters for tanh."""
    ulp = torch.pow(2.0, torch.floor(torch.log2(v.abs().clamp_min(1e-30))) - 7)
    near = ((v - _bf(v).double()).abs() - ulp / 2).abs() <= 2.0 ** -20 * v.abs()
    return torch.where(near & (v != 0), ulp, torch.zeros_like(v))


def _lin_grads(op, a, b, g):
    """Gradients of <op(a, b), g> with respect to a and b, for op linear in each argument (float64 autograd)."""
    a, b = a.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    return torch.autograd.grad(op(a, b), (a, b), g)


def _train_ref(op, x, w, b, act, dy, y_saved, round_y=True, res=None):
    """float64 reference of one bf16 training convolution with the rounding points of kernels.py (_Conv3x3TC,
    _ConvTranspose2xTC): operands rounded to bf16, y = bf16(act(op(x, w) + b)) (+ res in fp32) -- or, for the narrow fp32
    output stage (round_y=False), act(op(x, w) + b) (+ res) unrounded -- dz = act'(y as saved) * dy, dzb = bf16(dz),
    dx = bf16(input-grad(dzb, w)), dw = weight-grad(x, dzb), db = sum(dz).  Each value comes with its sum|terms|; the dz
    ties of _bf_tie_ulp come with what they can move dx and dw by."""
    xb, wb, b64 = _bf(x).double(), _bf(w).double(), b.double()
    z = _act64(act, op(xb, wb) + b64)
    s_z = op(xb.abs(), wb.abs()) + b64.abs()
    y = _bf(z).double() if round_y else z
    if res is not None:
        y, s_z = y + res.double(), s_z + res.double().abs()
    dz = _act_grad64(act, y_saved.detach().double().cpu()) * dy.double()
    dzb, tie = _bf(dz).double(), _bf_tie_ulp(dz)
    dx, dw = _lin_grads(op, xb, wb, dzb)
    s_dx, s_dw = _lin_grads(op, xb.abs(), wb.abs(), dzb.abs())
    t_dx, t_dw = _lin_grads(op, xb.abs(), wb.abs(), tie) if bool(tie.any()) else (torch.zeros_like(xb), torch.zeros_like(wb))
    return dict(y=y, s_y=s_z, dx=_bf(dx).double(), s_dx=s_dx, t_dx=t_dx, dw=dw, s_dw=s_dw, t_dw=t_dw,
                db=dz.sum(dim=(0, 1, 2)), s_db=dz.abs().sum(dim=(0, 1, 2)))


def _wgrad_tiles(n, h, w):
    """Tiles of the weight-gradient kernel (8 x 16 pixels); each adds its partial dW to every element with one atomic."""
    return n * -(-h // 8) * -(-w // 16)


def _assert_within(got, ref, bound, what):
    assert got is not None, what + ": missing"
    got = got.detach().double().cpu()
    assert tuple(got.shape) == tuple(ref.shape), (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    bad = ~(err <= bound)
    i = int(torch.argmax(err / bound.clamp_min(1e-30)))
    assert not bad.any(), "%s: %d/%d elements outside the bound; max err %.3e; worst err/bound %.3e / %.3e" % (
        what, int(bad.sum()), bad.numel(), err.max().item(), err.flatten()[i].item(), bound.flatten()[i].item())


@pytest.mark.parametrize("n,h,w,cin,cout,act", [
    (1, 16, 8, 64, 64, 0), (1, 32, 32, 64, 64, 1), (2, 48, 40, 64, 64, 2), (1, 19, 21, 16, 32, 2), (1, 32, 32, 32, 64, 0),
    (1, 16, 16, 128, 256, 2), (1, 16, 24, 256, 128, 2), (1, 64, 64, 64, 16, 0), (1, 128, 128, 64, 64, 1), (3, 32, 32, 128, 128, 0),
    (2, 16, 16, 512, 512, 1), (1, 32, 32, 256, 512, 1), (4, 64, 64, 256, 256, 1), (24, 32, 32, 512, 512, 1), (2, 256, 256, 64, 64, 1),
])
def test_conv3x3_tc_matches_oracle_on_bf16_operands(n, h, w, cin, cout, act):
    from tecogan_b200 import kernels as K
    x, wt, b = _bf(rnd(1, n, h, w, cin)), _bf(rnd(2, 3, 3, cin, cout) * (2.0 / (9 * cin) ** 0.5)), rnd(3, cout) * 0.1
    acts = {0: lambda v: v, 1: torch.relu, 2: O.lrelu}
    ref = acts[act](O.conv2d(x, wt, b))
    wpk = K.packed_weight(dev(wt), _p64(cin), cout)
    got = K.conv3x3_tc(_xpad(x), wpk, dev(b), cout=cout, act=act)
    torch.cuda.synchronize()
    assert_close(got, ref, 2e-3, 1.0 / 128, what="conv3x3_tc")
    # residual add
    res = _bf(rnd(4, n, h, w, cout))
    got = K.conv3x3_tc(_xpad(x), wpk, dev(b), cout=cout, act=0, res=dev(res).to(torch.bfloat16))
    assert_close(got, O.conv2d(x, wt, b) + res, 2e-3, 1.0 / 128, what="conv3x3_tc+res")


def _lin_chain_reference(x, layers, plan):
    """The chain in the oracle, with the kernel's rounding points: bf16 activations between layers, fp32 inside a layer."""
    bufs = {0: x}
    for (wt, b), (i, o, r, act) in zip(layers, plan):
        y = O.conv2d(bufs[i], wt, b)
        y = torch.relu(y) if act == 1 else (O.lrelu(y) if act == 2 else y)
        if r >= 0:
            y = y + bufs[r]
        bufs[o] = _bf(y)
    return bufs


@pytest.mark.parametrize("n,h,plan", [
    (1, 32, [(0, 1, -1, 1)]),
    (3, 32, [(0, 1, -1, 0)]),
    (5, 32, [(0, 1, -1, 1), (1, 2, -1, 1), (2, 1, -1, 1), (1, 2, 2, 2)]),     # in-place residual on buf_b, LeakyReLU
    (2, 32, [(0, 1, -1, 1), (1, 2, -1, 1), (2, 1, 1, 0)]),                  # input conv + one residual block (in-place residual)
    (150, 32, [(0, 1, -1, 1), (1, 2, -1, 1), (2, 1, 1, 0), (1, 2, -1, 1), (2, 1, 1, 0)]),   # > 132 images: more images than SMs
    (7, 32, [(0, 1, -1, 1)] + [(1, 2, -1, 1), (2, 1, 1, 0)] * 4),            # 9 layers: the weight ring wraps
], ids=["relu", "linear", "inplace_res_lrelu_on_b", "res_block", "images_gt_sms", "nine_layers"])
def test_conv3x3_lin_chain_matches_oracle_on_bf16_operands(n, h, plan):
    """teco_conv3x3_lin_tc: the multi-layer chain on 32x32 images in one launch (each image owned by one cluster across
    layers)."""
    from tecogan_b200 import kernels as K
    L = len(plan)
    x = _bf(rnd(1, n, h, 32, 64))
    layers = [(_bf(rnd(10 + l, 3, 3, 64, 64) * (1.5 / 24.0)), rnd(50 + l, 64) * 0.1) for l in range(L)]
    ref = _lin_chain_reference(x, layers, plan)
    assert K.conv3x3_lin_in_smem(n, h, 32, plan) and not K.conv3x3_lin_in_smem(n, h, 40, plan)
    assert not K.conv3x3_lin_in_smem(n, 6, 32, plan)
    wall = torch.cat([K.packed_weight(dev(wt), 64, 64) for wt, _ in layers]).contiguous()
    ball = torch.cat([dev(b) for _, b in layers]).contiguous()
    a = torch.zeros(n, h, 32, 64, device="cuda", dtype=torch.bfloat16)
    bb = torch.zeros_like(a)
    K.conv3x3_lin_chain(dev(x).to(torch.bfloat16), a, bb, wall, ball, plan)
    torch.cuda.synchronize()
    final = plan[-1][1]
    got = a if final == 1 else bb
    # chained layers: each adds ~1 bf16 ulp of rounding noise that the next layers spread
    assert_close(got, ref[final], 2e-3 * L, 1.0 / 128 * (1 + 0.5 * (L - 1)), what="conv3x3_lin chain (%d layers)" % L)
    if L == 1:
        # a single layer is the same arithmetic as teco_conv3x3_tc up to the fp32 summation order
        other = K.conv3x3_tc(dev(x).to(torch.bfloat16), wall, ball, cout=64, act=plan[0][3])
        assert (got.float() - other.float()).abs().max().item() <= 2.0 ** -6 * max(1.0, got.float().abs().max().item())


def test_conv3x3_lin_chain_rejects_what_the_cluster_kernel_does_not_run():
    """teco_conv3x3_lin_tc runs conv3x3_trunk_cluster_kernel and nothing else: images other than 32x32 and plans that are
    not trunk-shaped (a residual from a buffer the chain has not written) raise ValueError before any launch."""
    from tecogan_b200 import kernels as K
    one = [(0, 1, -1, 1)]
    nine = [(0, 1, -1, 1)] + [(1, 2, -1, 1), (2, 1, 1, 0)] * 4
    external_res = [(0, 1, 2, 2)]
    for n, h, w, plan in ((1, 4, 32, one), (7, 12, 32, nine), (5, 8, 32, external_res), (5, 32, 32, external_res),
                          (1, 64, 32, one), (1, 32, 40, one), (2, 32, 32, [(0, 2, -1, 1)])):
        assert not K.conv3x3_lin_in_smem(n, h, w, plan), (n, h, w, plan)
        x = torch.zeros(n, h, w, 64, device="cuda", dtype=torch.bfloat16)
        a, bb = torch.zeros_like(x), torch.zeros_like(x)
        wall = torch.zeros(len(plan) * 9 * 64 * 64, device="cuda", dtype=torch.bfloat16)
        ball = torch.zeros(len(plan), 64, device="cuda")
        with pytest.raises(ValueError, match="teco_conv3x3_lin_tc"):
            K.conv3x3_lin_chain(x, a, bb, wall, ball, plan)


@pytest.mark.parametrize("n,h,w", [(1, 16, 8), (1, 32, 32), (2, 24, 20), (1, 64, 64), (5, 128, 128), (40, 64, 64), (3, 144, 120)])
def test_conv_transpose_tc_matches_oracle_on_bf16_operands(n, h, w):
    from tecogan_b200 import kernels as K
    x, wt, b = _bf(rnd(1, n, h, w, 64)), _bf(rnd(2, 3, 3, 64, 64) * 0.06), rnd(3, 64) * 0.1
    ref = torch.relu(O.conv2d_transpose(x, wt, b))
    wpk = K.packed_weight(dev(wt), 64, 64, transpose_layout=True)
    got = K.conv3x3_tc(dev(x).to(torch.bfloat16), wpk, dev(b), cout=64, act=K.ACT_RELU, mode=1)
    assert tuple(got.shape) == (n, 2 * h, 2 * w, 64)
    assert_close(got, ref, 2e-3, 1.0 / 128, what="conv_transpose_tc")


def test_conv3x3_tc_fp32_output_stage():
    from tecogan_b200 import kernels as K
    x, wt, b = _bf(rnd(1, 1, 40, 24, 64)), _bf(rnd(2, 3, 3, 64, 3) * 0.05), rnd(3, 3) * 0.1
    bic = rnd(4, 1, 40, 24, 3, lo=0, hi=1)
    ref = (O.conv2d(x, wt, b) + bic) * 2 - 1
    wpk = K.packed_weight(dev(wt), 64, 16)
    out = torch.zeros(1, 40, 24, 3, device="cuda")
    K.conv3x3_tc(dev(x).to(torch.bfloat16), wpk, K.pad_bias(dev(b), 16), cout=16, out_f32=out, res_f32=dev(bic), post=(2.0, -1.0))
    assert_close(out, ref, 1e-4, what="output stage")


def test_conv3x3_tc_fp32_output_stage_streaming_from_hbm():
    """The 64->3 output stage on an input larger than L2 (many tiles per persistent CTA); checked against
    the oracle on a few sampled images."""
    from tecogan_b200 import kernels as K
    n, h, w = 48, 128, 128                      # 48 x 128 x 128 x 64 ch bf16 = 100 MB
    g = torch.Generator().manual_seed(7)
    x = torch.rand(n, h, w, 64, generator=g).to(torch.bfloat16)
    wt, b = _bf(rnd(2, 3, 3, 64, 3) * 0.05), rnd(3, 3) * 0.1
    bic = torch.rand(n, h, w, 3, generator=g)
    wpk = K.packed_weight(dev(wt), 64, 16)
    out = torch.zeros(n, h, w, 3, device="cuda")
    K.conv3x3_tc(x.cuda(), wpk, K.pad_bias(dev(b), 16), cout=16, out_f32=out, res_f32=bic.cuda(), post=(2.0, -1.0))
    torch.cuda.synchronize()
    for i in (0, 17, 47):
        ref = (O.conv2d(x[i:i + 1].float(), wt, b) + bic[i:i + 1]) * 2 - 1
        assert_close(out[i:i + 1], ref, 1e-4, what="output stage image %d" % i)


@pytest.mark.parametrize("n,h,w,c", [(3, 128, 128, 3), (2, 144, 180, 3), (1, 512, 512, 3), (40, 32, 32, 2), (7, 48, 22, 4)])
def test_kx_fused_narrow_output_stage_matches_oracle(n, h, w, c):
    """Many-tile fp32 output stages (Cout padded to 16, fp32 output straight from the accumulators): every
    width class (multiple of the tile width or not), with and without the bicubic residual."""
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(11)
    x = torch.rand(n, h, w, 64, generator=g).to(torch.bfloat16)
    wt, b = _bf(rnd(2, 3, 3, 64, c) * 0.05), rnd(3, c) * 0.1
    bic = torch.rand(n, h, w, c, generator=g)
    wpk = K.packed_weight(dev(wt), 64, 16)
    out = torch.zeros(n, h, w, c, device="cuda")
    K.conv3x3_tc(x.cuda(), wpk, K.pad_bias(dev(b), 16), cout=16, out_f32=out, res_f32=bic.cuda(), post=(2.0, -1.0))
    ref = (O.conv2d(x[:2].float(), wt, b) + bic[:2]) * 2 - 1
    assert_close(out[:2], ref, 1e-4, what="narrow output stage")
    out2 = torch.zeros(n, h, w, c, device="cuda")
    K.conv3x3_tc(x.cuda(), wpk, K.pad_bias(dev(b), 16), cout=16, act=K.ACT_TANH24, out_f32=out2)
    ref2 = torch.tanh(O.conv2d(x[-1:].float(), wt, b)) * 24.0
    assert_close(out2[-1:], ref2, 2e-4, what="narrow tanh head")


@pytest.mark.parametrize("n,h,w,cin,cout", [
    (1, 8, 16, 64, 64), (4, 32, 32, 64, 64), (2, 19, 21, 51, 64), (3, 16, 24, 128, 32), (2, 32, 32, 32, 256),
    (2, 9, 40, 256, 64),            # the transposed conv's space-to-depth shape: four 64-channel input blocks
    (2, 13, 21, 64, 4),             # Cout rounded up to 4 (the narrow generator / FNet output layers)
    (3, 5, 7, 32, 64),              # smaller than one 8 x 16 tile in both directions
])
def test_conv3x3_wgrad_tc_matches_autograd_on_bf16_operands(n, h, w, cin, cout):
    """wgmma weight gradient (pixels as the GEMM K dimension, MN-major operands, one accumulator per tap) against float64
    autograd of the oracle convolution on the same bf16-rounded x and dz; ragged sizes exercise the zero-filled tile edges.
    Bound per element (error model above): 8 K-steps per tile plus one atomicAdd per tile, (8 + tiles) * 2^-23 * sum|x dz|
    -- with the initial |dw| added to sum|terms| when accumulating onto a non-zero dw.  db: fp32 sum over the pixels,
    npix * 2^-23 * sum|dz|."""
    from tecogan_b200 import kernels as K
    x, dz = _bf(rnd(1, n, h, w, cin)), _bf(rnd(2, n, h, w, cout))
    ref, _ = _lin_grads(lambda c, a: O.conv2d(a, c), torch.zeros(3, 3, cin, cout, dtype=torch.float64), x.double(), dz.double())
    s_ref, _ = _lin_grads(lambda c, a: O.conv2d(a, c), torch.zeros(3, 3, cin, cout, dtype=torch.float64), x.double().abs(),
                          dz.double().abs())
    gamma = (8 + _wgrad_tiles(n, h, w)) * _STEP
    dw = torch.full((3, 3, cin, cout), 7.0, device="cuda")
    K.conv3x3_wgrad_tc(_xpad(x), _xpad(dz), dw, cin, cout)
    _assert_within(dw, ref, gamma * s_ref, "wgrad")
    dw0 = rnd(3, 3, 3, cin, cout, lo=-2.0, hi=2.0) * s_ref.max().item()
    dw = dev(dw0)
    K.conv3x3_wgrad_tc(_xpad(x), _xpad(dz), dw, cin, cout, accumulate=True)
    _assert_within(dw, dw0.double() + ref, gamma * (s_ref + dw0.double().abs()), "wgrad accumulate")
    db = K.bias_grad(dev(dz))
    npix = n * h * w
    _assert_within(db, dz.double().sum(dim=(0, 1, 2)), npix * _STEP * dz.double().abs().sum(dim=(0, 1, 2)), "bias grad")


# ------------------------------------------------------------------------------------ bf16 training convolutions
# The tests below call y.grad_fn.apply(dy): the autograd Function's backward itself, so they see every gradient it returns,
# including the None it must return for an input that needs no gradient.
_RELU, _LRELU, _TANH24 = 1, 2, 3


@pytest.mark.parametrize("n,h,w,cin,cout,act,res,x_grad,w_grad", [
    (2, 19, 13, 51, 64, _RELU, False, False, True),       # generator input stage (LR frame + warped s2d; no dx)
    (1, 21, 30, 64, 64, _RELU, False, True, True),        # generator residual block, conv_1
    (2, 17, 9, 64, 64, 0, True, True, True),              # generator residual block, conv_2 + residual
    (2, 23, 18, 64, 3, 0, True, True, True),              # generator output conv + fp32 bicubic residual
    (1, 5, 3, 64, 3, 0, True, True, True),                #   ... on an image smaller than one tile
    (12, 67, 150, 64, 3, 0, True, True, True),            #   ... more tiles than the persistent grid has CTAs
    (2, 18, 20, 6, 32, _LRELU, False, False, True),       # fnet input (two LR frames; no dx)
    (1, 5, 3, 32, 32, _LRELU, False, True, True),
    (1, 9, 11, 128, 256, _LRELU, False, True, True),
    (1, 13, 7, 256, 128, _LRELU, False, True, True),
    (2, 18, 20, 64, 32, _LRELU, False, True, True),
    (2, 17, 25, 32, 2, _TANH24, False, True, True),       # fnet output: tanh * 24 (the flow), narrow fp32 output stage
    (1, 12, 10, 3, 64, _RELU, False, True, False),        # VGG19 conv1_1: frozen weights, dx only
    (1, 6, 5, 256, 512, _RELU, False, True, False),       # VGG19 conv4_1
    (1, 5, 3, 512, 512, _RELU, False, True, False),       # VGG19 conv4_2 .. conv5_4
    (2, 11, 14, 27, 64, _LRELU, False, True, True),       # discriminator input stage
])
def test_conv3x3_train_tc_matches_float64_reference(n, h, w, cin, cout, act, res, x_grad, w_grad):
    """conv3x3_train_tc (the bf16 training convolution behind conv2() and the VGG trunk): forward, input, weight, bias and
    residual gradients against _train_ref, per element.  Tolerances from the error model above:
      y (Cout >= 16, bf16)       one bf16 ulp + (9 Cin_pad/16 + 3) * 2^-23 * sum|terms|   (K-steps, bias, act, residual)
      y (Cout < 16, fp32)        L * (9 Cin_pad/16 + 3) * 2^-23 * sum|terms|, L = 24 for tanh * 24 (its slope bound), plus
                                 4 fp32 ulps of |y| for tanhf and the * 24
      dx (bf16)                  one bf16 ulp + (9 Cout_pad/16 + 1) * 2^-23 * sum|w dzb|
      dw (fp32)                  (8 + weight-gradient tiles) * 2^-23 * sum|x dzb|
      db (fp32)                  (npix + 8) * 2^-23 * sum|dz|
    plus, for dx and dw, what the dz elements on a bf16 rounding tie (_bf_tie_ulp) can move them by.  The residual
    gradient is dy itself."""
    from tecogan_b200 import kernels as K
    x = rnd(1, n, h, w, cin)
    wt = rnd(2, 3, 3, cin, cout) * (3.0 / (9 * cin)) ** 0.5
    b = rnd(3, cout) * 0.1
    r = rnd(4, n, h, w, cout) if res else None
    dy = _bf(rnd(5, n, h, w, cout))
    K.tc_cache_clear()
    xg, wg, bg = dev(x).requires_grad_(x_grad), dev(wt).requires_grad_(w_grad), dev(b).requires_grad_(w_grad)
    y = K.conv3x3_train_tc(xg, wg, bg, act, None if r is None else dev(r))
    dyg = dev(dy)
    dx, dw, db, _, dres = y.grad_fn.apply(dyg)
    torch.cuda.synchronize()
    narrow = cout < 16
    ref = _train_ref(O.conv2d, x, wt, b, act, dy, y, round_y=not narrow, res=r)

    steps_f = 9 * _p64(cin) // 16 + 3
    if narrow:
        lip = 24.0 if act == _TANH24 else 1.0
        bound_y = lip * steps_f * _STEP * ref["s_y"] + (4 * _STEP * ref["y"].abs() if act == _TANH24 else 0.0)
    else:
        bound_y = _BF_ULP * ref["y"].abs() + steps_f * _STEP * ref["s_y"]
    _assert_within(y, ref["y"], bound_y, "y")
    if x_grad:
        steps_d = 9 * _p64(cout) // 16 + 1
        _assert_within(dx, ref["dx"], _BF_ULP * ref["dx"].abs() + steps_d * _STEP * ref["s_dx"] + ref["t_dx"], "dx")
    else:
        assert dx is None, "dx computed for an input that needs no gradient"
    if w_grad:
        gamma_w = (8 + _wgrad_tiles(n, h, w)) * _STEP
        _assert_within(dw, ref["dw"], gamma_w * ref["s_dw"] + ref["t_dw"], "dw")
        _assert_within(db, ref["db"], (n * h * w + 8) * _STEP * ref["s_db"], "db")
    else:
        assert dw is None and db is None, "weight gradient computed for frozen weights"
    if res:
        assert dres is not None and torch.equal(dres, dyg), "the residual gradient is dy"
    else:
        assert dres is None


@pytest.mark.parametrize("act", [0, _RELU, _LRELU])
@pytest.mark.parametrize("n,h,w", [(1, 5, 7), (2, 9, 40), (3, 32, 32)])
def test_conv_transpose2x_train_tc_matches_float64_reference(n, h, w, act):
    """conv_transpose2x_train_tc (conv2_tran 64 -> 64, bf16 training): the 4-phase forward, and both gradients through the
    space-to-depth rewrite -- a 256-channel dz feeding the weight-streaming path of teco_conv3x3_tc (dx) and the shifted
    operand of teco_conv3x3_wgrad_tc (dw) -- against _train_ref with the float64 transposed convolution.  Tolerances from
    the error model above:
      y (bf16)    one bf16 ulp + (9 * 64/16 + 3) * 2^-23 * sum|terms|   (at most all nine taps per output phase)
      dx (bf16)   one bf16 ulp + (9 * 256/16 + 1) * 2^-23 * sum|w dzb|
      dw (fp32)   (8 + weight-gradient tiles of the LR grid) * 2^-23 * sum|x dzb|
      db (fp32)   (npix + 8) * 2^-23 * sum|dz| over the 2x output."""
    from tecogan_b200 import kernels as K
    x = rnd(1, n, h, w, 64)
    wt = rnd(2, 3, 3, 64, 64) * (3.0 / (4 * 64)) ** 0.5
    b = rnd(3, 64) * 0.1
    dy = _bf(rnd(5, n, 2 * h, 2 * w, 64))
    K.tc_cache_clear()
    xg, wg, bg = dev(x).requires_grad_(True), dev(wt).requires_grad_(True), dev(b).requires_grad_(True)
    y = K.conv_transpose2x_train_tc(xg, wg, bg, act)
    dx, dw, db, _ = y.grad_fn.apply(dev(dy))
    torch.cuda.synchronize()
    ref = _train_ref(O.conv2d_transpose, x, wt, b, act, dy, y)
    _assert_within(y, ref["y"], _BF_ULP * ref["y"].abs() + (9 * 64 // 16 + 3) * _STEP * ref["s_y"], "y")
    _assert_within(dx, ref["dx"], _BF_ULP * ref["dx"].abs() + (9 * 256 // 16 + 1) * _STEP * ref["s_dx"] + ref["t_dx"], "dx")
    _assert_within(dw, ref["dw"], (8 + _wgrad_tiles(n, h, w)) * _STEP * ref["s_dw"] + ref["t_dw"], "dw")
    _assert_within(db, ref["db"], (4 * n * h * w + 8) * _STEP * ref["s_db"], "db")


def _pack_ref(w, cin_pad, cout_pad, flags, cin_perm=None):
    """teco_pack_conv3x3_bf16 restated in numpy: w [3,3,cin,cout] ([3,3,cout,cin] with flag bit 0; taps flipped with bit 1)
    -> bf16 bits [cin_pad/64][tap][cout_pad][16-byte chunk j ^ (co & 7)][8]; packed input channel k reads cin_perm[k]
    (-1: zero).  bf16 rounding is torch's round-to-nearest-even."""
    w = np.asarray(w, dtype=np.float32)
    if flags & 1:
        w = w.transpose(0, 1, 3, 2)
    if flags & 2:
        w = w[::-1, ::-1]
    cin, cout = w.shape[2], w.shape[3]
    w = w.reshape(9, cin, cout)
    src = np.asarray(cin_perm if cin_perm is not None else [k if k < cin else -1 for k in range(cin_pad)])
    full = np.zeros((9, cin_pad, cout_pad), dtype=np.float32)
    ok = (src >= 0) & (src < cin)
    full[:, ok, :cout] = w[:, src[ok], :]
    bits = torch.from_numpy(full).to(torch.bfloat16).view(torch.int16).numpy()
    blk = bits.reshape(9, cin_pad // 64, 8, 8, cout_pad).transpose(1, 0, 4, 2, 3)    # [blk][tap][co][j][e]
    co = np.arange(cout_pad)[:, None]
    return blk[:, :, co, np.arange(8)[None, :] ^ (co & 7), :].reshape(-1)


@pytest.mark.parametrize("cin,cout,cin_pad,cout_pad,flags,perm", [
    (64, 64, 64, 64, 0, False), (51, 64, 64, 64, 0, True), (64, 3, 64, 16, 0, False), (6, 32, 64, 32, 0, False),
    (256, 512, 256, 512, 0, False), (64, 64, 64, 64, 1, False), (64, 64, 64, 64, 3, False), (2, 32, 64, 64, 3, False),
    (3, 64, 64, 64, 3, False), (128, 256, 128, 256, 3, False), (64, 3, 64, 64, 3, False),
])
def test_packed_weight_layout_is_bit_exact(cin, cout, cin_pad, cout_pad, flags, perm):
    """K.packed_weight bit for bit against the SWIZZLE_128B layout restated on the host: separates a packing error from a
    kernel error.  cin / cout are the packed (GEMM) channel counts; with flag bit 0 the weights are stored [3,3,cout,cin].
    Flag 3 is the input-gradient packing of _Conv3x3TC: the weights of a cout -> cin convolution with the taps flipped
    (fnet 32 -> 2, generator 64 -> 3, fnet 256 -> 128, VGG 3 -> 64 above)."""
    from tecogan_b200 import kernels as K
    from tecogan_b200.tc_nets import GEN_CIN_PERM
    shape = (3, 3, cout, cin) if flags & 1 else (3, 3, cin, cout)
    wt = rnd(9, *shape) * 3.0
    p = GEN_CIN_PERM if perm else None
    got = K.packed_weight(dev(wt), cin_pad, cout_pad, flags, cin_perm=p).view(torch.int16).cpu().numpy()
    ref = _pack_ref(wt.numpy(), cin_pad, cout_pad, flags, p)
    assert got.shape == ref.shape and np.array_equal(got, ref), int((got != ref).sum())


@pytest.mark.parametrize("c", [8, 64, 256])
def test_fnet_bf16_glue_kernels_match_oracle(c):
    """The bf16 glue of FNet inference, on bf16-valued inputs with odd sizes.  maxpool2_bf16 is a max, so bit-exact;
    resize2x_bf16 is the oracle's legacy bilinear x2 (weights 0 and 1/2) in fp32 rounded once to bf16 -- at most one bf16
    ulp apart if the association differs; f32_to_bf16_pad (round-to-nearest-even, a channel offset into a wider pitch, the
    other channels untouched) and bf16_to_f32 (a source pitch wider than C) are exact."""
    from tecogan_b200 import kernels as K
    x = _bf(rnd(1, 2, 9, 7, c))
    xb = dev(x).to(torch.bfloat16)
    got = K.maxpool2_bf16(xb)
    assert torch.equal(got.float().cpu(), O.maxpool(x)), "maxpool2_bf16"
    got = K.resize2x_bf16(xb).float().cpu()
    ref = _bf(O.resize_bilinear_legacy(x, 18, 14))
    assert (got - ref).abs().le(_BF_ULP * ref.abs()).all(), "resize2x_bf16: max err %.3e" % (got - ref).abs().max().item()
    src = rnd(2, 2, 5, 3, c) * 3.0
    dst = torch.full((2, 5, 3, c + 24), 7.0, device="cuda", dtype=torch.bfloat16)
    K.f32_to_bf16_pad(dev(src), dst, c, c_off=16, scale=0.5, shift=0.5)
    want = torch.full((2, 5, 3, c + 24), 7.0, dtype=torch.bfloat16)
    want[..., 16:16 + c] = (src * 0.5 + 0.5).to(torch.bfloat16)
    assert torch.equal(dst.cpu().view(torch.int16), want.view(torch.int16)), "f32_to_bf16_pad"
    back = K.bf16_to_f32(dst[..., 16:].contiguous(), c)
    assert torch.equal(back.cpu(), want[..., 16:16 + c].float()), "bf16_to_f32"


def test_abi_rejects_bad_arguments_with_valueerror():
    from tecogan_b200 import kernels as K
    with pytest.raises(ValueError):
        K.conv3x3_tc(torch.zeros(1, 8, 8, 48, device="cuda", dtype=torch.bfloat16),
                     torch.zeros(9 * 48 * 16, device="cuda", dtype=torch.bfloat16), None, cout=16)
    with pytest.raises(ValueError):
        K.dense_image_warp(torch.zeros(1, 8, 8, 3, device="cuda"), torch.zeros(1, 8, 7, 2, device="cuda"))
    with pytest.raises(ValueError):
        K.conv2d(torch.zeros(1, 8, 8, 3), torch.zeros(3, 3, 3, 4), None)  # CPU tensors: no CPU path
