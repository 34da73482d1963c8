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


@pytest.mark.parametrize("h,w,fh,fw,B", [(16, 16, 16, 16, 1), (18, 22, 16, 16, 2), (36, 45, 32, 40, 1)])
def test_fused_feedback_kernel_matches_oracle_composition(h, w, fh, fw, B):
    """upscale_four(4*pad_sym(flow_lr)) -> dense_image_warp(pre_gen) -> space_to_depth, main.py:201,212-215."""
    from tecogan_b200 import kernels as K
    pre_gen, flow_lr = rnd(1, B, 4 * h, 4 * w, 3, lo=0, hi=1), rnd(2, B, fh, fw, 2, lo=-6, hi=6)
    fl = O.upscale_four(O.pad_symmetric_br(flow_lr, h - fh, w - fw) * 4.0)
    warped = O.dense_image_warp(pre_gen, fl)
    ref = O.space_to_depth4(warped)
    dst = torch.zeros(B, h, w, 48, device="cuda")
    wout = torch.zeros(B, 4 * h, 4 * w, 3, device="cuda")
    K.warp_s2d_fused(dev(pre_gen), dev(flow_lr), dst, 0, warped_out=wout)
    assert_close(wout, warped, 2e-5, what="fused warp")
    assert_close(dst, ref, 2e-5, what="fused s2d")
    # bf16 destination inside a 64-channel packed buffer, reading [-1,1] data with the deprocess folded in
    dst16 = torch.zeros(B, h, w, 64, device="cuda", dtype=torch.bfloat16)
    K.warp_s2d_fused(dev(pre_gen * 2 - 1), dev(flow_lr), dst16, 0, in_scale=0.5, in_shift=0.5)
    assert_close(dst16[..., :48], ref, 5e-3, what="fused s2d bf16")
    assert float(dst16[..., 48:].abs().max()) == 0.0
    # unaligned channel offset (reference channel order: LR first) takes the scalar store path
    dst51 = torch.zeros(B, h, w, 51, device="cuda")
    K.warp_s2d_fused(dev(pre_gen), dev(flow_lr), dst51, 3)
    assert_close(dst51[..., 3:], ref, 2e-5, what="fused s2d @3")


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
    (1, 4, [(0, 1, -1, 1)]),                                               # one strip: every row is top and bottom padding
    (3, 32, [(0, 1, -1, 0)]),
    (5, 8, [(0, 1, 2, 2)]),                                                # external residual from buf_b, LeakyReLU
    (2, 32, [(0, 1, -1, 1), (1, 2, -1, 1), (2, 1, 1, 0)]),                  # input conv + one residual block (in-place residual)
    (150, 32, [(0, 1, -1, 1), (1, 2, -1, 1), (2, 1, 1, 0), (1, 2, -1, 1), (2, 1, 1, 0)]),   # > 132 images: more images than SMs
    (7, 12, [(0, 1, -1, 1)] + [(1, 2, -1, 1), (2, 1, 1, 0)] * 4),            # 9 layers: weight double buffer wraps
])
def test_conv3x3_lin_chain_matches_oracle_on_bf16_operands(n, h, plan):
    """teco_conv3x3_lin_tc: the multi-layer chain on 32-pixel-wide images in one launch (CTA-local images across layers)."""
    from tecogan_b200 import kernels as K
    L = len(plan)
    x = _bf(rnd(1, n, h, 32, 64))
    ext = _bf(rnd(5, n, h, 32, 64))                                         # initial content of buf_b (external residual case)
    layers = [(_bf(rnd(10 + l, 3, 3, 64, 64) * (1.5 / 24.0)), rnd(50 + l, 64) * 0.1) for l in range(L)]
    ref = _lin_chain_reference(x, layers, plan) if plan[0][2] < 0 else None
    if ref is None:                                                          # single layer with the external residual
        (wt, b), (_, _, _, act) = layers[0], plan[0]
        ref = {1: _bf(O.lrelu(O.conv2d(x, wt, b)) + ext)}
    assert K.conv3x3_lin_supported(n, h, 32, L) and not K.conv3x3_lin_supported(n, h, 40, L) and not K.conv3x3_lin_supported(n, 6, 32, L)
    wall = torch.cat([K.packed_weight(dev(wt), 64, 64) for wt, _ in layers]).contiguous()
    ball = torch.cat([dev(b) for _, b in layers]).contiguous()
    a = torch.zeros(n, h, 32, 64, device="cuda", dtype=torch.bfloat16)
    bb = dev(ext).to(torch.bfloat16)
    K.conv3x3_lin_chain(dev(x).to(torch.bfloat16), a, bb, wall, ball, plan)
    torch.cuda.synchronize()
    final = plan[-1][1]
    got = a if final == 1 else bb
    # chained layers: each adds ~1 bf16 ulp of rounding noise that the next layers spread
    assert_close(got, ref[final], 2e-3 * L, 1.0 / 128 * (1 + 0.5 * (L - 1)), what="conv3x3_lin chain (%d layers)" % L)
    if L == 1:
        # a single layer is the same arithmetic as teco_conv3x3_tc up to the fp32 summation order
        other = K.conv3x3_tc(dev(x).to(torch.bfloat16), wall, ball, cout=64, act=plan[0][3], res=dev(ext).to(torch.bfloat16) if plan[0][2] >= 0 else None)
        assert (got.float() - other.float()).abs().max().item() <= 2.0 ** -6 * max(1.0, got.float().abs().max().item())


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


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 8, 16, 64, 64), (4, 32, 32, 64, 64), (2, 19, 21, 51, 64), (3, 16, 24, 128, 32), (2, 32, 32, 32, 256)])
def test_conv3x3_wgrad_tc_matches_autograd_on_bf16_operands(n, h, w, cin, cout):
    """wgmma weight gradient (pixels as the GEMM K dimension, MN-major operands, one accumulator per tap) against torch autograd
    of the oracle convolution on the same bf16-rounded x and dz; ragged sizes exercise the zero-filled tile edges."""
    from tecogan_b200 import kernels as K
    x, dz = _bf(rnd(1, n, h, w, cin)), _bf(rnd(2, n, h, w, cout))
    wt = torch.zeros(3, 3, cin, cout, requires_grad=True)
    (O.conv2d(x, wt, None) * dz).sum().backward()
    ref = wt.grad
    dw = torch.full((3, 3, cin, cout), 7.0, device="cuda")
    K.conv3x3_wgrad_tc(_xpad(x), _xpad(dz), dw, cin, cout)
    scale = ref.abs().max().item()
    per_tap = [round((dw.cpu()[t // 3, t % 3] - ref[t // 3, t % 3]).abs().max().item() / scale, 4) for t in range(9)]
    assert max(per_tap) < 2e-3, per_tap
    K.conv3x3_wgrad_tc(_xpad(x), _xpad(dz), dw, cin, cout, accumulate=True)
    assert (dw.cpu() - 2 * ref).abs().max().item() < 4e-3 * scale
    db = K.bias_grad(dev(dz))
    assert (db.cpu() - dz.sum(dim=(0, 1, 2))).abs().max().item() < 1e-3 * dz.abs().sum().item() ** 0.5


def test_abi_rejects_bad_arguments_with_valueerror():
    from tecogan_b200 import kernels as K
    with pytest.raises(ValueError):
        K.conv3x3_tc(torch.zeros(1, 8, 8, 48, device="cuda", dtype=torch.bfloat16),
                     torch.zeros(9 * 48 * 16, device="cuda", dtype=torch.bfloat16), None, cout=16)
    with pytest.raises(ValueError):
        K.dense_image_warp(torch.zeros(1, 8, 8, 3, device="cuda"), torch.zeros(1, 8, 7, 2, device="cuda"))
    with pytest.raises(ValueError):
        K.conv2d(torch.zeros(1, 8, 8, 3), torch.zeros(3, 3, 3, 4), None)  # CPU tensors: no CPU path
