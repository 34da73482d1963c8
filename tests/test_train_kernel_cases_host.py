"""CPU: the case tables of tests/train_kernel_cases.py reach every launch-geometry branch and input edge they claim, the
float64 restatements the GPU test compares the training-step kernels with agree with independent statements of the same
maths (oracle/teco_oracle.py where it has one, torch float64 autograd of the textbook formula otherwise), and the guards
that make bit equality possible hold."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests import train_kernel_cases as T

f64 = torch.float64


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(f64).requires_grad_(grad)


def _close(got, exp, rtol=1e-12, atol=0.0):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    assert got.shape == exp.shape
    assert (np.abs(got - exp) <= atol + rtol * np.abs(exp)).all(), float(np.abs(got - exp).max())


@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_case_tables_reach_every_required_key(family):
    table, _ = T.FAMILIES[family]
    reached = set().union(*(T.keys(family, name) for name in table))
    assert T.REQUIRED[family] <= reached, sorted(T.REQUIRED[family] - reached)


def test_launch_geometry_restatements():
    assert T.elt_launch(1) == (1, 1) and T.elt_launch(257) == (2, 1)
    assert T.elt_launch(16 * 132 * 256) == (2112, 1) and T.elt_launch(16 * 132 * 256 + 1) == (2112, 2)
    assert T.elt_launch(4096, per_block=1024) == (4, 4)
    assert T.warp_launch(5) == (8, 1) and T.warp_launch(16 * 132 * 8 + 1) == (16896, 2)
    assert T.bn_launch(192) == (1, 192, False) and T.bn_launch(1025) == (2, 513, False)
    assert T.bn_launch(24 * 64 * 64) == (96, 1024, False)
    blocks, ppb, capped = T.bn_launch(2 * 132 * 1024 + 1025)
    assert capped and blocks <= 264 and blocks * ppb >= 2 * 132 * 1024 + 1025 > (blocks - 1) * ppb
    assert T.bias_launch(7, 2) == (1, 1024, False) and T.bias_launch(681, 3) == (2, 680, False)
    blocks, ppb, capped = T.bias_launch(16 * 132 * 8 + 9, 256)
    assert capped and blocks <= 2112 and blocks * ppb >= 16 * 132 * 8 + 9 > (blocks - 1) * ppb
    assert sum(v.numel() for v in O.init_generator().values()) == T.GENERATOR_FLAT
    for name, c in T.BN.items():                                   # the split covers every pixel once at other SM counts too
        for sms in (108, 114, 132, 144):
            blocks, ppb, _ = T.bn_launch(c.npix, sms)
            assert (blocks - 1) * ppb < c.npix <= blocks * ppb and blocks <= 2 * sms, (name, sms)


# ------------------------------------------------------------------------------------------------------- batch norm
@pytest.mark.parametrize("name", [n for n, c in T.BN.items() if c.npix <= 8192])
def test_batchnorm_restatement_matches_oracle_autograd(name):
    c = T.BN[name]
    x, beta, dy = T.bn_inputs(name)
    mean, var = T.bn_stats_ref(x)
    y, _ = T.bn_apply_ref(x, beta, mean, var, c.lrelu)
    tx, tb = _t(x.reshape(1, 1, c.npix, c.C), True), _t(beta, True)
    ty = O.batchnorm_train(tx, tb, eps=T.BN_EPS)
    if c.lrelu:
        ty = O.lrelu(ty, alpha=T.F02)
    _close(y, ty.detach().numpy().reshape(c.npix, c.C), 1e-11, 1e-12)
    gx, gb = torch.autograd.grad(ty, [tx, tb], _t(dy.reshape(1, 1, c.npix, c.C)))
    dx, dbeta, sg, _, _, _ = T.bn_bwd_ref(x, y, dy, mean, var, c.lrelu)
    _close(dbeta, gb.numpy(), 1e-11, 1e-12)
    # dx is a difference of terms of size rstd |g|: judge it on that scale
    _close(dx, gx.numpy().reshape(c.npix, c.C), 0.0, 1e-9 * (1 + np.abs(dy).max()) / np.sqrt(var.min() + T.BN_EPS))


@pytest.mark.parametrize("name", [n for n, c in T.BN.items() if c.kind != "cont"])
def test_batchnorm_dyadic_cases_hold_their_guards(name):
    T.bn_guard(name)
    c = T.BN[name]
    x, _, _ = T.bn_inputs(name)
    mean, var = T.bn_stats_ref(x)
    if c.kind == "offset":                                          # what a one-pass variance would have to hold exactly
        with pytest.raises(AssertionError):
            T.exact((x.astype(np.float64) ** 2).sum(0), 4, "sum x^2")
        assert mean.min() >= 99
    assert np.array_equal(mean.astype(np.float32).astype(np.float64), mean)


# ----------------------------------------------------------------------------------------------------------- losses
@pytest.mark.parametrize("name", [n for n, c in T.L2.items() if c.npix <= 4096])
def test_l2_restatements_match_autograd(name):
    c = T.L2[name]
    a, b = T.loss_inputs(T.L2, name)
    val, da, _ = T.l2_ref(a, b, c.gscale)
    ta, tb = _t(a, True), _t(b)
    loss = ((ta - tb) ** 2).sum(dim=1).mean()
    _close(val, loss.item())
    _close(da, torch.autograd.grad(loss * c.gscale, ta)[0].numpy(), 1e-12)
    _close(T.l2_da_f32(a, b, c.gscale), da, 4 * 2.0 ** -23)


@pytest.mark.parametrize("name", [n for n, c in T.L1.items() if c.npix <= 4096])
def test_l1_restatements_match_autograd(name):
    c = T.L1[name]
    a, b = T.loss_inputs(T.L1, name)
    val, da, _ = T.l1_ref(a, b, c.gscale, c.per_pixel)
    ta, tb = _t(a, True), _t(b)
    loss = (ta - tb).abs().sum(dim=1).mean() if c.per_pixel else (ta - tb).abs().mean()
    _close(val, loss.item())
    _close(da, torch.autograd.grad(loss * c.gscale, ta)[0].numpy(), 1e-12)       # torch: sign(0) = 0 too
    g32 = T.l1_da_f32(a, b, c.gscale, c.per_pixel)
    _close(g32, da, 4 * 2.0 ** -23)
    assert not np.signbit(g32[(a == b)]).any()                     # +0 at d = +-0


@pytest.mark.parametrize("table", [T.L2, T.L1], ids=["l2", "l1"])
def test_loss_cases_that_claim_exact_scalars_hold_their_guards(table):
    for name, c in table.items():
        if T.loss_scalar_exact(c):
            T.loss_guard(table, name)


@pytest.mark.parametrize("name", [n for n, c in T.COS.items() if c.npix * c.C <= 2 ** 20])
def test_cosine_restatement_matches_autograd(name):
    c = T.COS[name]
    f, g = T.cos_inputs(T.COS, name)
    val, df, A, mag = T.cos_ref(f, g, c.gscale)
    tf, tg = _t(f, True), _t(g)
    un = tf / torch.sqrt((tf * tf).sum(dim=1, keepdim=True) + T.EPS12)
    vn = tg / torch.sqrt((tg * tg).sum(dim=1, keepdim=True) + T.EPS12)
    loss = 1.0 - (un * vn).sum(dim=1).mean()
    _close(val, loss.item(), 1e-12, 1e-14)
    _close(df, torch.autograd.grad(loss * c.gscale, tf)[0].numpy(), 1e-9, 1e-12 * np.abs(df).max())
    assert (mag >= np.abs(df) * (1 - 1e-12)).all() and A <= 1 + 1e-12
    _close(T.l2norm_ref(f), un.detach().numpy(), 1e-12)
    zf = (f == 0).all(1)
    assert (T.l2norm_ref(f)[zf] == 0).all()


@pytest.mark.parametrize("name", [n for n, c in T.GAN.items() if c.n <= 4096])
def test_gan_restatements_match_autograd(name):
    """Away from the saturated edges (where f + eps in fp32 is not f + eps) the fp32-argument restatement equals the
    reference's expressions (lib/Teco.py:376, 394-399); at the edges the two differ only by the rounding of the sum."""
    c = T.GAN[name]
    f, r = T.gan_inputs(name)
    val, mag = T.gan_ref(f, r)
    tf, tr = _t(f, True), _t(r, True)
    adv = (-torch.log(tf + T.EPS12)).mean()
    dis = (-(torch.log(1 - tf + T.EPS12) + torch.log(tr + T.EPS12))).mean()
    ref = [adv.item(), dis.item(), torch.log(tr + T.EPS12).mean().item(), tr.mean().item(), tf.mean().item()]
    _close(val, np.array(ref), 1e-6, 1e-7 * mag.max())
    assert (mag >= np.abs(val) * (1 - 1e-12)).all()
    ga, = torch.autograd.grad(adv * c.s_adv, tf, retain_graph=True)
    gf, gr = torch.autograd.grad(dis * c.s_dis, [tf, tr])
    e_adv, e_f, e_r = T.gan_grads_ref(f, r, c.s_adv, c.s_dis)
    _close(e_adv, ga.numpy()), _close(e_f, gf.numpy()), _close(e_r, gr.numpy())
    # the fp32 chain: three roundings, plus the rounding of the eps-shifted argument (relative 2^-24 of it, except where
    # 1 - f or f is below 2^-24 and eps itself decides the value)
    for got, exp, arg in zip(T.gan_grads_f32(f, r, c.s_adv, c.s_dis), (e_adv, e_f, e_r), (f, 1 - f.astype(np.float64), r)):
        ok = np.abs(arg) > 1e-3
        _close(got[ok], exp[ok], 5 * 2.0 ** -23)
        assert np.isfinite(got).all()


# ------------------------------------------------------------------------------------------------------------- Adam
@pytest.mark.parametrize("name", [n for n, c in T.ADAM.items() if c.n <= 1000])
def test_adam_restatement_matches_tf_adam(name):
    c = T.ADAM[name]
    p, m, v, g = T.adam_inputs(name)
    s = float(np.float32(c.gscale))
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))       # the moments use the betas as the kernel gets them
    opt = O.TFAdam(["a"], {"a": _t(p)}, lr=5e-5, beta1=b1, beta2=b2, eps=float(np.float32(1e-8)))
    opt.m["a"], opt.v["a"], opt.t = _t(m), _t(v), 2
    P = {"a": _t(p)}
    opt.apply(P, {"a": _t(g) * s})
    m1, v1, _, _, step = T.adam_ref(p, m, v, g, c.gscale, lr_t=5e-5 * (1 - b2 ** 3) ** 0.5 / (1 - b1 ** 3))
    _close(m1, opt.m["a"].numpy(), 1e-12), _close(v1, opt.v["a"].numpy(), 1e-12)
    # lr_t reaches the kernel as an fp32 number: 2^-24 relative
    _close(p.astype(np.float64) - step(m1, v1), P["a"].numpy(), 0.0, 2.0 ** -23 * np.abs(step(m1, v1)).max() + 1e-18)
    still = (g == 0) & (m == 0) & (v == 0)
    assert (step(m1, v1)[still] == 0).all()


# ------------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("act", list(T.ACT_NAMES))
def test_activation_restatements_match_torch(act):
    x = T.act_x("n257")
    tx = _t(x, True)
    ty = {T.ACT_NONE: lambda t: t * 1.0, T.ACT_RELU: torch.relu, T.ACT_LRELU02: lambda t: O.lrelu(t, alpha=T.F02),
          T.ACT_TANH24: lambda t: torch.tanh(t) * 24.0, T.ACT_SIGMOID: torch.sigmoid}[act](tx)
    y = T.act_ref(x, act)
    _close(y, ty.detach().numpy(), 1e-12, 1e-300)
    # derivative on the saved output equals autograd's away from the kinks (at x = +-0 ReLU's is 0, LeakyReLU's 1)
    dy = T.rng("act host").uniform(-1, 1, x.size)
    gx, = torch.autograd.grad(ty, tx, _t(dy))
    kink = (x == 0) if act in (T.ACT_RELU, T.ACT_LRELU02) else np.zeros(x.size, bool)
    got = T.act_bwd_ref(y, dy, act) if act != T.ACT_TANH24 else dy * 24.0 * (1.0 - (y / 24.0) ** 2)
    _close(got[~kink], gx.numpy()[~kink], 1e-9, 1e-12)
    y32, g32 = T.act_bwd_inputs("n257", act)
    if act != T.ACT_TANH24:                                        # the fp32 chains the GPU test holds to equal bits
        _close(T.act_bwd_f32(y32, g32, act), T.act_bwd_ref(y32, g32, act), 3 * 2.0 ** -23, 1e-44)
    if act == T.ACT_RELU:
        assert (T.act_bwd_ref(y32, g32, act)[y32 == 0] == 0).all()
    if act == T.ACT_LRELU02:
        assert (T.act_bwd_ref(y32, g32, act)[y32 == 0] == g32[y32 == 0]).all()


# ------------------------------------------------------------------------------------- bias gradient and conversions
def test_bias_cases_hold_their_guards_and_ignore_the_pad_channels():
    for name, c in T.BIAS.items():
        if c.npix > 100000:
            continue
        T.bias_guard(name)
        dy, db0 = T.bias_inputs(name)
        ref, mag = T.bias_ref(dy, db0, c.C, c.accumulate)
        exp = _t(dy)[:, :c.C].sum(0) + (_t(db0) if c.accumulate else 0)
        _close(ref, exp.numpy(), 0.0)
        assert (mag < T.BIAS_PAD / 4).all()


def test_bf16_rounding_restatement_matches_torch_and_u8_matches_numpy():
    r = T.rng("bf16 host")
    v = T.bf16_midpoint_values(r, (4096,))
    low = v.view(np.uint32) & 0xFFFF
    assert (low == 0x8000).sum() > 500 and np.isfinite(v).all()
    got = T.bf16_rne_bits(v).view(np.int16)
    assert np.array_equal(got, torch.from_numpy(v).to(torch.bfloat16).view(torch.int16).numpy())
    b = T.bf16_values(r, (4096,))
    assert np.isfinite(b).all() and np.array_equal(torch.from_numpy(b).to(torch.bfloat16).float().numpy().view(np.int32), b.view(np.int32))
    x = T.u8_inputs()
    q = T.u8_ref(x)
    assert np.array_equal(q, np.clip(x * np.float32(255.0), 0, 255).astype(np.uint8))
    assert set(q.tolist()) == set(range(256))
