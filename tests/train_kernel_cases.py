"""Case tables of tests/test_gpu_train_kernels_exact.py, their seeded inputs, float64 restatements of the training-step
kernels as they state their arithmetic (csrc/eltwise.cu, bias_grad_kernel of csrc/conv_simt.cu; formulas in
include/teco.h), and a host restatement of the launch geometry and the edges each case reaches.

Inputs that claim bit equality sit on dyadic grids; `exact(a, e, what)` asserts that values are multiples of 2^-e and
smaller than 2^24 of those units, so they are fp32 numbers.  For a reduction the guard is applied to the sum of the
absolute values of the terms: every partial sum is then an fp32 number too, whatever order the per-thread loops, the
block trees and the atomics add them in, and whether or not the compiler contracted a multiply into the add.

`keys(family, name, sms)` classifies a case at 132 SMs (H100 SXM); the GPU test recomputes it from the device's SM
count.  tests/test_train_kernel_cases_host.py checks that every family reaches every key of REQUIRED, that the
restatements agree with independent statements of the same maths, and that the guards hold.

Launch geometry restated here:
  grid_for(n, per_block)  blocks = clamp(ceil(n / per_block), 1, 16 SMs), 256 threads each, grid-stride loop.  The
                          elementwise kernels use per_block = 256, the loss reductions 1024, the warp-per-pixel kernels
                          (cosine, l2norm) n = 32 npix.
  batch-norm split        blocks = min(ceil(npix / 1024), 2 SMs); ppb = ceil(npix / blocks); blocks = ceil(npix / ppb);
                          256 / C pixel lanes per block, threads with lane >= 256 / C idle.
  bias-gradient split     ppb = 8 (256 / C); blocks = ceil(npix / ppb); above 16 SMs blocks, ppb and blocks are recomputed
                          as for batch-norm.
"""
from collections import namedtuple

import numpy as np

from tests.resample_cases import bf16_rne_bits, grid, rng, uniform  # noqa: F401  (re-exported to the tests)

TPB = 256
U = 2.0 ** -24                                    # unit roundoff of fp32
EPS12 = float(np.float32(1e-12))                  # the 1e-12f of the cosine / l2norm kernels and FLAGS.EPS as the ABI gets it
BN_EPS = float(np.float32(1e-3))
ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_TANH24, ACT_SIGMOID = 0, 1, 2, 3, 4
F02 = float(np.float32(0.2))                      # the kernels' 0.2f
INV24 = float(np.float32(1.0) / np.float32(24.0))  # their 1.0f / 24.0f


def exact(a, e, what):
    """Every value of `a` is a multiple of 2^-e and smaller than 2^24 of those units: representable in fp32."""
    s = np.asarray(a, np.float64) * 2.0 ** e
    assert np.array_equal(s, np.round(s)), "%s: off the 2^-%d grid" % (what, e)
    assert np.abs(s).max(initial=0) < 2 ** 24, "%s: %g units of 2^-%d do not fit 24 bits" % (what, np.abs(s).max(), e)


def _cdiv(a, b):
    return -(-a // b)


def pow2(n):
    return n & (n - 1) == 0


def elt_launch(n, sms=132, per_block=TPB):
    """(blocks, grid-stride passes) of grid_for(n, per_block)."""
    blocks = max(1, min(_cdiv(n, per_block), 16 * sms))
    return blocks, _cdiv(n, blocks * TPB)


def warp_launch(npix, sms=132):
    """(warps in the grid, pixels the busiest warp takes) of the warp-per-pixel kernels."""
    warps = elt_launch(32 * npix, sms)[0] * (TPB // 32)
    return warps, _cdiv(npix, warps)


def bn_launch(npix, sms=132):
    """(blocks, pixels per block, capped) of the batch-norm statistics kernels."""
    blocks = _cdiv(npix, 1024)
    capped = blocks > 2 * sms
    blocks = min(blocks, 2 * sms)
    ppb = _cdiv(npix, blocks)
    return _cdiv(npix, ppb), ppb, capped


def bias_launch(npix, C, sms=132):
    """(blocks, pixels per block, capped) of bias_grad_kernel."""
    ppb = 8 * (256 // C)
    blocks = _cdiv(npix, ppb)
    capped = blocks > 16 * sms
    if capped:
        ppb = _cdiv(npix, 16 * sms)
        blocks = _cdiv(npix, ppb)
    return blocks, ppb, capped


def split_steps(blocks, ppb, C):
    """Additions the longest chain of a split per-channel reduction makes: a thread's serial loop over its pixels, the
    block's 256 / C lanes, and one atomic per lane (batch-norm) or per block (bias gradient) -- bounded by the former."""
    ppar = 256 // C
    return _cdiv(ppb, ppar) + ppar * blocks


def reduce_steps(n, sms, per_block=1024):
    """Additions on the longest chain of a loss scalar: grid-stride passes, warp and block trees (5 + 5), the scaling by
    1 / n, one atomic per block."""
    blocks, passes = elt_launch(n, sms, per_block)
    return passes + 11 + blocks


def _elt_keys(n, sms, per_block=TPB):
    k = set()
    k |= {"eltwise: >1 grid-stride pass"} if elt_launch(n, sms, per_block)[1] > 1 else set()
    k |= {"eltwise: n%256!=0"} if n % TPB else set()
    k |= {"eltwise: n==1"} if n == 1 else set()
    return k


# ------------------------------------------------------------------------------------------------------- batch norm
# kind: "dyadic"  x = m_c + d on the 2^-2 grid with the d of each channel summing to zero (pairs +-d, |d| <= 2), so the
#                 mean is m_c and sum d^2 / npix one correctly rounded division: stats are exact at any npix
#       "offset"  the same around m_c = 100 + ...: sum x^2 does not fit fp32, a one-pass variance cannot be exact
#       "cont"    continuous inputs, held to bounds
# The discriminator's layers at batch 4, RNN_N 10 with ping-pong (24 triplets): 24 x 64 x 64 x 64, 24 x 32 x 32 x 64,
# 24 x 16 x 16 x 128, 24 x 8 x 8 x 256.
Bn = namedtuple("Bn", "npix C lrelu kind")
BN = {
    "1px_c1": Bn(1, 1, 1, "dyadic"),
    "192px_c64": Bn(192, 64, 1, "dyadic"),
    "192px_c3_nolrelu": Bn(192, 3, 0, "dyadic"),
    "1024px_c48": Bn(1024, 48, 1, "dyadic"),
    "1025px_c100": Bn(1025, 100, 0, "dyadic"),
    "1025px_c128": Bn(1025, 128, 1, "dyadic"),
    "8192px_c64_offset100": Bn(8192, 64, 1, "offset"),
    "disc_24x64x64_c64": Bn(24 * 64 * 64, 64, 1, "dyadic"),
    "disc_24x32x32_c64": Bn(24 * 32 * 32, 64, 1, "dyadic"),
    "disc_24x16x16_c128": Bn(24 * 16 * 16, 128, 1, "dyadic"),
    "disc_24x8x8_c256": Bn(24 * 8 * 8, 256, 1, "dyadic"),
    "capped_c3_nolrelu": Bn(2 * 132 * 1024 + 1025, 3, 0, "dyadic"),
    "1000px_c100_cont": Bn(1000, 100, 1, "cont"),
    "3001px_c256_cont_nolrelu": Bn(3001, 256, 0, "cont"),
}


def bn_inputs(name):
    """x [npix, C], beta [C] (2^-3 grid, every third channel 0), dy [npix, C] (2^-4 grid)."""
    c, r = BN[name], rng("bn " + name)
    if c.kind == "cont":
        x = (r.standard_normal((c.npix, c.C)) * 3 + 1).astype(np.float32)
        return x, r.uniform(-1, 1, c.C).astype(np.float32), r.uniform(-1, 1, (c.npix, c.C)).astype(np.float32)
    half = c.npix // 2
    d = r.randint(-8, 9, (half, c.C)) / 4.0
    d = np.concatenate((d, -d, np.zeros((c.npix - 2 * half, c.C))))[r.permutation(c.npix)]
    m = r.randint(-4, 5, c.C) / 4.0 + (100.0 if c.kind == "offset" else 0.0)
    beta = uniform(r, (c.C,), 3)
    beta[::3] = 0
    return (m + d).astype(np.float32), beta, uniform(r, (c.npix, c.C), 4)


def bn_stats_ref(x):
    """float64 mean and biased two-pass variance per channel."""
    x = x.astype(np.float64)
    mean = x.mean(0)
    return mean, ((x - mean) ** 2).mean(0)


def bn_apply_ref(x, beta, mean, var, lrelu):
    """y = (x - mean) rsqrt(var + eps) + beta (+ LeakyReLU 0.2 on v >= 0) from given statistics; also xhat."""
    xhat = (x.astype(np.float64) - mean) / np.sqrt(var + BN_EPS)
    v = xhat + beta.astype(np.float64)
    return (np.where(v >= 0, v, F02 * v) if lrelu else v), xhat


def bn_bwd_ref(x, y, dy, mean, var, lrelu):
    """g = dy (y < 0 ? 0.2 : 1); dbeta = sum g; dx = rstd (g - mean(g) - xhat mean(g xhat)).  Returns dx, dbeta,
    sum |g|, sum |g xhat|, g, xhat."""
    rstd = 1.0 / np.sqrt(var + BN_EPS)
    xhat = (x.astype(np.float64) - mean) * rstd
    g = dy.astype(np.float64)
    if lrelu:
        g = np.where(y < 0, F02 * g, g)
    n = x.shape[0]
    dx = rstd * (g - g.sum(0) / n - xhat * ((g * xhat).sum(0) / n))
    return dx, g.sum(0), np.abs(g).sum(0), np.abs(g * xhat).sum(0), g, xhat


def bn_guard(name):
    """The dyadic cases: x, the deviations and their squares, and every partial sum of them, are fp32 numbers."""
    c = BN[name]
    x, beta, dy = bn_inputs(name)
    mean, _ = bn_stats_ref(x)
    exact(x, 2, name + " x"), exact(np.abs(x).sum(0), 2, name + " sum |x|")
    exact(mean, 2, name + " mean")
    d = x.astype(np.float64) - mean
    exact((d * d).sum(0), 4, name + " sum (x - mean)^2")
    exact(np.abs(dy).sum(0), 4, name + " sum |dy|")
    assert c.npix < 2 ** 24


def _bn_keys(name, sms):
    c = BN[name]
    x, beta, _ = bn_inputs(name)
    blocks, ppb, capped = bn_launch(c.npix, sms)
    k = {"bn: lrelu" if c.lrelu else "bn: no lrelu", "bn: one block" if blocks == 1 else "bn: multi block"}
    k |= {"bn: last block short"} if c.npix % ppb else set()
    k |= {"bn: blocks capped"} if capped else set()
    k |= {"bn: C∤256"} if 256 % c.C else set()
    k |= {"bn: ppar==%d" % (256 // c.C)} if c.C >= 128 else set()
    k |= {"bn: npix==1"} if c.npix == 1 else set()
    k |= {"bn: npix not 2^k"} if not pow2(c.npix) else set()
    k |= {"bn: mean far from zero"} if c.kind == "offset" else set()
    k |= {"bn: continuous"} if c.kind == "cont" else set()
    k |= {"bn: disc layer"} if name.startswith("disc_") else set()
    k |= {"bn: apply >1 grid-stride pass"} if elt_launch(c.npix * c.C, sms)[1] > 1 else set()
    if c.kind != "cont":
        mean, var = bn_stats_ref(x)
        y, _ = bn_apply_ref(x, beta, mean, var, c.lrelu)
        k |= {"bn: y==0"} if (y == 0).any() else set()
    return k


# --------------------------------------------------------------------------------------------------- L2 / L1 losses
# kind: "dyadic" a, b on the 2^-4 grid in [-1, 1]; "coarse" on {-1/2, 0, 1/2} (the multi-pass cases: sum d^2 must fit);
# "cont" continuous.  Every seventh element has a == b, and element 3 has a = -0, b = +0 (d = -0).  The L2 loss is always
# a mean over pixels (per_pixel = 1).
Loss = namedtuple("Loss", "npix C gscale kind per_pixel")
L2 = {
    "1px_c3": Loss(1, 3, 1.0, "dyadic", 1),
    "4x16x16_c3_gs": Loss(1024, 3, 0.25, "dyadic", 1),
    "content_64x128x128_c3": Loss(2 ** 20, 3, 1.0, "coarse", 1),
    "1001px_c3_cont": Loss(1001, 3, 1.0 / 3.0, "cont", 1),
}
L1 = {
    "1px_c1": Loss(1, 1, 1.0, "dyadic", 0),
    "pingpong_4096px_c4_gs": Loss(4096, 4, 0.5, "dyadic", 0),
    "layer_2048px_c64_per_pixel": Loss(2048, 64, 1.0, "dyadic", 1),
    "multi_pass_c3_per_pixel": Loss(2 ** 18, 3, 0.25, "coarse", 1),
    "1001px_c3_cont": Loss(1001, 3, 1.0 / 3.0, "cont", 0),
}


def loss_inputs(table, name):
    c, r = table[name], rng("loss " + name)
    sh = (c.npix, c.C)
    if c.kind == "cont":
        a, b = r.uniform(-1, 1, sh).astype(np.float32), r.uniform(-1, 1, sh).astype(np.float32)
    elif c.kind == "coarse":
        a, b = (r.randint(-1, 2, sh) / 2.0).astype(np.float32), (r.randint(-1, 2, sh) / 2.0).astype(np.float32)
    else:
        a, b = uniform(r, sh, 4), uniform(r, sh, 4)
    a, b = a.ravel(), b.ravel()
    a[::7] = b[::7]
    if a.size > 3:
        a[3], b[3] = -0.0, 0.0
    return a.reshape(sh), b.reshape(sh)


def loss_den(c):
    return c.npix if c.per_pixel else c.npix * c.C


def loss_scalar_exact(c):
    return c.kind != "cont" and pow2(loss_den(c))


def l2_ref(a, b, gscale):
    """mean over pixels of sum_c (a - b)^2 and d(gscale loss) / da = 2 d gscale / npix; also sum d^2."""
    d = a.astype(np.float64) - b.astype(np.float64)
    return (d * d).sum() / a.shape[0], 2.0 * d * gscale / a.shape[0], (d * d).sum()


def l2_da_f32(a, b, gscale):
    """The kernel's fp32 chain 2.f * d * inv_npix * gscale, left to right (no multiply-add in it to contract)."""
    inv = np.float32(1.0) / np.float32(a.shape[0])
    return ((np.float32(2.0) * (a - b)) * inv) * np.float32(gscale)


def l1_ref(a, b, gscale, per_pixel):
    d = a.astype(np.float64) - b.astype(np.float64)
    den = a.shape[0] if per_pixel else a.size
    return np.abs(d).sum() / den, np.sign(d) * gscale / den, np.abs(d).sum()


def l1_da_f32(a, b, gscale, per_pixel):
    """sign(d) * inv_den * gscale in fp32, sign(+-0) = 0; inv_den = 1 / npix or 1 / ((float)npix * (float)C)."""
    n, C = a.shape
    inv = np.float32(1.0) / (np.float32(n) if per_pixel else np.float32(n) * np.float32(C))
    d = a - b
    s = np.where(d > 0, np.float32(1), np.where(d < 0, np.float32(-1), np.float32(0))).astype(np.float32)
    return (s * inv) * np.float32(gscale)


def loss_guard(table, name):
    c = table[name]
    a, b = loss_inputs(table, name)
    d = a.astype(np.float64) - b.astype(np.float64)
    e = 1 if c.kind == "coarse" else 4
    exact(d, e, name + " d")
    exact((d * d).sum() if table is L2 else np.abs(d).sum(), 2 * e if table is L2 else e, name + " sum of terms")


def _loss_keys(table):
    def f(name, sms):
        c = table[name]
        a, b = loss_inputs(table, name)
        d = a - b
        fam = "l2" if table is L2 else "l1"
        k = _elt_keys(a.size, sms, 4 * TPB)
        k |= {fam + ": d==0"} if (d == 0).any() else set()
        k |= {fam + ": d==-0"} if ((d == 0) & np.signbit(d)).any() else set()
        k |= {fam + ": gscale!=1"} if c.gscale != 1 else set()
        k |= {fam + ": per_pixel"} if c.per_pixel else set()
        k |= {fam + ": exact scalar"} if loss_scalar_exact(c) else {fam + ": bounded scalar"}
        k |= {fam + ": blocks capped"} if _cdiv(a.size, 4 * TPB) > 16 * sms else set()
        return k
    return f


# ---------------------------------------------------------------------------------------- cosine loss / channel L2 norm
# Post-ReLU features (about half the elements 0), f twice and g half the scale; from pixel 1 on, every fourth pixel has
# f = 0, the next g = 0, and every eighth both.
Cos = namedtuple("Cos", "npix C gscale df_null")
COS = {
    "1px_c3": Cos(1, 3, 1.0, 0),
    "5px_c48_gs": Cos(5, 48, 0.5, 0),
    "5px_c64_nodf": Cos(5, 64, 1.0, 1),
    "5px_c512": Cos(5, 512, 1.0, 0),
    "76x8x8_c128": Cos(76 * 8 * 8, 128, 1.0, 0),
    "76x8x8_c256_gs": Cos(76 * 8 * 8, 256, 1.0 / 3.0, 0),
    "above_warps_c64": Cos(16 * 132 * 8 + 77, 64, 1.0, 0),
}
L2NORM = {
    "1px_c3": Cos(1, 3, 1.0, 0),
    "5px_c64": Cos(5, 64, 1.0, 0),
    "76x8x8_c128": Cos(76 * 8 * 8, 128, 1.0, 0),
    "7px_c256": Cos(7, 256, 1.0, 0),
    "9px_c512": Cos(9, 512, 1.0, 0),
    "above_warps_c64": Cos(16 * 132 * 8 + 77, 64, 1.0, 0),
}


def cos_inputs(table, name):
    c, r = table[name], rng("cos " + name)
    f = (2.0 * np.maximum(r.standard_normal((c.npix, c.C)), 0)).astype(np.float32)
    g = (0.5 * np.maximum(r.standard_normal((c.npix, c.C)), 0)).astype(np.float32)
    f[:, 0] += np.float32(0.5)                                # no accidental all-zero pixel at C = 3
    g[:, 0] += np.float32(0.25)
    p = np.arange(c.npix)
    f[(p % 4 == 1) | (p % 8 == 3)] = 0
    g[(p % 4 == 2) | (p % 8 == 3)] = 0
    return f, g


def cos_ref(f, g, gscale):
    """1 - mean_p <f, g> / (nf ng), nf = sqrt(|f|^2 + 1e-12f), and d(gscale loss) / df = k1 g + k2 f with
    k1 = -gscale / (npix nf ng), k2 = gscale cos / (npix nf^2).  Also per pixel A = sum |f g| / (nf ng) >= |cos| and the
    magnitudes |k1 g| and (A gscale / (npix nf^2)) |f| the gradient bound is stated in."""
    f, g = f.astype(np.float64), g.astype(np.float64)
    n = f.shape[0]
    nf, ng = np.sqrt((f * f).sum(1) + EPS12), np.sqrt((g * g).sum(1) + EPS12)
    cosv = (f * g).sum(1) / (nf * ng)
    A = np.abs(f * g).sum(1) / (nf * ng)
    k1, k2 = -gscale / (n * nf * ng), gscale * cosv / (n * nf * nf)
    df = k1[:, None] * g + k2[:, None] * f
    mag = np.abs(k1[:, None] * g) + (gscale * A / (n * nf * nf))[:, None] * np.abs(f)
    return 1.0 - cosv.mean(), df, A.mean(), mag


def l2norm_ref(f):
    f = f.astype(np.float64)
    return f / np.sqrt((f * f).sum(1, keepdims=True) + EPS12)


def _cos_keys(table):
    def f(name, sms):
        c = table[name]
        ft, gt = cos_inputs(table, name)
        zf, zg = (ft == 0).all(1), (gt == 0).all(1)
        fam = "cos" if table is COS else "l2norm"
        k = {fam + ": C=%d" % c.C}
        k |= {fam + ": zero f"} if (zf & ~zg).any() else set()
        k |= {fam + ": C%32!=0"} if c.C % 32 else set()
        k |= {fam + ": >1 pixel per warp"} if warp_launch(c.npix, sms)[1] > 1 else set()
        k |= {fam + ": npix==1"} if c.npix == 1 else set()
        if table is COS:
            k |= {"cos: zero g"} if (zg & ~zf).any() else set()
            k |= {"cos: zero f and g"} if (zf & zg).any() else set()
            k |= {"cos: df NULL"} if c.df_null else set()
            k |= {"cos: gscale!=1"} if c.gscale != 1 else set()
        return k
    return f


# --------------------------------------------------------------------------------------------------------- GAN loss
# null: which gradient pointers are NULL.  The first elements of d_fake and elements 7.. of d_real hold GAN_EDGES.
Gan = namedtuple("Gan", "n s_adv s_dis null")
GAN = {
    "n1": Gan(1, 1.0, 1.0, ()),
    "edges_n300_scaled": Gan(300, 0.5, 0.25, ()),
    "disc_24x8x8x1": Gan(24 * 8 * 8, 1.0, 1.0, ()),
    "n300_no_adv": Gan(300, 1.0, 1.0, ("adv",)),
    "n300_no_dis_f": Gan(300, 1.0, 0.5, ("dis_f",)),
    "n300_no_dis_r": Gan(300, 0.5, 1.0, ("dis_r",)),
    "n300_value_only": Gan(300, 1.0, 1.0, ("adv", "dis_f", "dis_r")),
    "multi_pass_n100001": Gan(100001, 1.0, 1.0, ()),
}
GAN_EDGES = np.float32([0.0, 1.0, 2.0 ** -24, 1.0 - 2.0 ** -24, 1e-45, 1.0 - 2.0 ** -23, 0.5])


def gan_inputs(name):
    c, r = GAN[name], rng("gan " + name)
    f, rl = r.uniform(0.05, 0.95, c.n).astype(np.float32), r.uniform(0.05, 0.95, c.n).astype(np.float32)
    f[:7] = GAN_EDGES[:c.n]
    rl[7:14] = GAN_EDGES[:max(0, min(7, c.n - 7))]
    return f, rl


def gan_fp32_arguments(f, r):
    """The fp32 values the kernel takes logarithms and reciprocals of: f + eps, (1 - f) + eps, r + eps."""
    e = np.float32(EPS12)
    return f + e, (np.float32(1) - f) + e, r + e


def gan_ref(f, r):
    """The five means in float64 from the fp32 arguments, and per scalar the mean of |terms|."""
    fe, f1e, re = (v.astype(np.float64) for v in gan_fp32_arguments(f, r))
    lf, l1f, lr = np.log(fe), np.log(f1e), np.log(re)
    val = np.array([(-lf).mean(), (-(l1f + lr)).mean(), lr.mean(), r.astype(np.float64).mean(), f.astype(np.float64).mean()])
    mag = np.array([np.abs(lf).mean(), (np.abs(l1f) + np.abs(lr)).mean(), np.abs(lr).mean(), np.abs(r).mean(dtype=np.float64),
                    np.abs(f).mean(dtype=np.float64)])
    return val, mag


def gan_grads_f32(f, r, s_adv, s_dis):
    """-inv s_adv / (f + eps), inv s_dis / (1 - f + eps), -inv s_dis / (r + eps) as the kernel's fp32 chain (IEEE
    multiplies and divisions, nothing to contract)."""
    fe, f1e, re = gan_fp32_arguments(f, r)
    inv = np.float32(1.0) / np.float32(f.size)
    return (-inv * np.float32(s_adv)) / fe, (inv * np.float32(s_dis)) / f1e, (-inv * np.float32(s_dis)) / re


def gan_grads_ref(f, r, s_adv, s_dis):
    """d(s_adv out0) / df, d(s_dis out1) / df, d(s_dis out1) / dr in float64 at the exact (not eps-shifted) formulas'
    arguments f + eps, 1 - f + eps, r + eps."""
    f, r, n = f.astype(np.float64), r.astype(np.float64), f.size
    return -s_adv / (n * (f + EPS12)), s_dis / (n * (1 - f + EPS12)), -s_dis / (n * (r + EPS12))


def _gan_keys(name, sms):
    c = GAN[name]
    f, r = gan_inputs(name)
    k = _elt_keys(c.n, sms, 4 * TPB)
    for v, t in ((f, "f"), (r, "r")):
        k |= {"gan: %s==0" % t} if (v == 0).any() else set()
        k |= {"gan: %s==1" % t} if (v == 1).any() else set()
        k |= {"gan: %s==1-2^-24" % t} if (v == np.float32(1 - 2.0 ** -24)).any() else set()
        k |= {"gan: %s==2^-24" % t} if (v == np.float32(2.0 ** -24)).any() else set()
    k |= {"gan: %s NULL" % p for p in c.null}
    k |= {"gan: scales!=1"} if c.s_adv != 1 and c.s_dis != 1 else set()
    k |= {"gan: disc shape"} if c.n == 24 * 8 * 8 else set()
    return k


# ------------------------------------------------------------------------------------------------------------- Adam
# One TF-Adam step at t = 3 of lr 5e-5.  Of every ten elements, number 5 has g = 0 and number 9 has g = m = v = 0.
Adam = namedtuple("Adam", "n gscale")
GENERATOR_FLAT = 1286723                          # floats of the generator's parameters (16 residual blocks)
ADAM = {
    "n1": Adam(1, 1.0),
    "n255_gs": Adam(255, 0.25),
    "n257_gs3": Adam(257, 1.0 / 3.0),
    "n1000": Adam(1000, 1.0),
    "above_cap_gs": Adam(16 * 132 * 256 + 257, 0.25),
    "generator_flat_gs3": Adam(GENERATOR_FLAT, 1.0 / 3.0),
}
ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8
ADAM_LR_T = 5e-5 * (1 - ADAM_B2 ** 3) ** 0.5 / (1 - ADAM_B1 ** 3)


def adam_inputs(name):
    """p ~ 0.1 N, m ~ 0.01 N, v = (0.01 N)^2, |g| log-uniform in [1e-8, 1]: sqrt(v') runs from far below eps to far above."""
    c, r = ADAM[name], rng("adam " + name)
    p = (0.1 * r.standard_normal(c.n)).astype(np.float32)
    m = (0.01 * r.standard_normal(c.n)).astype(np.float32)
    v = ((0.01 * r.standard_normal(c.n)) ** 2).astype(np.float32)
    g = (np.where(r.rand(c.n) < 0.5, -1.0, 1.0) * 10.0 ** r.uniform(-8, 0, c.n)).astype(np.float32)
    g[5::10] = 0
    g[9::10], m[9::10], v[9::10] = 0, 0, 0
    return p, m, v, g


def adam_ref(p, m, v, g, gscale, lr_t=ADAM_LR_T, b1=ADAM_B1, b2=ADAM_B2, eps=ADAM_EPS):
    """float64 of m' = b1 m + (1 - b1) g s, v' = b2 v + (1 - b2) (g s)^2 on the fp32 constants the kernel gets (b1, b2, s
    rounded to fp32; 1.f - b1 and 1.f - b2 are exact fp32 subtractions).  Returns m', v', their two terms each, and a
    function p'(m', v') so that the parameter update can be judged from the kernel's own rounded moments."""
    b1, b2, s, lr_t, eps = (float(np.float32(t)) for t in (b1, b2, gscale, lr_t, eps))
    p, m, v, g = (t.astype(np.float64) for t in (p, m, v, g))
    gi = g * s
    m_terms, v_terms = (b1 * m, (1.0 - b1) * gi), (b2 * v, (1.0 - b2) * gi * gi)

    def step(m1, v1):
        return lr_t * m1.astype(np.float64) / (np.sqrt(v1.astype(np.float64)) + eps)
    return m_terms[0] + m_terms[1], v_terms[0] + v_terms[1], m_terms, v_terms, step


def _adam_keys(name, sms):
    c = ADAM[name]
    p, m, v, g = adam_inputs(name)
    k = _elt_keys(c.n, sms)
    k |= {"adam: gscale!=1"} if c.gscale != 1 else set()
    k |= {"adam: gscale not dyadic"} if c.gscale * 2 ** 10 % 1 else set()
    k |= {"adam: g==0"} if ((g == 0) & (v != 0)).any() else set()
    k |= {"adam: g==0 v==0 m==0"} if ((g == 0) & (v == 0) & (m == 0)).any() else set()
    k |= {"adam: generator size"} if c.n == GENERATOR_FLAT else set()
    return k


# ------------------------------------------------------------------------------------------------------ activations
ACT_NAMES = {ACT_NONE: "none", ACT_RELU: "relu", ACT_LRELU02: "lrelu", ACT_TANH24: "tanh24", ACT_SIGMOID: "sigmoid"}
ACT_SIZES = {"n1": 1, "n257": 257, "above_cap": 16 * 132 * 256 + 300}
ACT_X_EDGES = np.float32([0.0, -0.0, 1e-45, -1e-45, 1e-30, -1e-30, 0.5, -0.5, 3.0, -3.0, 10.0, -10.0, 20.0, -20.0,
                          100.0, -100.0])
# outputs the backward kernels must classify: +-0 (ReLU `>` against LeakyReLU `>=`), +-tiny, tanh at saturation,
# sigmoid at 0 and 1
ACT_Y_EDGES = {
    ACT_NONE: np.float32([0.0, -0.0, 1.0, -1.0]),
    ACT_RELU: np.float32([0.0, -0.0, 1e-45, 1e-30, 1.0, -1.0]),
    ACT_LRELU02: np.float32([0.0, -0.0, 1e-45, -1e-45, 1e-30, -1e-30, 1.0, -1.0]),
    ACT_TANH24: np.float32([0.0, -0.0, 24.0, -24.0, 23.999998, -23.999998, 12.0, -1e-30]),
    ACT_SIGMOID: np.float32([0.0, 1.0, 0.5, 1e-30, 1.0 - 2.0 ** -24, 0.25]),
}


def act_x(size):
    """Forward inputs: the edge table (as much as fits), then 3 N(0, 1)."""
    n, r = ACT_SIZES[size], rng("act " + size)
    x = (3.0 * r.standard_normal(n)).astype(np.float32)
    x[:ACT_X_EDGES.size] = ACT_X_EDGES[:n]
    return x


def act_bwd_inputs(size, act):
    """Saved outputs: the edge table, then values of the activation's range; and the incoming gradient."""
    n, r = ACT_SIZES[size], rng("act_bwd %s %d" % (size, act))
    y = act_ref(3.0 * r.standard_normal(n), act).astype(np.float32)
    e = ACT_Y_EDGES[act]
    y[:e.size] = e[:n]
    return y, r.uniform(-1, 1, n).astype(np.float32)


def act_ref(v, act):
    """float64 activation of the pre-activation v."""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore"):
        return {ACT_NONE: lambda: v, ACT_RELU: lambda: np.maximum(v, 0.0), ACT_LRELU02: lambda: np.where(v >= 0, v, F02 * v),
                ACT_TANH24: lambda: 24.0 * np.tanh(v), ACT_SIGMOID: lambda: 1.0 / (1.0 + np.exp(-v))}[act]()


def act_bwd_ref(y, dy, act):
    """float64 derivative on the saved output: ReLU y > 0, LeakyReLU y >= 0 ? 1 : 0.2, tanh24 24 (1 - (y / 24)^2) with
    y / 24 as y times the fp32 constant 1 / 24, sigmoid y (1 - y)."""
    y, g = y.astype(np.float64), dy.astype(np.float64)
    if act == ACT_RELU:
        return np.where(y > 0, g, 0.0)
    if act == ACT_LRELU02:
        return np.where(y >= 0, g, F02 * g)
    if act == ACT_TANH24:
        t = y * INV24
        return g * 24.0 * (1.0 - t * t)
    if act == ACT_SIGMOID:
        return g * y * (1.0 - y)
    return g


def act_bwd_f32(y, dy, act):
    """The fp32 chains without a multiply-add to contract: ReLU, LeakyReLU (0.2f * g) and sigmoid ((g * v) * (1.f - v))."""
    if act == ACT_RELU:
        return np.where(y > 0, dy, np.float32(0))
    if act == ACT_LRELU02:
        return np.where(y >= 0, dy, np.float32(0.2) * dy)
    if act == ACT_SIGMOID:
        return (dy * y) * (np.float32(1) - y)
    return dy


def _act_keys(size, sms):
    n = ACT_SIZES[size]
    k = _elt_keys(n, sms)
    for act, e in ACT_Y_EDGES.items():
        e = e[:n]
        z = e == 0
        k |= {"act: y==0"} if (z & ~np.signbit(e)).any() and act in (ACT_RELU, ACT_LRELU02) else set()
        k |= {"act: y==-0"} if (z & np.signbit(e)).any() and act in (ACT_RELU, ACT_LRELU02) else set()
        k |= {"tanh: |y|==24"} if act == ACT_TANH24 and (np.abs(e) == 24).any() else set()
        k |= {"sigmoid: y==0"} if act == ACT_SIGMOID and z.any() else set()
        k |= {"sigmoid: y==1"} if act == ACT_SIGMOID and (e == 1).any() else set()
    x = act_x(size)
    k |= {"act: x==-0"} if ((x == 0) & np.signbit(x)).any() else set()
    k |= {"tanh: saturating x"} if (np.abs(x) >= 20).any() else set()
    k |= {"sigmoid: |x|==100"} if (np.abs(x) == 100).any() else set()
    return k


# ---------------------------------------------------------------------------------------------------- bias gradient
# dy [npix, cpitch] on the 2^-2 grid in [-1, 1]; the channels from C on hold 2^20, which no sum can absorb unnoticed.
# With accumulate, db starts from values on the 2^-2 grid; without, from 1e30.
Bias = namedtuple("Bias", "npix C cpitch accumulate")
BIAS = {
    "c1_1px": Bias(1, 1, 1, 0),
    "c2_7px_pitch8_acc": Bias(7, 2, 8, 1),
    "c3_679px": Bias(8 * 85 - 1, 3, 3, 0),
    "c3_681px_pitch51_acc": Bias(8 * 85 + 1, 3, 51, 1),
    "c4_513px": Bias(8 * 64 + 1, 4, 4, 0),
    "c64_31px_pitch128": Bias(8 * 4 - 1, 64, 128, 0),
    "c100_17px_acc": Bias(8 * 2 + 1, 100, 100, 1),
    "c256_9px": Bias(9, 256, 256, 0),
    "c256_capped_acc": Bias(16 * 132 * 8 + 9, 256, 256, 1),
    "c2_capped_pitch3": Bias(16 * 132 * 8 * 128 + 129, 2, 3, 0),
}
BIAS_PAD = 2.0 ** 20


def bias_inputs(name):
    c, r = BIAS[name], rng("bias " + name)
    dy = np.full((c.npix, c.cpitch), BIAS_PAD, np.float32)
    dy[:, :c.C] = uniform(r, (c.npix, c.C), 2)
    db0 = (r.randint(-40, 41, c.C) / 4.0).astype(np.float32) if c.accumulate else np.full(c.C, 1e30, np.float32)
    return dy, db0


def bias_ref(dy, db0, C, accumulate):
    """db[c] (+)= sum over pixels of dy[pixel, c], c < C; also the sum of |terms|."""
    s = dy[:, :C].astype(np.float64).sum(0)
    a = np.abs(dy[:, :C]).astype(np.float64).sum(0)
    return (s + db0, a + np.abs(db0)) if accumulate else (s, a)


def bias_guard(name):
    c = BIAS[name]
    dy, db0 = bias_inputs(name)
    exact(bias_ref(dy, db0, c.C, c.accumulate)[1], 2, name + " sum |dy|")


def _bias_keys(name, sms):
    c = BIAS[name]
    blocks, ppb, capped = bias_launch(c.npix, c.C, sms)
    ppar = 256 // c.C
    k = {"bias: C=%d" % c.C, "bias: one block" if blocks == 1 else "bias: multi block"}
    k |= {"bias: pitched"} if c.cpitch > c.C else set()
    k |= {"bias: accumulate"} if c.accumulate else {"bias: overwrite"}
    k |= {"bias: capped"} if capped else set()
    k |= {"bias: last block short"} if c.npix % ppb else set()
    k |= {"bias: C∤256"} if 256 % c.C else set()
    k |= {"bias: npix<ppar"} if c.npix < ppar else set()
    k |= {"bias: npix==8ppar-1"} if c.npix == 8 * ppar - 1 else set()
    k |= {"bias: npix==8ppar+1"} if c.npix == 8 * ppar + 1 else set()
    return k


# ------------------------------------------------------------------------------------------------------ conversions
# fp32 -> bf16 rows: npix, C, src_cpitch, dst_cpitch (teco_f32_to_bf16_rowpad writes the whole padded row)
Rows = namedtuple("Rows", "npix C src_cpitch dst_cpitch")
ROWPAD = {
    "c3_to_64": Rows(37, 3, 3, 64),
    "c51_pitch64_to_64": Rows(19, 51, 64, 64),
    "c64_dense": Rows(33, 64, 64, 64),
    "above_cap_c48_to_64": Rows((16 * 132 * 256) // 64 + 5, 48, 48, 64),
}
# bf16 -> fp32: npix, C, src_cpitch, dst_cpitch (channels from C on of dst are left alone)
FROM_BF16 = {
    "c3_from_64": Rows(37, 3, 64, 3),
    "c3_from_64_pitch8": Rows(37, 3, 64, 8),
    "c64_dense": Rows(33, 64, 64, 64),
    "above_cap_c48_pitch51": Rows((16 * 132 * 256) // 48 + 7, 48, 64, 51),
}


def bf16_midpoint_values(r, shape):
    """fp32 values of magnitude around 1: a quarter sit exactly between two bf16 neighbours (low 16 bits 0x8000, with
    the bit above even or odd), a quarter one fp32 ulp to either side of such a midpoint, the rest arbitrary."""
    n = int(np.prod(shape))
    b = (r.randint(0, 2 ** 16, n).astype(np.uint32) | (r.randint(0x3E00, 0x4080, n).astype(np.uint32) << 16))
    b |= (r.randint(0, 2, n).astype(np.uint32) << 31)
    kind = r.randint(0, 4, n)
    low = np.where(kind == 0, 0x8000, np.where(kind == 1, np.where(r.rand(n) < 0.5, 0x7FFF, 0x8001), b & 0xFFFF))
    return ((b & np.uint32(0xFFFF0000)) | low.astype(np.uint32)).view(np.float32).reshape(shape)


def bf16_values(r, shape):
    """Arbitrary finite bf16 numbers as fp32."""
    b = r.randint(0, 2 ** 16, int(np.prod(shape))).astype(np.uint32)
    b = np.where((b & 0x7F80) == 0x7F80, b & 0xBFFF, b)          # no inf / NaN
    return (b << 16).astype(np.uint32).view(np.float32).reshape(shape)


def rows_inputs(table, name):
    c, r = table[name], rng("rows " + name)
    if table is ROWPAD:
        return bf16_midpoint_values(r, (c.npix, c.src_cpitch))
    return bf16_values(r, (c.npix, c.src_cpitch)), uniform(r, (c.npix, c.dst_cpitch), 7)


def _rows_keys(table):
    def f(name, sms):
        c = table[name]
        k = {"rows: src pitched"} if c.src_cpitch > c.C else set()
        k |= {"rows: dst pitched"} if c.dst_cpitch > c.C else set()
        n = c.npix * (c.dst_cpitch if table is ROWPAD else c.C)
        k |= {"rows: >1 grid-stride pass"} if elt_launch(n, sms)[1] > 1 else set()
        if table is ROWPAD:
            v = rows_inputs(table, name)[:, :c.C].view(np.uint32)
            low, odd = v & 0xFFFF, (v >> 16) & 1
            k |= {"rows: midpoint to even (down)"} if ((low == 0x8000) & (odd == 0)).any() else set()
            k |= {"rows: midpoint to even (up)"} if ((low == 0x8000) & (odd == 1)).any() else set()
        return k
    return f


def u8_inputs():
    """k / 255 in fp32 and its two fp32 neighbours for k = 0 .. 255, then negatives, values above 1 and -0."""
    k = (np.arange(256, dtype=np.float32) / np.float32(255))
    x = np.concatenate((k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)),
                        np.float32([-0.0, -1e-30, -0.5, -7.0, 1.0000001, 1.5, 300.0, 1e30, -1e30])))
    return x.astype(np.float32)


def u8_ref(x):
    """clip(x * 255, 0, 255) in fp32, truncated (save_img, lib/ops.py:521-523)."""
    return np.clip(x.astype(np.float32) * np.float32(255), np.float32(0), np.float32(255)).astype(np.uint8)


FAMILIES = {
    "bn": (BN, _bn_keys),
    "l2": (L2, _loss_keys(L2)),
    "l1": (L1, _loss_keys(L1)),
    "cos": (COS, _cos_keys(COS)),
    "l2norm": (L2NORM, _cos_keys(L2NORM)),
    "gan": (GAN, _gan_keys),
    "adam": (ADAM, _adam_keys),
    "act": (ACT_SIZES, _act_keys),
    "bias": (BIAS, _bias_keys),
    "rowpad": (ROWPAD, _rows_keys(ROWPAD)),
    "from_bf16": (FROM_BF16, _rows_keys(FROM_BF16)),
}

REQUIRED = {
    "bn": {"bn: one block", "bn: multi block", "bn: last block short", "bn: blocks capped", "bn: C∤256", "bn: ppar==1",
           "bn: ppar==2", "bn: npix==1", "bn: npix not 2^k", "bn: mean far from zero", "bn: lrelu", "bn: no lrelu", "bn: y==0",
           "bn: continuous", "bn: disc layer", "bn: apply >1 grid-stride pass"},
    "l2": {"eltwise: >1 grid-stride pass", "eltwise: n%256!=0", "l2: d==0", "l2: gscale!=1", "l2: exact scalar",
           "l2: bounded scalar", "l2: blocks capped"},
    "l1": {"eltwise: >1 grid-stride pass", "eltwise: n%256!=0", "eltwise: n==1", "l1: d==0", "l1: d==-0", "l1: gscale!=1",
           "l1: per_pixel", "l1: exact scalar", "l1: bounded scalar"},
    "cos": {"cos: zero f", "cos: zero g", "cos: zero f and g", "cos: C%32!=0", "cos: >1 pixel per warp", "cos: npix==1",
            "cos: df NULL", "cos: gscale!=1"} | {"cos: C=%d" % c for c in (3, 48, 64, 128, 256, 512)},
    "l2norm": {"l2norm: zero f", "l2norm: C%32!=0", "l2norm: >1 pixel per warp"} | {"l2norm: C=%d" % c for c in (3, 64, 128, 256, 512)},
    "gan": {"eltwise: >1 grid-stride pass", "eltwise: n%256!=0", "eltwise: n==1", "gan: f==0", "gan: f==1", "gan: r==0",
            "gan: r==1", "gan: f==1-2^-24", "gan: f==2^-24", "gan: r==1-2^-24", "gan: r==2^-24", "gan: adv NULL",
            "gan: dis_f NULL", "gan: dis_r NULL", "gan: scales!=1", "gan: disc shape"},
    "adam": {"eltwise: >1 grid-stride pass", "eltwise: n%256!=0", "eltwise: n==1", "adam: gscale!=1", "adam: gscale not dyadic",
             "adam: g==0", "adam: g==0 v==0 m==0", "adam: generator size"},
    "act": {"eltwise: >1 grid-stride pass", "eltwise: n%256!=0", "eltwise: n==1", "act: y==0", "act: y==-0", "tanh: |y|==24",
            "sigmoid: y==0", "sigmoid: y==1", "act: x==-0", "tanh: saturating x", "sigmoid: |x|==100"},
    "bias": {"bias: pitched", "bias: accumulate", "bias: overwrite", "bias: capped", "bias: one block", "bias: multi block",
             "bias: last block short", "bias: C∤256", "bias: npix<ppar", "bias: npix==8ppar-1", "bias: npix==8ppar+1"}
    | {"bias: C=%d" % c for c in (1, 2, 3, 4, 64, 100, 256)},
    "rowpad": {"rows: src pitched", "rows: dst pitched", "rows: >1 grid-stride pass", "rows: midpoint to even (down)",
               "rows: midpoint to even (up)"},
    "from_bf16": {"rows: src pitched", "rows: dst pitched", "rows: >1 grid-stride pass"},
}


def keys(family, name, sms=132):
    return FAMILIES[family][1](name, sms)
