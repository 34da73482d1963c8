"""generator_F, fnet and the VGG19 trunk of the bf16 training graph in float64, rounded exactly where the training
kernels of tecogan_b200/kernels.py round, forward and backward, and the operands on which that restatement is exact, so
the autograd graph lib/frvsr.py and lib/Teco.py::_vgg_raw build under train precision 'bf16' can be compared with it bit
for bit: outputs, every weight and bias gradient and the input gradient.

The reference walks the oracle's parameter names and layer order (oracle/teco_oracle.py generator_F, fnet and
vgg19_features), not the device's wiring.  TrainRounding(on=False) makes every rounding point the identity, and the
reference is then the oracle's own float64 autograd, op for op.  With rounding on, every 3x3 convolution and transposed
convolution (_Conv3x3TC, _ConvTranspose2xTC) computes
  forward   xb = bf16(x), z = f32(conv(xb, bf16(w)) + b);
            Cout >= 16: y = f32(bf16(act(z))), then + res rounded once to fp32 (resblock conv_2; teco_bf16_to_f32_add);
            Cout < 16 (the fp32 output stage): y = z + res in fp32 (generator 64 -> 3, res the device's bicubic, a
            constant: bicubic_four has no gradient), or tanh(z) * 24 (FNet's flow head);
  backward  dz = act_bwd(y, dy) (train_kernel_cases.act_bwd_f32), dzb = bf16(dz), dx = f32(bf16(conv_T(dzb, bf16(w)))),
            dw = f32(sum xb dzb), db = sum dz (fp32 dz, not dzb), and the residual's gradient is dy itself.
The glue is fp32: max-pool (the gradient to the first maximum in TL, TR, BL, BR order), the legacy x2 resize and its
scattered gradient, preprocess 2 v - 1, the VGG input's 127.5 x + 127.5 - VGG_MEAN, and autograd's fp32 sum where a
tensor has two consumers (a resblock's input, a VGG tap).

Guards, run before every sum when a check is given, fail a case whose operands leave the regime where the device's
fp32 result is determined, instead of letting it pass by luck:
  * forward conv: nets_exact.nets_check (one product per output channel, or every term on one grid within 2^22 units);
  * dgrad, wgrad: every term of an output channel is a multiple of g = the smallest product of its factors' per-channel
    grid units, and sum|terms| <= 2^22 g for every output -- then every fp32 partial sum is exact in any order (the
    argument of test_gpu_conv_exact.py, applied per channel);
  * resize forward: nets_exact.resize_check; resize gradient: terms on lsb(g) / 4, sum|terms| within 2^22 units;
  * every fp32 sum of two gradients autograd makes is exact.
A bias gradient is a sum of fp32 dz over the pixels.  Where dz of a channel is on one grid within 2^22 units that sum is
exact; elsewhere (LeakyReLU's negative branch, whose dz = 0.2f * g carries a full significand, and the flow head) its
summation order is not pinned and the reference gives the interval [lo, hi] the device's sum must lie in: the float64
sum widened by n 2^-24 sum|dz| (bias_bounds).

The flow head's backward is the one rounding the host cannot pin: act_bwd computes g * 24 * (1 - t t), t = y * (1/24),
and the compiler may contract 1 - t t into an FMA.  Both candidates are computed from the device's flow (TrainRounding's
`flow`); a guard requires them to round to the same bf16 everywhere, which determines dzb and so the head's dx and dw and
everything below the head, and the head's bias interval spans both candidates' sums.

Operands: nets_exact's generator set with sparse +-1 upstream gradients (sparse_grad); nets_exact's FNet sets, 'nonneg'
and 'signed' forward, 'signed' backward with a few sparse +-1 upstream flow gradients (see FNET_BWD_CASES for why); the
VGG trunk with one power-of-two weight per output channel (every layer one product, 16 layers deep) and inputs k/256, on
which 127.5 x + 127.5 is exact in fp32 whether or not it is contracted, with k/16 gradients at its taps.  A weight
gradient sums x dzb over every pixel of a layer, which is why the upstream gradients are sparse: dense k/16 gradients
leave the exact regime by orders of magnitude at 2 x 128 x 128 pixels.

Feature names (layer_features) restate with tests/conv_paths.py which kernel each forward launch, each input-gradient
launch (flag-3 packing, Cout_pad -> Cin_pad; the transposed conv's on the space-to-depth gradient, 4 Cout -> Cin) and
each weight-gradient launch reaches."""
from collections import namedtuple
from fractions import Fraction

import numpy as np
import torch
import torch.nn.functional as F

from oracle import teco_oracle as O
from tecogan_b200._ffi import ACT_LRELU02, ACT_NONE, ACT_RELU, ACT_TANH24
from tests import nets_exact as E
from tests.conv_paths import ACT_NAMES, features, route, wgrad_features
from tests.resample_cases import windows
from tests.test_gpu_conv_exact import EXACT_SPAN, REL_BOUND, _grid, _is_f32
from tests.test_gpu_resample_exact import _resize_ref
from tests.train_kernel_cases import act_bwd_f32

GEN, FNET = E.GEN, E.FNET
INV24 = np.float32(1.0 / 24.0)
U32 = 2.0 ** -24                       # fp32 unit roundoff


# ------------------------------------------------------------------------------------------------------ rounding points
class TrainRounding:
    """The training kernels' rounding points (on) or none (off).  check: run the guards.  flow: the device's flow, which
    the head's backward starts from (default: this forward's flow rounded to fp32).  After a backward, bias[what] holds
    the interval (lo, hi) of each bias gradient and layers the (what, input shape, weight shape) of every conv run."""

    def __init__(self, on=True, check=False, flow=None):
        self.on, self.check, self.flow = on, check, flow
        self.bias, self.layers = {}, []

    def f32(self, v):
        return v.float().double() if self.on else v

    def bf16(self, v):
        return v.float().to(torch.bfloat16).double() if self.on else v

    def add(self, a, b):
        return (a.float() + b.float()).double() if self.on else a + b

    def join(self, what, t):
        """t has two consumers: autograd adds their gradients in fp32, which the guard requires to be exact."""
        if self.check and t.requires_grad:
            def hook(g):
                assert _is_f32(g), what + ": the fp32 sum of two gradients is not exact"
            t.register_hook(hook)
        return t


# ----------------------------------------------------------------------------------------------------------- guards
def lsb_elem(t):
    """Largest power of two dividing each element (float64); inf for zeros."""
    m, e = torch.frexp(t)
    mi = (m.abs() * 2.0 ** 53).long()
    low = torch.ldexp((mi & -mi).double(), e - 53)
    return torch.where(t == 0, torch.full_like(low, float("inf")), low)


def lsb_channels(t):
    """Per channel (last axis) the largest power of two dividing every element; inf for an all-zero channel."""
    return lsb_elem(t.reshape(-1, t.shape[-1])).amin(0)


def _assert_span(what, s_terms, g):
    """sum|terms| <= 2^22 g, g broadcast against s_terms (per output channel)."""
    bad = s_terms > EXACT_SPAN * g
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: sum|terms| %.4g > 2^22 g = %.4g at %s" % (
            what, float(s_terms[i]), float((EXACT_SPAN * g.expand_as(s_terms))[i]), i))


def _conv_op(transpose):
    return O.conv2d_transpose if transpose else O.conv2d


def _grads(transpose, x, w, dz):
    """(d conv / dx, d conv / dw) for the upstream dz, float64 (the float64 sums of the device's dgrad and wgrad)."""
    with torch.enable_grad():
        xx, ww = x.detach().requires_grad_(), w.detach().requires_grad_()
        return torch.autograd.grad(_conv_op(transpose)(xx, ww), (xx, ww), dz)


def _backward_guards(what, transpose, xb, wb, dzb, need_dw):
    """dgrad: dx[.., ci] sums dzb[.., co] w[t, ci, co] (transposed: w[t, co, ci]); wgrad: dw[t, ci, co] sums xb[.., ci]
    dzb[.., co].  Per-channel grid units, sum|terms| from the same sums on magnitudes."""
    s_dx, s_dw = _grads(transpose, xb.abs(), wb.abs(), dzb.abs())
    lx, lw, ldz = lsb_channels(xb), lsb_elem(wb), lsb_channels(dzb)
    ldz_w = ldz.view(1, 1, -1, 1) if transpose else ldz.view(1, 1, 1, -1)
    g_dx = (lw * ldz_w).amin(dim=(0, 1, 2 if transpose else 3))               # per ci
    _assert_span(what + " dgrad", s_dx, g_dx)
    if need_dw:
        g_dw = ldz.view(-1, 1) * lx.view(1, -1) if transpose else lx.view(-1, 1) * ldz.view(1, -1)
        _assert_span(what + " wgrad", s_dw, g_dw)


def bias_bounds(dz):
    """Per channel (lo, hi) of an fp32 sum of dz in any order: the float64 sum where every partial sum is exact (terms
    on the channel's grid within 2^22 units), else the float64 sum +- n 2^-24 sum|dz| (n terms)."""
    d = dz.reshape(-1, dz.shape[-1])
    s, a = d.sum(0), d.abs().sum(0)
    exact = a <= EXACT_SPAN * lsb_channels(d)
    err = torch.where(exact, torch.zeros_like(a), (d != 0).sum(0).double() * U32 * a)
    return s - err, s + err


# ------------------------------------------------------------------------------------------------ flow head backward
def _round_f32(q):
    """Fraction -> the nearest fp32 (ties to even), as a Python float."""
    f = np.float32(float(q))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - q)
        even = (np.array(c, np.float32).view(np.uint32) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, float(c))
    return best[1]


def tanh24_bwd_candidates(y, dy):
    """act_bwd_kernel's g * 24 * (1 - t t), t = y * (1/24), in fp32 from the fp32 flow y: (1 - t t) rounded twice, and
    contracted into fma(-t, t, 1).  float64 tensors of fp32 values."""
    y32, g32 = y.float().cpu(), dy.float().cpu()
    t = y32 * torch.tensor(INV24)
    g24 = g32 * 24.0
    s1 = 1.0 - t * t
    s2 = torch.tensor([_round_f32(1 - Fraction(float(v)) ** 2) for v in t.flatten().tolist()],
                      dtype=torch.float32).view(t.shape)
    return (g24 * s1).double().to(y.device), (g24 * s2).double().to(y.device)


def _bf16_bits(v):
    return v.float().to(torch.bfloat16).view(torch.int16)


# ------------------------------------------------------------------------------------------------------ the layers
def _act_fwd(R, z, act):
    if act == ACT_RELU:
        return F.relu(z)
    if act == ACT_LRELU02:
        return E.Rounding(R.on).lrelu(z)
    return z


def _act_bwd(R, act, y, dy):
    if not R.on:
        return {ACT_RELU: lambda: torch.where(y > 0, dy, 0.0 * dy), ACT_LRELU02: lambda: torch.where(y >= 0, dy, 0.2 * dy),
                ACT_NONE: lambda: dy}[act]()
    y32, g32 = y.detach().float().cpu().numpy(), dy.detach().float().cpu().numpy()
    return torch.from_numpy(act_bwd_f32(y32, g32, act)).double().to(y.device)


class _Conv(torch.autograd.Function):
    """One conv2 / conv2_tran of the training graph (see the module docstring).  spec: (R, what, act, transpose)."""

    @staticmethod
    def forward(ctx, x, w, b, res, spec):
        R, what, act, transpose = spec
        xb, wb = R.bf16(x), R.bf16(w)
        R.layers.append((what, tuple(x.shape), tuple(w.shape)))
        if R.check:
            E.nets_check("conv", what, xb, wb, b, None, transpose)
        z = R.f32(_conv_op(transpose)(xb, wb, b))
        if w.shape[3 - int(transpose)] < 16:               # the fp32 output stage
            y = torch.tanh(z) * 24.0 if act == ACT_TANH24 else z
        else:
            y = R.bf16(_act_fwd(R, z, act))
        if res is not None:
            y = R.add(y, res)
        ctx.spec = spec
        ctx.save_for_backward(xb, wb, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        R, what, act, transpose = ctx.spec
        xb, wb, y = ctx.saved_tensors
        if act == ACT_TANH24 and R.on:
            flow = R.flow if R.flow is not None else R.f32(y)
            cands = tanh24_bwd_candidates(flow, dy)
            bad = _bf16_bits(cands[0]) != _bf16_bits(cands[1])
            assert not bool(bad.any()), "%s: the two act_bwd candidates round to different bf16 at %d elements" % (
                what, int(bad.sum()))
            dz = cands[0]
            lo, hi = zip(*(bias_bounds(c) for c in cands))
            bounds = (torch.minimum(*lo), torch.maximum(*hi))
        else:
            t = y / 24.0
            dz = dy * 24.0 * (1.0 - t * t) if act == ACT_TANH24 else _act_bwd(R, act, y, dy)
            bounds = bias_bounds(dz)
        dzb = R.bf16(dz)
        need_dw = ctx.needs_input_grad[1]
        if R.check:
            _backward_guards(what, transpose, xb, wb, dzb, need_dw)
        dx, dw = _grads(transpose, xb, wb, dzb)
        dx, dw, db = R.bf16(dx), R.f32(dw) if need_dw else None, None
        if need_dw and ctx.needs_input_grad[2]:
            db = dz.sum(dim=(0, 1, 2))
            prev = R.bias.get(what)                          # a layer applied again (reuse=True) sums its bias gradients
            R.bias[what] = bounds if prev is None else (prev[0] + bounds[0], prev[1] + bounds[1])
        return dx, dw, db, (dy if ctx.needs_input_grad[3] else None), None


def conv(R, p, what, x, act, res=None, transpose=False):
    return _Conv.apply(x, p[what + "/weights"], p[what + "/biases"], res, (R, what, act, transpose))


class _MaxPool(torch.autograd.Function):
    """2x2 max-pool, stride 2, the odd row / column dropped; the gradient goes to the first maximum of each window in
    TL, TR, BL, BR order (teco_maxpool2_f32 / _bwd_f32, as tests/test_gpu_resample_exact.py restates them)."""

    @staticmethod
    def forward(ctx, x):
        win = windows(x.detach().cpu().numpy())
        ctx.shape, ctx.best, ctx.device = x.shape, win.argmax(3), x.device
        return torch.from_numpy(win.max(3)).to(x.device)

    @staticmethod
    def backward(ctx, g):
        N, H, W, C = ctx.shape
        oh, ow = H // 2, W // 2
        gn = g.detach().cpu().numpy()
        dwin = np.where(np.arange(4)[None, None, None, :, None] == ctx.best[:, :, :, None], gn[:, :, :, None], 0.0)
        dx = np.zeros((N, H, W, C))
        dx[:, :2 * oh, :2 * ow] = dwin.reshape(N, oh, ow, 2, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, 2 * oh, 2 * ow, C)
        return torch.from_numpy(dx).to(ctx.device)


class _Resize2x(torch.autograd.Function):
    """Legacy bilinear x2 in fp32 (teco_resize_bilinear_f32) and its scattered gradient; both exact under the guards."""

    @staticmethod
    def forward(ctx, x, R, what):
        if R.check:
            E.resize_check(what, x)
        ctx.R, ctx.what, ctx.x = R, what, x.detach()
        n, h, w, c = x.shape
        return O.resize_bilinear_legacy(x.detach().cpu(), 2 * h, 2 * w).to(x.device)

    @staticmethod
    def backward(ctx, g):
        x = ctx.x
        _, _, _, dx, sg, _ = _resize_ref(x.cpu().numpy(), g.detach().cpu().numpy(), g.shape[1], g.shape[2])
        dx, sg = torch.from_numpy(dx), torch.from_numpy(sg)
        if ctx.R.check:
            unit = lsb_elem(g.cpu()).min() / 4                # the terms g (1 - wy)(1 - wx) with weights 0, 1/2
            assert bool((sg <= EXACT_SPAN * unit).all()), ctx.what + ": resize gradient sums leave the exact regime"
        return dx.to(x.device), None, None


# ----------------------------------------------------------------------------------------------------- the networks
def generator_train_ref(p, gen_inputs, num_resblock, R, bic):
    """O.generator_F on the training kernels' rounding points.  bic: the bicubic residual, a constant (the device's
    teco_bicubic4_f32 of the LR channels; bicubic_four has no gradient)."""
    def cv(name, x, act, res=None, transpose=False):
        return conv(R, p, GEN + name, x, act, res, transpose)

    net = cv("input_stage/conv/Conv", gen_inputs, ACT_RELU)
    for i in range(1, num_resblock + 1):
        R.join("resblock_%d input" % i, net)                  # conv_1's input and conv_2's residual
        r = cv("resblock_%d/conv_1/Conv" % i, net, ACT_RELU)
        net = cv("resblock_%d/conv_2/Conv" % i, r, ACT_NONE, res=net)
    for i in (1, 2):
        net = cv("conv_tran2highres/conv_tran%d/Conv2d_transpose" % i, net, ACT_RELU, transpose=True)
    net = cv("output_stage/conv/Conv", net, ACT_NONE, res=bic.detach())
    return R.f32(net * 2.0 - 1.0)                             # preprocess: 2 v is exact, so FMA or not is one rounding


def fnet_train_ref(p, fnet_input, R):
    """O.fnet on the training kernels' rounding points: [n, h, w, 6] -> flow (float64; the device's is within
    REL_BOUND)."""
    net = fnet_input
    for name in E.ENCODERS + E.DECODERS:
        net = conv(R, p, FNET + name + "/conv_1/Conv", net, ACT_LRELU02)
        net = conv(R, p, FNET + name + "/conv_2/Conv", net, ACT_LRELU02)
        net = _MaxPool.apply(net) if name in E.ENCODERS else _Resize2x.apply(net, R, name)
    net = conv(R, p, FNET + "output_stage/conv1/Conv", net, ACT_LRELU02)
    return conv(R, p, FNET + "output_stage/conv2/Conv", net, ACT_TANH24)


VGG_MEAN32 = torch.tensor(O.VGG_MEAN, dtype=torch.float32).double()


def vgg_train_ref(p, x_pm1, R):
    """lib/Teco.py::_vgg_raw on the training kernels' rounding points: {tap: raw post-ReLU map} for O.VGG_TAPS."""
    net = R.f32(R.f32(x_pm1 * 127.5 + 127.5) - (VGG_MEAN32 if R.on else torch.tensor(O.VGG_MEAN, dtype=torch.float64))
                .to(x_pm1.device))
    out = {}
    for blk, reps, _, _ in O.VGG_CFG:
        for j in range(1, reps + 1):
            name = "vgg_19/conv%d/conv%d_%d" % (blk, blk, j)
            net = conv(R, p, name, net, ACT_RELU)
            if name in O.VGG_TAPS:
                out[name] = R.join(name, net)                 # the tap's upstream gradient and the next layer's
        if blk < 5:
            net = _MaxPool.apply(net)
    return out


# ------------------------------------------------------------------------------------------------------ operands
def grad_grid(seed, shape):
    """Upstream gradients k/16, |k| <= 16."""
    return _grid(np.random.RandomState(seed), shape, 2.0 ** -4, 16)


def sparse_grad(seed, shape, density=1.0 / 512):
    """Upstream gradients +-1 on a `density` fraction of the elements, else 0: the weight-gradient sums over every pixel
    of a layer then stay within 2^22 units of their grid (dense k/16 gradients do not, at 2 x 128 x 128 pixels)."""
    r = np.random.RandomState(seed)
    return torch.from_numpy(np.where(r.rand(*shape) < density, r.choice([-1.0, 1.0], size=shape), 0.0) + 0.0)


def vgg_operands(seed, n, h, w):
    """(params, input [n, h, w, 3] in [-1, 1]): one weight +-2^-1, +-1 or +-2 per output channel at a random tap and input
    channel, biases k/16; the input k/256, so 127.5 x + 127.5 = 255 (k + 256) / 512 is exact in fp32."""
    rng = np.random.RandomState(seed)
    p = {}
    for blk, reps, cin, cout in O.VGG_CFG:
        c = cin
        for j in range(1, reps + 1):
            name = "vgg_19/conv%d/conv%d_%d" % (blk, blk, j)
            flat = np.zeros((9 * c, cout))
            flat[rng.randint(0, 9 * c, size=cout), np.arange(cout)] = (
                rng.choice([-1.0, 1.0], size=cout) * 2.0 ** rng.randint(-1, 2, size=cout))
            p[name + "/weights"] = torch.from_numpy(flat.reshape(3, 3, c, cout) + 0.0)
            p[name + "/biases"] = _grid(rng, (cout,), 2.0 ** -4, 64)
            c = cout
    x = torch.from_numpy(rng.randint(-256, 257, size=(n, h, w, 3)) / 256.0)
    return p, x


# ------------------------------------------------------------------------------------------------------ case tables
Layer = namedtuple("Layer", "what n h w cin cout act res transpose wgrad dgrad")


def gen_layers(B, h, w, N):
    """Every conv of generator_F in order; h, w: the layer's input size."""
    out = [Layer(GEN + "input_stage/conv/Conv", B, h, w, 51, 64, ACT_RELU, False, False, True, True)]
    for i in range(1, N + 1):
        out += [Layer(GEN + "resblock_%d/conv_1/Conv" % i, B, h, w, 64, 64, ACT_RELU, False, False, True, True),
                Layer(GEN + "resblock_%d/conv_2/Conv" % i, B, h, w, 64, 64, ACT_NONE, True, False, True, True)]
    for i, s in ((1, 1), (2, 2)):
        out.append(Layer(GEN + "conv_tran2highres/conv_tran%d/Conv2d_transpose" % i, B, s * h, s * w, 64, 64, ACT_RELU,
                         False, True, True, True))
    return out + [Layer(GEN + "output_stage/conv/Conv", B, 4 * h, 4 * w, 64, 3, ACT_NONE, True, False, True, True)]


def fnet_layers(n, h, w, backward=False):
    """FNet's convs; backward: their input and weight gradients are launched (and checked) too."""
    b = backward
    out = []
    for (name, cin, cout), (lh, lw) in zip(O.FNET_LAYERS, E.fnet_level_sizes(h, w)):
        out += [Layer(FNET + name + "/conv_1/Conv", n, lh, lw, cin, cout, ACT_LRELU02, False, False, b, b),
                Layer(FNET + name + "/conv_2/Conv", n, lh, lw, cout, cout, ACT_LRELU02, False, False, b, b)]
    lh, lw = [2 * v for v in E.fnet_level_sizes(h, w)[-1]]
    return out + [Layer(FNET + "output_stage/conv1/Conv", n, lh, lw, 64, 32, ACT_LRELU02, False, False, b, b),
                  Layer(FNET + "output_stage/conv2/Conv", n, lh, lw, 32, 2, ACT_TANH24, False, False, b, b)]


def vgg_layers(n, h, w):
    out = []
    for blk, reps, cin, cout in O.VGG_CFG:
        c = cin
        for j in range(1, reps + 1):
            out.append(Layer("vgg_19/conv%d/conv%d_%d" % (blk, blk, j), n, h, w, c, cout, ACT_RELU, False, False, False, True))
            c = cout
        h, w = h // 2, w // 2
    return out


def _pad64(c):
    return (c + 63) // 64 * 64


def layer_launches(L):
    """(forward, dgrad, wgrad or None) launches of one layer as (kind, args): 'conv' args for conv_paths.features
    (mode, n, h, w, cin, cout, act, bias, res, y, f32c, res_f32), 'wgrad' args for wgrad_features."""
    if L.transpose:
        fwd = (1, L.n, L.h, L.w, 64, L.cout, L.act, True, "", True, 0, False)
        dgrad = (0, L.n, L.h, L.w, 4 * L.cout, L.cin, ACT_NONE, False, "", True, 0, False)
        wg = (L.n, L.h, L.w, 4 * L.cout, L.cin)
    else:
        cip, cop = _pad64(L.cin), _pad64(L.cout)
        if L.cout < 16:
            fwd = (0, L.n, L.h, L.w, cip, 16, L.act, True, "", False, L.cout, L.res)
        else:
            fwd = (0, L.n, L.h, L.w, cip, cop, L.act, True, "", True, 0, False)
        dgrad = (0, L.n, L.h, L.w, cop, cip, ACT_NONE, False, "", True, 0, False)
        wg = (L.n, L.h, L.w, L.cin, L.cout if L.cout % 4 == 0 else (L.cout + 3) // 4 * 4)
    return fwd, dgrad if L.dgrad else None, wg if L.wgrad else None


def layer_features(L):
    """Keys reached by one layer: conv_paths.features of its forward launch, the same prefixed 'dgrad ' for its input
    gradient, wgrad_features (with 'wgrad cin=', and 'wgrad cout=C run as 4' for a narrow layer) for its weight
    gradient, and 'fp32 output stage + residual' / 'fp32 output stage tanh24' for the narrow convolutions."""
    fwd, dgrad, wg = layer_launches(L)
    out = features(*fwd) | ({"dgrad " + k for k in features(*dgrad)} if dgrad else set())
    if not L.transpose and L.cout < 16:
        out.add("fp32 output stage " + ("+ residual" if L.res else ACT_NAMES[L.act]))
    if wg is not None:
        out |= wgrad_features(*wg) | {"wgrad cin=%d" % L.cin}
        if wg[4] != L.cout:
            out.add("wgrad cout=%d run as %d" % (L.cout, wg[4]))
    return out


def kernels_reached(layers):
    """Kernel instances of every forward and dgrad launch."""
    out = set()
    for L in layers:
        for mode, n, h, w, cin, cout, act, bias, res, y, f32c, res_f32 in filter(None, layer_launches(L)[:2]):
            out.add(route(mode, cin, cout, bool(res), False, f32c > 0, y).kernel)
    return out


# generator_F: batch, LR size, residual blocks, operand seed and the density of the sparse +-1 upstream gradient on the HR
# output.  A weight gradient sums x dzb over every pixel of a layer, so the more pixels a layer has and the deeper the
# gradient spreads, the sparser it must start for every sum to stay within 2^22 units of its grid: 2 x 32 x 32 with 16
# residual blocks needs 1/8192 (12 non-zero elements), where 1/512 exceeds the bound by up to 1.2x in the trunk.
GenCase = namedtuple("GenCase", "B h w N seed density")
GEN_CASES = {"2x32x32 N=3": GenCase(2, 32, 32, 3, 5002, 1.0 / 512), "2x32x32 N=16": GenCase(2, 32, 32, 16, 5003, 1.0 / 8192),
             "1x13x19 N=3": GenCase(1, 13, 19, 3, 5001, 1.0 / 512), "1x13x19 N=16": GenCase(1, 13, 19, 16, 5000, 1.0 / 512)}
# fnet forward, both operand sets: (n, h, w)
FNET_CASES = {"2x32x32": (2, 32, 32), "1x24x40": (1, 24, 40)}
# fnet forward and backward on the 'signed' operands, seeded by `seed`, with a few sparse +-1 upstream flow gradients.
# The 'signed' set keeps every activation within a few binades (8 significant bits each, one channel per product), so
# a weight gradient's sum stays exact while it has only a few non-zero dz per channel; its LeakyReLU takes the negative
# branch on about half the channels, so dz = 0.2f g is not bf16-exact there and the bias gradient reads it.  The
# 'nonneg' set cannot have an exact backward: its activations carry up to 16 significant bits, so one product x dzb
# alone has 24.  At these densities the guards also reject most seeds (a miss of 1.02x to 2x over 2^22 units at the
# decoders' or encoder_1's weight gradient), and on others a gradient walks off the map through a padded tap and the
# input gradient vanishes; with these seeds every guard passes and the input and every parameter get a non-zero
# gradient.
FnetBwd = namedtuple("FnetBwd", "n h w seed density")
FNET_BWD_CASES = {"2x32x32": FnetBwd(2, 32, 32, 5125, 0.0007), "1x24x40": FnetBwd(1, 24, 40, 5170, 0.003)}
VGG_CASES = {"1x64x64": (1, 64, 64), "1x40x56": (1, 40, 56)}

REQUIRED = {
    "ws<0>", "ws<0> cin=64", "ws<0> res=none", "ws<0> ragged", "wgmma<64> smaller than a tile", "ws<0> act=relu",
    "ws<0> act=lrelu", "ws<0> act=none",
    "ws<1>", "ws<1> act=relu", "ws<1> ragged",
    "wgmma<64> resident", "wgmma<64> streamed", "wgmma<64> cin=128", "wgmma<64> cin=256", "wgmma<64> cin=512",
    "dgrad ws<0>", "dgrad ws<0> bias=None", "dgrad wgmma<64> resident", "dgrad wgmma<64> streamed",
    "dgrad wgmma<64> cin=256", "dgrad wgmma<64> cin=512",
    "wgmma<16> out_f32", "wgmma<16> fnet head", "fp32 output stage + residual", "fp32 output stage tanh24",
    "wgrad padded channels", "wgrad several tiles", "wgrad ragged", "wgrad cin=51", "wgrad cin=64", "wgrad cout=3 run as 4",
    # FNet's backward
    "wgrad cin=6", "wgrad cin=32", "wgrad cin=128", "wgrad cin=256", "wgrad cout=32", "wgrad cout=128",
    "wgrad cout=256", "wgrad cout=2 run as 4", "dgrad wgmma<64> cin=128", "dgrad wgmma<64> nsplit>1",
}


def case_layers():
    """{case name: layers} over every table."""
    out = {"gen " + k: gen_layers(*v[:4]) for k, v in GEN_CASES.items()}
    out.update({"fnet " + k: fnet_layers(*v) for k, v in FNET_CASES.items()})
    out.update({"fnet backward " + k: fnet_layers(*v[:3], backward=True) for k, v in FNET_BWD_CASES.items()})
    out.update({"vgg " + k: vgg_layers(*v) for k, v in VGG_CASES.items()})
    return out


def fnet_seed(name, signed):
    return 5100 + 10 * sorted(FNET_CASES).index(name) + int(signed)


def vgg_seed(name):
    return 5200 + sorted(VGG_CASES).index(name)
