"""generator_F and fnet in float64, rounded exactly where the bf16 plans of tecogan_b200/tc_nets.py round, and the
operands on which that restatement is exact, so GeneratorPlan and FNetPlan can be compared with it bit for bit.

The reference walks the oracle's parameter names and layer order (oracle/teco_oracle.py generator_F and fnet, i.e. the
reference's lib/frvsr.py), not tc_nets, so it cannot share the plans' wiring.  Rounding(on=False) makes every rounding
point the identity and the reference is then the oracle's own float64 arithmetic, op for op.  With rounding on:
  generator  x_in = bf16(inputs); input conv and conv_1: bf16(relu(conv + b)); conv_2: bf16((conv + b) + a);
             conv_tran1/2: bf16(relu(convT + b)); output: ((conv + b) + bic) * 2 - 1 in fp32, in the kernel's order, with
             bic given (the device's bicubic4, tested on its own in test_gpu_resample_exact.py);
  fnet       every conv: bf16(lrelu(conv + b)) with lrelu(v) = v >= 0 ? v : fp32(0.2f v); max-pool exact; the x2 resize
             the fp32 blend rounded once to bf16; the head tanh(conv + b) * 24.
Each conv's conv + b is first rounded to fp32, which is what the device computes when its fp32 accumulator holds the
exact sum of the products.  A check hook runs on every conv and resize before its result is used; the guards below make
it fail a layer whose operands leave the regime where that holds, instead of letting the case pass by luck:
  * exact_check: products on g = lsb(x) lsb(w), bias and residual on g, sum|terms| <= 2^22 g per output -- every
    partial sum is exact in fp32 whatever the MMA order (the argument of test_gpu_conv_exact.py), so is conv + b (+ res);
  * one_product_check: each output channel has one non-zero weight, a power of two, so the accumulator holds the single
    product x w exactly and the device rounds x w + b once; the float64 sum x w + b must itself be exact;
  * resize_check: every intermediate of the kernel's blend (x1 - x0, x0 + d / 2, bottom - top, top + e / 2) is exact in
    fp32, so no FMA contraction or order of the kernel can change the blend.
Operand sets (builders below):
  generator  inputs k/16, a dense input conv with weights m/128 and biases on 2^-11, sparse +-1 weights with biases on
             2^-11 everywhere else (trunk, both transposed convs, the 64 -> 3 output conv): every buffer on 2^-11;
  fnet "nonneg"  frames k/16 in [0, 1], non-negative sparse weights m/64 (about eight per output) and biases in
             [0.5, 1) on 2^-10: LeakyReLU is the identity, every buffer from encoder_1 on is >= 0.5, so on 2^-8, and
             below 256 -- every conv, pool and resize up to the head is exact and mixes many inputs; the head's weights
             are signed m/1024;
  fnet "signed"  encoder_1/conv_1 dense signed m/128 (exact regime), then every output channel of every later layer,
             the head included, reads one input channel at one tap through +-2^-3 or +-2^-4 and adds an fp32 bias of
             magnitude in [1, 2): |x w| < 0.35, so every pre-activation is a rounded fp32 value of magnitude in
             [0.65, 2.35], LeakyReLU's negative branch runs on about half of each layer's channels, and every buffer
             stays within a few binades, so the resize blends stay exact.
Feature names for the case tables (gen_features, fnet_features) restate the plans' choices on the host the way
tests/conv_paths.py restates the kernels' dispatch."""
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import teco_oracle as O
from tests.conv_paths import MAX_CLUSTERS, MAX_SLOTS, TILE_COLS, TILE_ROWS, tiles
from tests.test_gpu_conv_exact import _assert_exact_regime, _grid, _is_f32

GEN = "generator/generator_unit/"
FNET = "fnet/autoencode_unit/"
ENCODERS = ("encoder_1", "encoder_2", "encoder_3")
DECODERS = ("decoder_1", "decoder_2", "decoder_3")
_F32_02 = torch.tensor(np.float32(0.2), dtype=torch.float32)


# ------------------------------------------------------------------------------------------------------ rounding points
class Rounding:
    """The device's rounding points (on) or none (off: the oracle's float64 arithmetic).  check(kind, what, *operands) is
    called before every conv (kind 'conv': x, w, b, residual or None) and resize (kind 'resize': its input)."""

    def __init__(self, on=True, check=None):
        self.on, self.check = on, check

    def f32(self, v):
        return v.float().double() if self.on else v

    def bf16(self, v):
        return v.float().to(torch.bfloat16).double() if self.on else v

    def add(self, a, b):
        """a + b of two fp32 values, rounded once to fp32 (the epilogues' residual adds)."""
        return (a.float() + b.float()).double() if self.on else a + b

    def lrelu(self, z):
        if not self.on:
            return O.lrelu(z)
        z32 = z.float()
        return torch.where(z32 >= 0, z32, _F32_02.to(z32.device) * z32).double()

    def preprocess(self, v):
        return O.preprocess(v.float()).double() if self.on else O.preprocess(v)

    def conv(self, what, x, w, b, res=None, transpose=False):
        if self.check is not None:
            self.check("conv", what, x, w, b, res, transpose)
        op = O.conv2d_transpose if transpose else O.conv2d
        return self.f32(op(x, w, b))

    def resize(self, what, x):
        if self.check is not None:
            self.check("resize", what, x)
        oh, ow = x.shape[1] * 2, x.shape[2] * 2
        y = O.resize_bilinear_legacy(x.cpu(), oh, ow).to(x.device)   # the oracle builds its weights on the CPU
        return self.bf16(y)


# --------------------------------------------------------------------------------------------------------- references
def generator_ref(p, gen_inputs, num_resblock, R, bic=None):
    """O.generator_F with R's rounding points; returns every buffer GeneratorPlan exposes (x_in in reference channel
    order, 51 channels).  bic: bicubic_four of the LR frame (default: the oracle's)."""
    def w_b(name):
        return p[GEN + name + "/weights"], p[GEN + name + "/biases"]

    out = {}
    x = out["x_in"] = R.bf16(gen_inputs)
    net = out["a"] = R.bf16(F.relu(R.conv("input_stage", x, *w_b("input_stage/conv/Conv"))))
    for i in range(1, num_resblock + 1):
        r = out["b"] = R.bf16(F.relu(R.conv("resblock_%d/conv_1" % i, net, *w_b("resblock_%d/conv_1/Conv" % i))))
        net = out["a"] = R.bf16(R.add(R.conv("resblock_%d/conv_2" % i, r, *w_b("resblock_%d/conv_2/Conv" % i), res=net), net))
    for i in (1, 2):
        name = "conv_tran2highres/conv_tran%d/Conv2d_transpose" % i
        net = out["u%d" % i] = R.bf16(F.relu(R.conv("conv_tran%d" % i, net, *w_b(name), transpose=True)))
    net = R.conv("output_stage", net, *w_b("output_stage/conv/Conv"))
    if bic is None:
        bic = O.bicubic_four(gen_inputs[..., 0:3])
    out["out"] = R.preprocess(R.add(net, bic))
    return out


def fnet_ref(p, fnet_input, R):
    """O.fnet with R's rounding points; returns x_in, levels [(conv_1 output, conv_2 output, pooled / resized)] for
    encoder_1 .. decoder_3, the head's first conv output o1, the head's pre-activation z and the flow."""
    def layer(name, x):
        w, b = p[FNET + name + "/weights"], p[FNET + name + "/biases"]
        return R.bf16(R.lrelu(R.conv(name, x, w, b)))

    out = {"levels": []}
    net = out["x_in"] = R.bf16(fnet_input)
    for name in ENCODERS + DECODERS:
        t1 = layer(name + "/conv_1/Conv", net)
        t2 = layer(name + "/conv_2/Conv", t1)
        net = O.maxpool(t2) if name in ENCODERS else R.resize(name, t2)
        out["levels"].append((t1, t2, net))
    o1 = out["o1"] = layer("output_stage/conv1/Conv", net)
    w, b = p[FNET + "output_stage/conv2/Conv/weights"], p[FNET + "output_stage/conv2/Conv/biases"]
    z = out["z"] = R.conv("output_stage/conv2/Conv", o1, w, b)
    out["flow"] = torch.tanh(z) * 24.0
    return out


# ------------------------------------------------------------------------------------------------------------ guards
def _cpu(t):
    return None if t is None else t.cpu()


def exact_check(what, x, w, b, res, transpose):
    op = O.conv2d_transpose if transpose else O.conv2d
    s_terms = op(x.abs(), w.abs()) + b.abs() + (res.abs() if res is not None else 0.0)
    _assert_exact_regime(what, _cpu(x), _cpu(w), s_terms, _cpu(b), *([_cpu(res)] if res is not None else []))


def one_product_check(what, x, w, b, res, transpose):
    assert res is None and not transpose, what + ": one-product layers have no residual and are not transposed"
    nz = (w != 0).reshape(-1, w.shape[-1]).sum(0)
    assert bool((nz == 1).all()), what + ": an output channel has %d non-zero weights" % int(nz.max())
    m, _ = torch.frexp(w[w != 0])
    assert bool((m.abs() == 0.5).all()), what + ": a weight is not a power of two"
    assert bool((x.float().to(torch.bfloat16).double() == x).all()), what + ": input not bf16"
    acc = O.conv2d(x, w)
    assert _is_f32(acc), what + ": x w not exact in fp32"
    z = acc + b
    bb = z - acc                              # TwoSum: the float64 sum is exact iff its error term is zero
    assert bool((((acc - (z - bb)) + (b - bb)) == 0).all()), what + ": x w + b not exact in float64"


def resize_check(what, x):
    """Every intermediate of resize2x_bf16_kernel's fp32 blend is exact in fp32 (x: [n, h, w, c] float64, bf16 values)."""
    n, h, w, c = x.shape
    iy, ix = torch.arange(2 * h, device=x.device), torch.arange(2 * w, device=x.device)
    y0, x0 = iy >> 1, ix >> 1
    y1 = torch.where(iy & 1 == 1, torch.clamp(y0 + 1, max=h - 1), y0)
    x1 = torch.where(ix & 1 == 1, torch.clamp(x0 + 1, max=w - 1), x0)
    wy = torch.where(iy & 1 == 1, 0.5, 0.0).double().view(1, -1, 1, 1)
    wx = torch.where(ix & 1 == 1, 0.5, 0.0).double().view(1, 1, -1, 1)
    a, bt = x[:, y0], x[:, y1]
    terms = []
    for row in (a, bt):
        d = row[:, :, x1] - row[:, :, x0]
        terms += [d, d * wx, row[:, :, x0] + d * wx]
    e = terms[5] - terms[2]
    terms += [e, e * wy, terms[2] + e * wy]
    for i, t in enumerate(terms):
        assert _is_f32(t), "%s: resize blend intermediate %d not exact in fp32" % (what, i)


def nets_check(kind, what, *args):
    """The guard of every case: exact_check, or one_product_check where every output channel has one non-zero weight;
    resize_check on every resize."""
    if kind == "resize":
        return resize_check(what, *args)
    x, w, b, res, transpose = args
    if not transpose and res is None and bool(((w != 0).reshape(-1, w.shape[-1]).sum(0) == 1).all()):
        return one_product_check(what, *args)
    return exact_check(what, *args)


# ------------------------------------------------------------------------------------------------------------ operands
def _sparse(rng, shape, density, values):
    keep = rng.rand(*shape) < density
    return torch.from_numpy(np.where(keep, values, 0.0) + 0.0)


def generator_operands(seed, B, h, w, N):
    """(params, inputs [B, h, w, 51]) on the grids above, float64.  Image i depends only on (seed, i), so the first k
    images of a batch are the k images of the smaller batch."""
    rng = np.random.RandomState(seed)
    p = {}
    p[GEN + "input_stage/conv/Conv/weights"] = _grid(rng, (3, 3, 51, 64), 2.0 ** -7, 16)
    p[GEN + "input_stage/conv/Conv/biases"] = _grid(rng, (64,), 2.0 ** -11, 2048)

    def sparse_layer(name, shape, density, bias_k):
        p[GEN + name + "/weights"] = _sparse(rng, shape, density, rng.choice([-1.0, 1.0], size=shape))
        p[GEN + name + "/biases"] = _grid(rng, (shape[2] if "transpose" in name else shape[3],), 2.0 ** -11, bias_k)
    for i in range(1, N + 1):
        sparse_layer("resblock_%d/conv_1/Conv" % i, (3, 3, 64, 64), 1.0 / 576, 256)
        sparse_layer("resblock_%d/conv_2/Conv" % i, (3, 3, 64, 64), 1.0 / 576, 256)
    for i in (1, 2):
        sparse_layer("conv_tran2highres/conv_tran%d/Conv2d_transpose" % i, (3, 3, 64, 64), 6.0 / 576, 512)
    sparse_layer("output_stage/conv/Conv", (3, 3, 64, 3), 6.0 / 576, 2048)
    x = torch.stack([_grid(np.random.RandomState([seed, i]), (h, w, 51), 2.0 ** -4, 16) for i in range(B)])
    return p, x


def fnet_operands(seed, n, h, w, signed):
    """(params, frame pairs [n, h, w, 6]) of operand set 'signed' or 'nonneg' (see the module docstring), float64."""
    rng = np.random.RandomState(seed)
    p = {}
    layers = [(name + "/conv_%d/Conv" % k, cin if k == 1 else cout, cout)
              for name, cin, cout in O.FNET_LAYERS for k in (1, 2)]
    layers += [("output_stage/conv1/Conv", 64, 32), ("output_stage/conv2/Conv", 32, 2)]
    for li, (name, cin, cout) in enumerate(layers):
        shape = (3, 3, cin, cout)
        head = li == len(layers) - 1
        if signed and li == 0:
            wt = _grid(rng, shape, 2.0 ** -7, 4)
            b = _grid(rng, (cout,), 2.0 ** -11, 2048)
        elif signed:
            flat = np.zeros((9 * cin, cout))
            flat[rng.randint(0, 9 * cin, size=cout), np.arange(cout)] = (
                rng.choice([-1.0, 1.0], size=cout) * 2.0 ** -rng.randint(3, 5, size=cout))
            wt = torch.from_numpy(flat.reshape(shape) + 0.0)
            b = torch.from_numpy(rng.choice([-1.0, 1.0], size=cout) *
                                 rng.uniform(1.0, 2.0, size=cout).astype(np.float32).astype(np.float64))
        elif head:
            wt = _sparse(rng, shape, 8.0 / (9 * cin), rng.randint(-16, 17, size=shape) / 1024.0)
            b = _grid(rng, (cout,), 2.0 ** -11, 1024)
        else:
            wt = _sparse(rng, shape, 8.0 / (9 * cin), rng.randint(1, 17, size=shape) / 64.0)
            b = torch.from_numpy(0.5 + rng.randint(0, 512, size=cout) * 2.0 ** -10)
        p[FNET + name + "/weights"], p[FNET + name + "/biases"] = wt, b
    x = torch.stack([torch.from_numpy(np.random.RandomState([seed, i]).randint(0, 17, size=(h, w, 6)) / 16.0)
                     for i in range(n)])
    return p, x


# ------------------------------------------------------------------------------------------------------ case tables
# Generator cases: batch B = b_g * G + b_1 with G = teco_conv3x3_lin_clusters() (MAX_CLUSTERS on a full H100 SXM), LR
# size, residual blocks, and the trunk route: True / False forces plan.lin, None keeps the plan's own choice.
GenCase = namedtuple("GenCase", "b_g b_1 h w N lin")
GEN_CASES = {
    "B=G lin": GenCase(1, 0, 32, 32, 16, None),
    "B=G per-layer": GenCase(1, 0, 32, 32, 16, False),
    "B=2G+1 lin": GenCase(2, 1, 32, 32, 16, True),
    "36x45": GenCase(0, 1, 36, 45, 16, None),
    "N=10 per-layer": GenCase(0, 4, 32, 32, 10, None),
    "N=10 lin": GenCase(0, 4, 32, 32, 10, True),
}
GEN_REQUIRED = {"gen trunk one launch", "gen trunk per layer", "gen trunk one launch, clusters run 3 clips",
                "gen N=16", "gen N=10", "gen ragged LR tiles", "gen ragged HR tiles", "gen HR width 180"}

FNET_SHAPES = {"264x32x32": (264, 32, 32), "1x144x176": (1, 144, 176), "3x40x56": (3, 40, 56), "5x8x8": (5, 8, 8)}
FNET_REQUIRED = (
    {"fnet %s on %s" % (name, path) for name in ENCODERS + DECODERS for path in ("im2col", "conv3x3_tc")} |
    {"fnet %s pool fused" % name for name in ENCODERS[:2]} | {"fnet %s pool separate" % name for name in ENCODERS} |
    {"fnet pool separate after conv3x3_tc", "fnet tiles>grid", "fnet odd level size",
     "fnet 1x1 bottom"})


def gen_seed(name):
    return 1000 + sorted(GEN_CASES).index(name)


def fnet_seed(shape, signed):
    return 2000 + 10 * sorted(FNET_SHAPES).index(shape) + int(signed)


def gen_batch(c, G):
    return c.b_g * G + c.b_1


def gen_lin(c, G):
    """plan.lin as the case runs it: forced, or tc_nets' own rule (32 x 32, the batch fills 0.8 of its rounds)."""
    if c.lin is not None:
        return c.lin
    B = gen_batch(c, G)
    return c.h == 32 and c.w == 32 and B >= 0.8 * G * -(-B // G)


def gen_features(c, G=MAX_CLUSTERS):
    B = gen_batch(c, G)
    out = {"gen N=%d" % c.N, "gen HR width %d" % (4 * c.w)}
    if gen_lin(c, G):
        out.add("gen trunk one launch")
        if -(-B // G) >= 3:
            out.add("gen trunk one launch, clusters run 3 clips")
    else:
        out.add("gen trunk per layer")
    if c.h % TILE_ROWS or c.w % TILE_COLS:
        out.add("gen ragged LR tiles")            # the trunk and conv_tran1 run partial 16 x 8 tiles
    if (2 * c.h) % TILE_ROWS or (2 * c.w) % TILE_COLS or (4 * c.w) % TILE_COLS:
        out.add("gen ragged HR tiles")            # conv_tran2 or the output stage does
    return out


def fnet_level_sizes(h, w):
    """(H, W) of each level's convolutions, encoder_1 .. decoder_3."""
    sizes = [(h, w)]
    for _ in range(3):
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    for _ in range(2):
        sizes.append((sizes[-1][0] * 2, sizes[-1][1] * 2))
    return sizes


def fnet_small(h, w):
    """Per level: runs on teco_conv3x3_im2col_tc (a level smaller than one 16 x 8 tile of an image)."""
    return [lh < TILE_ROWS or lw < TILE_COLS for lh, lw in fnet_level_sizes(h, w)]


def fnet_fused(h, w):
    """Per level: the max-pool is fused into conv_2 (an encoder on conv3x3_tc whose conv_2 has one 64-channel block)."""
    small = fnet_small(h, w)
    return [i < 3 and not small[i] and -(-cout // 64) == 1 for i, (_, _, cout) in enumerate(O.FNET_LAYERS)]


def fnet_features(n, h, w):
    small, fused = fnet_small(h, w), fnet_fused(h, w)
    out = set()
    for i, (name, _, _) in enumerate(O.FNET_LAYERS):
        out.add("fnet %s on %s" % (name, "im2col" if small[i] else "conv3x3_tc"))
        if i < 3:
            out.add("fnet %s pool %s" % (name, "fused" if fused[i] else "separate"))
            if not fused[i] and not small[i]:
                out.add("fnet pool separate after conv3x3_tc")
    sizes = fnet_level_sizes(h, w)
    if any(lh % 2 or lw % 2 for lh, lw in sizes[:4]):
        out.add("fnet odd level size")
    if sizes[3] == (1, 1):
        out.add("fnet 1x1 bottom")
    if tiles(n, h, w) > MAX_SLOTS:
        out.add("fnet tiles>grid")                # encoder_1's persistent tile walk wraps
    return out
