"""Case tables of tests/test_gpu_conv_simt_exact.py: the fp32 direct convolution teco_conv2d_f32 and its weight gradient
teco_conv2d_wgrad_f32 (csrc/conv_simt.cu), float64 restatements of both in the kernels' order, seeded grid operands, and a
host restatement of the launch geometry that classifies which edges each case reaches.

Why bit equality can be required (the argument of tests/test_gpu_conv_exact.py): x = k/16 and w = m/128 (or dy = m/128)
with |k|, |m| <= 16, so every product is a multiple of g = 2^-11; bias, residual and a prior dw sit on 2^-11 too, and a
prior db and the dy it sums on 2^-7.  If the sum of the magnitudes of an output's terms is at most 2^22 g, every partial
sum is a multiple of g below 2^23 g, an fp32 number, whatever the tile order, the split of the pixel range, the atomic
order, and whether the compiler contracted a multiply into the add.  `fwd_ref` / `wgrad_ref` return that sum of
magnitudes next to the value, and `guard` checks it per output.  Large-M weight-gradient cases use operands in
{-1, 0, 1} / 16 and {-1, 0, 1} / 128 so that they stay inside it.

What the epilogue does to the exact z = acc + bias is restated in numpy float32 (`epilogue`): act, + res, then
v * post_scale + post_shift.  Where the compiler may contract a multiply with the add after it (LeakyReLU's 0.2f * v
followed by a residual, and the post transform) both roundings are candidates; the contracted one is computed in float64,
which `_fma` checks is exact, and rounded once.  tanh * 24 and the sigmoid are returned as a float64 value and held to
a relative bound.

Launch geometry restated here (conv_simt.cu):
  forward       grid = (ceil(M / 64), ceil(Cout / 64)), M = N OH OW; cchunks = ceil(Cin / 16) channel chunks per tap;
                A loads four channels at once when Cin % 4 == 0 and in_cpitch % 4 == 0 (a_vec), B when Cout % 4 == 0.
  weight grad   ci_tiles = ceil(Cin / 64), co_tiles = ceil(Cout / 64), base = ci_tiles KH KW co_tiles;
                splits = ceil(4 SMs / base), capped at ceil(M / 256) and at least 1; pps = ceil(M / splits) rounded up to
                16; splits = ceil(M / pps).  A is vectorised as in the forward, B when Cout % 4 == 0 and
                out_cpitch % 4 == 0.
`keys(family, name, sms)` classifies a case at 132 SMs (H100 SXM); the GPU test recomputes it from the device.

LAYERS lists every teco_conv2d_f32 / teco_conv2d_wgrad_f32 launch the networks make, keyed by `launch_key`, for each
of the runs of the GPU census test; LAYER_CASES turns each key into a case at a small spatial size.
"""
from collections import namedtuple

import numpy as np

from tests.resample_cases import rng

BM, BN, BK = 64, 64, 16
NONE, RELU, LRELU, TANH24, SIGMOID = range(5)
ACT_NAMES = ("none", "relu", "lrelu", "tanh24", "sigmoid")
G = 2.0 ** -11                      # grid of every product, bias, residual and prior dw
G_DB = 2.0 ** -7                    # grid of dy and of the bias gradient
EXACT_SPAN = 2.0 ** 22
REL_BOUND = 2.0 ** -21              # tanhf / expf: 2 ulp each, * 24, 1 + e and the division 1/2 ulp each
F02 = np.float32(0.2)
ID_MAP = (1, 0, 1, 0)


def _cdiv(a, b):
    return -(-a // b)


def same_pad(n, k, s):
    """TF 'SAME' padding before, and the output size (kernels.same_pad)."""
    out = _cdiv(n, s)
    return max((out - 1) * s + k - n, 0) // 2, out


def phase_taps(k, pad, a):
    from tecogan_b200.kernels import _phase_taps
    return _phase_taps(k, pad, a)


# ------------------------------------------------------------------------------------------------------ descriptors
# One teco_conv2d_f32 launch.  x [N,H,W,in_cp] (channels >= Cin hold NaN), w [KH,KW,Cin,Cout], y [N,out_H,out_W,out_cp]
# with output pixel (oy, ox) at (oy sy + oy0, ox sx + ox0), out_map = (sy, oy0, sx, ox0).  post = (scale, shift).
Fwd = namedtuple("Fwd", "N H W OH OW out_H out_W KH KW stride pad_t pad_l Cin Cout in_cp out_cp out_map act bias res post")
# One teco_conv2d_wgrad_f32 launch: x as above, dy [N,out_H,out_W,out_cp] read through out_map; dw [KH,KW,Cin,Cout].
# ops: "grid" (x k/16, dy m/128, |k|, |m| <= 16) or "unit" (k, m in {-1, 0, 1}).
Wg = namedtuple("Wg", "N H W OH OW out_H out_W KH KW stride pad_t pad_l Cin Cout in_cp out_cp out_map accumulate db ops")


def fwd(N, H, W, KH, KW, Cin, Cout, *, stride=1, pad=None, OH=None, OW=None, in_cp=None, out_cp=None, out_map=ID_MAP,
        act=NONE, bias=True, res=False, post=(1.0, 0.0)):
    pad_t, pad_l = pad if pad is not None else (same_pad(H, KH, stride)[0], same_pad(W, KW, stride)[0])
    OH = same_pad(H, KH, stride)[1] if OH is None else OH
    OW = same_pad(W, KW, stride)[1] if OW is None else OW
    sy, _, sx, _ = out_map
    return Fwd(N, H, W, OH, OW, OH * sy, OW * sx, KH, KW, stride, pad_t, pad_l, Cin, Cout, in_cp or Cin, out_cp or Cout,
               tuple(out_map), act, bias, res, tuple(post))


def wg(N, H, W, KH, KW, Cin, Cout, *, stride=1, pad=None, OH=None, OW=None, in_cp=None, out_cp=None, out_map=ID_MAP,
       accumulate=0, db=True, ops="grid"):
    f = fwd(N, H, W, KH, KW, Cin, Cout, stride=stride, pad=pad, OH=OH, OW=OW, in_cp=in_cp, out_cp=out_cp, out_map=out_map)
    return Wg(f.N, f.H, f.W, f.OH, f.OW, f.out_H, f.out_W, f.KH, f.KW, f.stride, f.pad_t, f.pad_l, f.Cin, f.Cout, f.in_cp,
              f.out_cp, f.out_map, accumulate, db, ops)


def launch_key(c):
    """(entry, KH, KW, stride, pad_t, pad_l, Cin, Cout, in_cpitch, out_cpitch, out_map, act, bias?, res?, post,
    accumulate, db?) of a case; N, H and W are free."""
    if isinstance(c, Fwd):
        return ("fwd", c.KH, c.KW, c.stride, c.pad_t, c.pad_l, c.Cin, c.Cout, c.in_cp, c.out_cp, c.out_map, c.act,
                bool(c.bias), bool(c.res), tuple(float(v) for v in c.post), 0, False)
    return ("wgrad", c.KH, c.KW, c.stride, c.pad_t, c.pad_l, c.Cin, c.Cout, c.in_cp, c.out_cp, c.out_map, NONE, False,
            False, (1.0, 0.0), int(c.accumulate), bool(c.db))


def desc_key(entry, d, bias=False, res=False, accumulate=0, db=False):
    """launch_key of a recorded call: d is the ConvDesc it was given."""
    m = (d.out_sy, d.out_oy, d.out_sx, d.out_ox)
    if entry == "fwd":
        return ("fwd", d.KH, d.KW, d.stride, d.pad_t, d.pad_l, d.Cin, d.Cout, d.in_cpitch, d.out_cpitch, m, d.act,
                bool(bias), bool(res), (float(d.post_scale), float(d.post_shift)), 0, False)
    return ("wgrad", d.KH, d.KW, d.stride, d.pad_t, d.pad_l, d.Cin, d.Cout, d.in_cpitch, d.out_cpitch, m, NONE, False,
            False, (1.0, 0.0), int(accumulate), bool(db))


# -------------------------------------------------------------------------------------------------------- layer table
# The launches of kernels._Conv2d / _ConvTranspose2x for one network layer, at the spatial size `hw` of its input.
def conv_launches(Cin, Cout, K=3, stride=1, act=NONE, bias=True, res=False, dgrad=True, wgrad=True, grad=True,
                  N=2, hw=(9, 11)):
    H, W = hw
    f = fwd(N, H, W, K, K, Cin, Cout, stride=stride, act=act, bias=bias, res=res)
    out = [f]
    if not grad:
        return out
    if dgrad and stride == 1:
        out.append(fwd(N, f.OH, f.OW, K, K, Cout, Cin, pad=(K - 1 - f.pad_t, K - 1 - f.pad_l), OH=H, OW=W, bias=False))
    elif dgrad:
        assert stride == 2 and H % 2 == 0 and W % 2 == 0 and f.pad_t == f.pad_l
        out += transpose_phases(N, f.OH, f.OW, K, Cout, Cin, f.pad_t, NONE, False)
    if wgrad:
        out.append(wg(N, H, W, K, K, Cin, Cout, stride=stride, pad=(f.pad_t, f.pad_l), OH=f.OH, OW=f.OW, db=bias))
    return out


def transpose_phases(N, H, W, K, Cin, Cout, pad, act, bias):
    """The four sub-pixel launches of kernels.conv_transpose2x_raw: x [N,H,W,Cin] -> y [N,2H,2W,Cout]."""
    out = []
    for a in (0, 1):
        kys, pt = phase_taps(K, pad, a)
        for b in (0, 1):
            kxs, pl = phase_taps(K, pad, b)
            out.append(fwd(N, H, W, len(kys), len(kxs), Cin, Cout, pad=(pt, pl), OH=H, OW=W, out_map=(2, a, 2, b),
                           act=act, bias=bias))
    return out


def tconv_launches(Cin, Cout, act=RELU, N=2, hw=(5, 7), grad=True):
    H, W = hw
    out = transpose_phases(N, H, W, 3, Cin, Cout, 0, act, True)
    if grad:
        out.append(fwd(N, 2 * H, 2 * W, 3, 3, Cout, Cin, stride=2, pad=(0, 0), OH=H, OW=W, bias=False))
        out.append(wg(N, 2 * H, 2 * W, 3, 3, Cout, Cin, stride=2, pad=(0, 0), OH=H, OW=W, db=False))
    return out


def generator_launches(grad=True):
    out = conv_launches(51, 64, act=RELU, grad=grad)
    out += conv_launches(64, 64, act=RELU, grad=grad) + conv_launches(64, 64, res=True, grad=grad)
    out += tconv_launches(64, 64, grad=grad)
    return out + conv_launches(64, 3, res=True, grad=grad)


FNET = [(6, 32), (32, 32), (32, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 128), (128, 128),
        (128, 64), (64, 64), (64, 32)]


def fnet_launches(grad=True):
    out = []
    for i, (ci, co) in enumerate(FNET):
        out += conv_launches(ci, co, act=LRELU, dgrad=i > 0, grad=grad)
    return out + conv_launches(32, 2, act=TANH24, grad=grad)


VGG = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 256), (256, 512),
       (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512)]


def vgg_launches(dgrad_layers):
    """VGG19's frozen convolutions: forward on all sixteen, the input gradient through the first `dgrad_layers`."""
    out = []
    for i, (ci, co) in enumerate(VGG):
        out += conv_launches(ci, co, act=RELU, dgrad=i < dgrad_layers, wgrad=False, hw=(6, 5))
    return out


DISC_BLOCKS = [(64, 64), (64, 64), (64, 128), (128, 256)]


def disc_launches(grad=True):
    out = conv_launches(27, 64, act=LRELU, grad=grad)
    for ci, co in DISC_BLOCKS:
        out += conv_launches(ci, co, K=4, stride=2, bias=False, hw=(10, 12), grad=grad)
    return out + conv_launches(256, 1, K=1, hw=(3, 5), grad=grad)


def lpips_launches():
    """LPIPS-AlexNet's five convolutions (lpips.ALEXNET_CONVS): relu1 of a 35 x 39 crop is 8 x 9 and reads taps past its
    bottom and right edges; relu2 .. relu5 at 3 x 4 (a 3 x 4 pool output)."""
    return [fwd(2, 35, 39, 11, 11, 3, 64, stride=4, pad=(2, 2), OH=8, OW=8 + 1, act=RELU),
            fwd(2, 3, 4, 5, 5, 64, 192, pad=(2, 2), OH=3, OW=4, act=RELU),
            fwd(2, 3, 4, 3, 3, 192, 384, pad=(1, 1), OH=3, OW=4, act=RELU),
            fwd(2, 3, 4, 3, 3, 384, 256, pad=(1, 1), OH=3, OW=4, act=RELU),
            fwd(2, 3, 4, 3, 3, 256, 256, pad=(1, 1), OH=3, OW=4, act=RELU)]


VGG_DGRAD_LAYERS = 16
# run of the census test -> its launches.  A trainer's constructor materialises its variables with one no-grad forward
# of the graph at fp32 precision (lib/Teco.py), so a bf16 TecoGAN step also launches the forward of every generator,
# FNet and discriminator layer here; VGG19 is not among them, as in bf16 training it always runs on wgmma.  In the step
# itself only the discriminator's dense layer (1 x 1, Cout 1) takes this kernel, forward and both gradients.
LAYER_RUNS = {
    "fp32 FRVSR step": lambda: generator_launches() + fnet_launches(),
    "fp32 TecoGAN step": lambda: generator_launches() + fnet_launches() + vgg_launches(VGG_DGRAD_LAYERS) + disc_launches(),
    "bf16 TecoGAN step": lambda: (generator_launches(grad=False) + fnet_launches(grad=False) + disc_launches(grad=False)
                                  + conv_launches(256, 1, K=1, hw=(3, 5))),
    "fp32 inference": lambda: generator_launches(grad=False) + fnet_launches(grad=False),
    "LPIPS.features": lpips_launches,
}
LAYERS = {run: {launch_key(c) for c in make()} for run, make in LAYER_RUNS.items()}


def _layer_cases():
    seen = {}
    for make in LAYER_RUNS.values():
        for c in make():
            seen.setdefault(launch_key(c), c)
    out = {}
    for k, c in seen.items():
        if isinstance(c, Fwd):
            name = "layer fwd %dx%d s%d p%d,%d %d->%d map%s %s%s%s" % (
                c.KH, c.KW, c.stride, c.pad_t, c.pad_l, c.Cin, c.Cout, "".join(map(str, c.out_map)), ACT_NAMES[c.act],
                "" if c.bias else " nobias", " res" if c.res else "")
        else:
            name = "layer wgrad %dx%d s%d p%d,%d %d->%d%s" % (c.KH, c.KW, c.stride, c.pad_t, c.pad_l, c.Cin, c.Cout,
                                                             " db" if c.db else "")
        out[name] = c
    return out


LAYER_CASES = _layer_cases()

# ------------------------------------------------------------------------------------------------------- ABI edges
FWD_EDGES = {
    "tail_65_tiles_c8": fwd(3, 37, 37, 3, 3, 8, 8, act=RELU),
    "one_tile_cin13_cout3": fwd(1, 5, 7, 3, 3, 13, 3, act=LRELU),
    "cout1_sigmoid": fwd(2, 7, 9, 3, 3, 20, 1, act=SIGMOID),
    "cout2_tanh_pitched": fwd(2, 6, 5, 3, 3, 7, 2, act=TANH24, in_cp=9, out_cp=5),
    "cout100_cin36_pitch38_res": fwd(2, 9, 7, 3, 3, 36, 100, in_cp=38, out_cp=103, act=RELU, res=True),
    "cin512_cout130_1x1": fwd(2, 6, 7, 1, 1, 512, 130, act=NONE),
    "lrelu_res_post": fwd(2, 8, 9, 3, 3, 24, 68, act=LRELU, res=True, post=(-1.5, 0.25)),
    "none_nobias_post_half": fwd(3, 11, 13, 3, 3, 16, 64, bias=False, post=(0.5, -0.75)),
    "relu_res_nobias_pitched_out": fwd(2, 10, 6, 3, 3, 64, 64, act=RELU, bias=False, res=True, out_cp=67),
    "sigmoid_stride2_pad01": fwd(2, 13, 10, 3, 3, 12, 20, stride=2, pad=(0, 1), OH=6, OW=5, act=SIGMOID),
    "tanh_5x5_stride2_pad21": fwd(2, 14, 15, 5, 5, 8, 24, stride=2, pad=(2, 1), OH=7, OW=7, act=TANH24),
    "kernel_3x2_phase01_pad10": fwd(2, 6, 5, 3, 2, 40, 36, pad=(1, 0), OH=6, OW=5, out_map=(2, 0, 2, 1), act=LRELU,
                                    res=True),
    "phase10_in_pitch_out_pitch": fwd(1, 4, 9, 2, 2, 64, 70, pad=(0, 1), OH=4, OW=9, out_map=(2, 1, 2, 0),
                                      in_cp=66, out_cp=72, act=RELU, post=(2.0, 0.5)),
    "stride4_11x11_odd": fwd(1, 33, 37, 11, 11, 3, 5, stride=4, pad=(2, 3), OH=7, OW=8, act=NONE),
}

WGRAD_EDGES = {
    "one_split_c512": wg(1, 10, 15, 3, 3, 512, 512, db=False),
    "splits_short_last": wg(3, 37, 41, 3, 3, 16, 8),
    "ci_co_tiles_scalar_a": wg(2, 9, 10, 1, 1, 130, 70, in_cp=131),
    "scalar_b_out_pitch": wg(2, 12, 11, 3, 3, 20, 8, out_cp=10),
    "cout3_db": wg(2, 8, 8, 3, 3, 5, 3),
    "strided_map_acc": wg(2, 6, 7, 2, 2, 24, 12, pad=(1, 0), OH=6, OW=7, out_map=(2, 1, 2, 0), accumulate=1),
    "accumulate_stride2_4x4": wg(2, 12, 10, 4, 4, 12, 16, stride=2, accumulate=1),
    "large_m_unit_ops": wg(2, 300, 300, 1, 1, 4, 4, ops="unit"),
    "large_m_unit_ops_acc_nodb": wg(1, 257, 263, 3, 3, 8, 4, ops="unit", accumulate=1, db=False),
}

FAMILY_CASES = {"fwd": {**LAYER_CASES, **FWD_EDGES}, "wgrad": {**LAYER_CASES, **WGRAD_EDGES}}
FWD_CASES = {k: c for k, c in FAMILY_CASES["fwd"].items() if isinstance(c, Fwd)}
WGRAD_CASES = {k: c for k, c in FAMILY_CASES["wgrad"].items() if isinstance(c, Wg)}


# --------------------------------------------------------------------------------------------------- launch geometry
def fwd_launch(c):
    M = c.N * c.OH * c.OW
    return dict(M=M, tiles=_cdiv(M, BM), co_tiles=_cdiv(c.Cout, BN), cchunks=_cdiv(c.Cin, BK),
                a_vec=c.Cin % 4 == 0 and c.in_cp % 4 == 0, b_vec=c.Cout % 4 == 0)


def wgrad_launch(c, sms=132):
    M = c.N * c.OH * c.OW
    ci_tiles, co_tiles = _cdiv(c.Cin, BM), _cdiv(c.Cout, BN)
    base = ci_tiles * c.KH * c.KW * co_tiles
    splits = _cdiv(4 * sms, base)
    splits = max(1, min(splits, _cdiv(M, 256), 65535))
    pps = _cdiv(_cdiv(M, splits), BK) * BK
    return dict(M=M, ci_tiles=ci_tiles, co_tiles=co_tiles, splits=_cdiv(M, pps), pps=pps,
                a_vec=c.Cin % 4 == 0 and c.in_cp % 4 == 0, b_vec=c.Cout % 4 == 0 and c.out_cp % 4 == 0)


def _fwd_keys(name, sms):
    c = FWD_CASES[name]
    L = fwd_launch(c)
    k = {"fwd: act=" + ACT_NAMES[c.act], "fwd: stride=%d" % c.stride}
    k |= {"fwd: K=%d" % c.KH} if c.KH == c.KW else {"fwd: KH!=KW"}
    k |= {"fwd: M%64!=0"} if L["M"] % BM else set()
    k |= {"fwd: one pixel tile"} if L["tiles"] == 1 else set()
    k |= {"fwd: >64 pixel tiles"} if L["tiles"] > 64 else set()
    k |= {"fwd: Cout%64!=0"} if c.Cout % BN else set()
    k |= {"fwd: >1 Cout tile"} if L["co_tiles"] > 1 else set()
    k |= {"fwd: Cout=%d" % c.Cout} if c.Cout <= 3 else set()
    k |= {"fwd: scalar B"} if not L["b_vec"] else set()
    k |= {"fwd: Cin%16!=0"} if c.Cin % BK else set()
    k |= {"fwd: Cin%4!=0"} if c.Cin % 4 else set()
    k |= {"fwd: scalar A, Cin%4==0"} if c.Cin % 4 == 0 and not L["a_vec"] else set()
    k |= {"fwd: Cin=512"} if c.Cin == 512 else set()
    k |= {"fwd: in_cpitch>Cin"} if c.in_cp > c.Cin else set()
    k |= {"fwd: out_cpitch>Cout"} if c.out_cp > c.Cout else set()
    k |= {"fwd: phase map %d%d" % (c.out_map[1], c.out_map[3])} if c.out_map[0] == 2 else set()
    k |= {"fwd: pad_t!=pad_l"} if c.pad_t != c.pad_l else set()
    k |= {"fwd: taps past the bottom"} if (c.OH - 1) * c.stride - c.pad_t + c.KH > c.H else set()
    k |= {"fwd: taps past the right"} if (c.OW - 1) * c.stride - c.pad_l + c.KW > c.W else set()
    k |= {"fwd: residual"} if c.res else set()
    k |= {"fwd: no bias"} if not c.bias else set()
    k |= {"fwd: post!=(1,0)"} if c.post != (1.0, 0.0) else set()
    return k


def _wgrad_keys(name, sms):
    c = WGRAD_CASES[name]
    L = wgrad_launch(c, sms)
    k = {"wgrad: one split" if L["splits"] == 1 else "wgrad: several splits"}
    k |= {"wgrad: short last split"} if L["splits"] > 1 and L["M"] % L["pps"] else set()
    k |= {"wgrad: ci_tiles>1"} if L["ci_tiles"] > 1 else set()
    k |= {"wgrad: co_tiles>1"} if L["co_tiles"] > 1 else set()
    k |= {"wgrad: scalar A"} if not L["a_vec"] else set()
    k |= {"wgrad: scalar B, Cout%4==0"} if c.Cout % 4 == 0 and not L["b_vec"] else set()
    k |= {"wgrad: Cout%4!=0"} if c.Cout % 4 else set()
    k |= {"wgrad: strided out map"} if c.out_map != ID_MAP else set()
    k |= {"wgrad: stride=%d" % c.stride}
    k |= {"wgrad: accumulate"} if c.accumulate else {"wgrad: overwrite"}
    k |= {"wgrad: db"} if c.db else {"wgrad: db NULL"}
    k |= {"wgrad: sparse operands"} if c.ops == "unit" else set()
    return k


FAMILIES = {"fwd": (FWD_CASES, _fwd_keys), "wgrad": (WGRAD_CASES, _wgrad_keys)}

REQUIRED = {
    "fwd": {"fwd: M%64!=0", "fwd: one pixel tile", "fwd: >64 pixel tiles", "fwd: Cout%64!=0", "fwd: >1 Cout tile",
            "fwd: Cout=1", "fwd: Cout=2", "fwd: Cout=3", "fwd: scalar B", "fwd: Cin%16!=0", "fwd: Cin%4!=0",
            "fwd: scalar A, Cin%4==0", "fwd: in_cpitch>Cin", "fwd: out_cpitch>Cout", "fwd: pad_t!=pad_l",
            "fwd: taps past the bottom", "fwd: taps past the right", "fwd: residual", "fwd: no bias", "fwd: post!=(1,0)",
            "fwd: Cin=512"}
    | {"fwd: phase map %d%d" % (a, b) for a in (0, 1) for b in (0, 1)}
    | {"fwd: stride=%d" % s for s in (1, 2, 4)} | {"fwd: K=%d" % k for k in (1, 3, 4, 5, 11)}
    | {"fwd: act=" + a for a in ACT_NAMES},
    "wgrad": {"wgrad: one split", "wgrad: several splits", "wgrad: short last split", "wgrad: ci_tiles>1",
              "wgrad: co_tiles>1", "wgrad: scalar A", "wgrad: scalar B, Cout%4==0", "wgrad: Cout%4!=0",
              "wgrad: strided out map", "wgrad: accumulate", "wgrad: overwrite", "wgrad: db", "wgrad: db NULL",
              "wgrad: stride=2", "wgrad: sparse operands"},
}


def keys(family, name, sms=132):
    return FAMILIES[family][1](name, sms)


# ---------------------------------------------------------------------------------------------------------- operands
def _ints(r, shape, kmax):
    return r.randint(-kmax, kmax + 1, size=shape).astype(np.float64)


def _mapped(c, a):
    """The [N,OH,OW,Cout] view of an output-shaped array a [N,out_H,out_W,out_cp] at the case's output map."""
    sy, oy, sx, ox = c.out_map
    return a[:, oy:oy + (c.OH - 1) * sy + 1:sy, ox:ox + (c.OW - 1) * sx + 1:sx, :c.Cout]


def out_mask(c):
    """True where the launch writes: mapped pixels, channels < Cout."""
    m = np.zeros((c.N, c.out_H, c.out_W, c.out_cp), bool)
    _mapped(c, m)[...] = True
    return m


def fwd_inputs(name):
    """x [N,H,W,in_cp] (NaN beyond Cin), w [KH,KW,Cin,Cout], bias [Cout] or None, res [N,out_H,out_W,out_cp] or None
    (NaN outside the written elements), all float32."""
    c, r = FWD_CASES[name], rng("conv_simt fwd " + name)
    x = np.full((c.N, c.H, c.W, c.in_cp), np.nan, np.float32)
    x[..., :c.Cin] = _ints(r, (c.N, c.H, c.W, c.Cin), 16) / 16
    w = (_ints(r, (c.KH, c.KW, c.Cin, c.Cout), 16) / 128).astype(np.float32)
    b = (_ints(r, (c.Cout,), 2048) * G).astype(np.float32) if c.bias else None
    res = None
    if c.res:
        res = np.where(out_mask(c), _ints(r, (c.N, c.out_H, c.out_W, c.out_cp), 4096) * G, np.nan).astype(np.float32)
    return x, w, b, res


def wgrad_inputs(name):
    """x [N,H,W,in_cp], dy [N,out_H,out_W,out_cp] (NaN outside the read elements), dw0 [KH,KW,Cin,Cout] and db0 [Cout]
    (the prior contents the kernel accumulates onto, or the sentinel it overwrites), all float32."""
    c, r = WGRAD_CASES[name], rng("conv_simt wgrad " + name)
    kx, kd = (16, 16) if c.ops == "grid" else (1, 1)
    x = np.full((c.N, c.H, c.W, c.in_cp), np.nan, np.float32)
    x[..., :c.Cin] = _ints(r, (c.N, c.H, c.W, c.Cin), kx) / 16
    dy = np.where(out_mask(c), _ints(r, (c.N, c.out_H, c.out_W, c.out_cp), kd) / 128, np.nan).astype(np.float32)
    if c.accumulate:
        dw0 = (_ints(r, (c.KH, c.KW, c.Cin, c.Cout), 4096) * G).astype(np.float32)
        db0 = (_ints(r, (c.Cout,), 64) * G_DB).astype(np.float32)
    else:
        dw0 = np.full((c.KH, c.KW, c.Cin, c.Cout), 1e30, np.float32)
        db0 = np.full((c.Cout,), 1e30, np.float32)
    return x, dy, dw0, db0


# ------------------------------------------------------------------------------------------------ float64 restatements
def _patches(c, x):
    """For each tap (ky, kx): x at (oy stride - pad_t + ky, ox stride - pad_l + kx), zero outside the image, as
    [N,OH,OW,Cin] float64."""
    s = c.stride
    pb = max(0, (c.OH - 1) * s - c.pad_t + c.KH - c.H)
    pr = max(0, (c.OW - 1) * s - c.pad_l + c.KW - c.W)
    xp = np.zeros((c.N, c.H + c.pad_t + pb, c.W + c.pad_l + pr, c.Cin))
    xp[:, c.pad_t:c.pad_t + c.H, c.pad_l:c.pad_l + c.W] = x[..., :c.Cin]
    for ky in range(c.KH):
        for kx in range(c.KW):
            yield ky, kx, xp[:, ky:ky + (c.OH - 1) * s + 1:s, kx:kx + (c.OW - 1) * s + 1:s]


def fwd_ref(c, x, w, bias, res):
    """z = sum over taps and channels of x w + bias (float64, [N,OH,OW,Cout]) and the sum of the magnitudes of its terms
    with the residual's (the guard's operand)."""
    acc = np.zeros((c.N, c.OH, c.OW, c.Cout))
    mag = np.zeros_like(acc)
    w = np.asarray(w, np.float64)
    for ky, kx, p in _patches(c, np.asarray(x, np.float64)):
        acc += p @ w[ky, kx]
        mag += np.abs(p) @ np.abs(w[ky, kx])
    if bias is not None:
        acc += bias
        mag += np.abs(bias.astype(np.float64))
    if res is not None:
        mag += np.abs(_mapped(c, res.astype(np.float64)))
    return acc, mag


def _fma(a, b, s):
    """a * b + s rounded once to fp32 (float64 operands that are fp32 numbers: the product is exact in float64); asserts
    that the float64 sum is exact too (the error term of Knuth's two-sum is zero)."""
    p = a * b
    t = p + s
    bv = t - p
    err = (p - (t - bv)) + (s - bv)
    assert not np.any(err), "fused sum not exact in float64"
    return t.astype(np.float32)


def epilogue(c, z, res):
    """fp32 outputs the kernel may produce from the exact z (float64): a list of candidate arrays [N,OH,OW,Cout], or
    for tanh * 24 and the sigmoid (float64 value, bound)."""
    if c.act in (TANH24, SIGMOID):
        assert res is None and c.post == (1.0, 0.0), "the bound does not model a residual or the post transform"
        v = np.tanh(z) * 24.0 if c.act == TANH24 else 1.0 / (1.0 + np.exp(-z))
        return v, REL_BOUND * np.abs(v)
    z32 = z.astype(np.float32)
    assert np.array_equal(z32.astype(np.float64), z), "z is not an fp32 number"
    if c.act == RELU:
        v = [np.maximum(z32, np.float32(0))]
    elif c.act == LRELU:
        v = [np.where(z32 >= 0, z32, F02 * z32)]
    else:
        v = [z32]
    if res is not None:
        r = _mapped(c, res)
        out = [v[0] + r]
        if c.act == LRELU:           # fmaf(0.2f, v, res)
            out.append(np.where(z32 >= 0, out[0], _fma(np.float64(F02), z, r.astype(np.float64))))
        v = out
    ps, sh = np.float32(c.post[0]), np.float32(c.post[1])
    out = []
    for a in v:
        out.append(a * ps + sh)
        if c.post != (1.0, 0.0):     # fmaf(v, post_scale, post_shift)
            out.append(_fma(a.astype(np.float64), np.float64(ps), np.float64(sh)))
    return out


def wgrad_ref(c, x, dy, dw0, db0):
    """(dw, |dw| terms, db, |db| terms) in float64: dw[ky,kx,ci,co] = sum over output pixels of the tap's input times
    dy at the mapped position, db[co] = sum of dy; with accumulate, plus the prior contents."""
    d = _mapped(c, np.asarray(dy, np.float64)).reshape(-1, c.Cout)
    dw = np.zeros((c.KH, c.KW, c.Cin, c.Cout))
    mag = np.zeros_like(dw)
    for ky, kx, p in _patches(c, np.asarray(x, np.float64)):
        p = p.reshape(-1, c.Cin)
        dw[ky, kx] = p.T @ d
        mag[ky, kx] = np.abs(p).T @ np.abs(d)
    db, dbm = d.sum(0), np.abs(d).sum(0)
    if c.accumulate:
        dw, mag = dw + dw0, mag + np.abs(dw0.astype(np.float64))
        db, dbm = db + db0, dbm + np.abs(db0.astype(np.float64))
    return dw, mag, db, dbm


def guard(mag, g, what):
    """Every partial sum of every output is an fp32 number: sum|terms| <= 2^22 g."""
    worst = float(np.max(mag, initial=0.0))
    assert worst <= EXACT_SPAN * g, "%s: sum|terms| %.6g > 2^22 g = %.6g" % (what, worst, EXACT_SPAN * g)


def on_grid(a, g, what):
    a = np.asarray(a, np.float64)
    a = a[np.isfinite(a)]
    assert np.array_equal(a / g, np.round(a / g)), "%s: off the %g grid" % (what, g)


def fwd_guard(name):
    c = FWD_CASES[name]
    x, w, b, res = fwd_inputs(name)
    on_grid(x, 2.0 ** -4, name + " x")
    on_grid(w, 2.0 ** -7, name + " w")
    for a, n in ((b, "bias"), (res, "res")):
        if a is not None:
            on_grid(a, G, name + " " + n)
    guard(fwd_ref(c, x, w, b, res)[1], G, name)


def wgrad_guard(name):
    c = WGRAD_CASES[name]
    x, dy, dw0, db0 = wgrad_inputs(name)
    on_grid(x, 2.0 ** -4, name + " x")
    on_grid(dy, G_DB, name + " dy")
    if c.accumulate:
        on_grid(dw0, G, name + " dw0")
        on_grid(db0, G_DB, name + " db0")
    _, mag, _, dbm = wgrad_ref(c, x, dy, dw0, db0)
    guard(mag, G, name + " dw")
    guard(dbm, G_DB, name + " db")


# --------------------------------------------------------------------------------------------------- 3x3 / 2 max-pool
def maxpool3s2_ref(x):
    """torch MaxPool2d(3, 2) as lpips.cu's maxpool3s2_kernel states it: start at the window's first element, then in row
    order take v when v > m or v is NaN (so the first of tied maxima and the last NaN win)."""
    N, H, W, C = x.shape
    OH, OW = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    m = x[:, 0:2 * OH - 1:2, 0:2 * OW - 1:2].copy()
    for dy in range(3):
        for dx in range(3):
            v = x[:, dy:dy + 2 * OH - 1:2, dx:dx + 2 * OW - 1:2]
            take = (v > m) | np.isnan(v)
            m = np.where(take, v, m)
    return m
