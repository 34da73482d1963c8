"""Every bf16 tensor-core convolution path -- teco_conv3x3_tc on each kernel instance it dispatches to, the multi-layer
chain teco_conv3x3_lin_tc and the weight gradient teco_conv3x3_wgrad_tc -- against a float64 reference, bit for bit.

Why bit equality can be required: products of bf16 operands are exact in fp32.  If every product, bias and residual of an
output is a multiple of a grid unit g and the sum of their magnitudes is at most 2^22 g, every partial sum is a multiple of
g below 2^23 g, so it is representable in fp32 (one bit of margin under the 24-bit significand).  The fp32 accumulator
then holds the exact float64 value whatever the MMA order, K-step split, persistent-tile walk or atomic order.  The
operands below sit on such grids -- x = k/16 and weights m/128 with |k|, |m| <= 16 (products on 2^-11), bias, residuals
and fp32 residuals on 2^-11 -- and a host guard (_assert_exact_regime) checks the condition per output before comparing,
so a case that leaves the regime fails instead of passing by luck.  What is left is the epilogue, restated in the
kernels' order: + bias, activation, + residual, round to nearest even (torch's bf16 conversion):
  * none / ReLU: exact, and the bf16 rounding alone is checked; each such case must hit exact rounding midpoints, so
    ties-to-even is exercised;
  * LeakyReLU: np.float32(0.2) * v rounded to fp32; followed by a residual, nvcc may contract the multiply and the add
    into one FMA, so exactly the two candidate roundings are accepted;
  * tanh * 24 and the sigmoid go through tanhf / expf (2 ulp each) and an IEEE division: the float64 value with a
    relative bound of 2^-21 (at least four fp32 ulps).  A bf16 output may take the neighbouring bf16 value only where
    that bound straddles a rounding midpoint; fp32 outputs must lie within the bound.
tests/conv_paths.py restates the dispatch on the host; the CPU test keeps the case tables honest about the paths they
reach, and the GPU routing test checks that restatement against the kernels the profiler sees."""
import re
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.conv_paths import ACT_NAMES, features, lin_features, route, wgrad_features

NONE, RELU, LRELU, TANH24, SIGMOID = range(5)
SENT_BF16 = -1.0e30            # prefilled outputs: no case can produce it
SENT_F32 = -3.0e38
EXACT_SPAN = 2.0 ** 22         # sum|terms| <= 2^22 g
REL_BOUND = 2.0 ** -21         # tanhf, expf: 2 ulp; *24, 1 + e, the division: 1/2 ulp each

# One teco_conv3x3_tc launch.  res: '' / 'sep' / 'inplace'; f32c: channels of the fp32 output (0: none); shift: added to
# every bias (the fp32 sigmoid case shifts its inputs to where expf's argument is large); reaches: keys of
# conv_paths.features the case must reach.
Case = namedtuple("Case", "mode n h w cin cout act bias res y f32c res_f32 post shift reaches")


def C(mode, n, h, w, cin, cout, act, reaches, bias=True, res="", y=True, f32c=0, res_f32=False, post=(1.0, 0.0), shift=0.0):
    return Case(mode, n, h, w, cin, cout, act, bias, res, y, f32c, res_f32, post, shift, set(reaches))


CASES = {
    # conv3x3_ws_kernel<0>
    "ws0_relu_inplace_many_tiny": C(0, 560, 5, 6, 64, 64, RELU, {
        "ws<0> act=relu", "ws<0> res=inplace", "ws<0> smaller than a tile", "ws<0> tiles>grid", "ws<0> ragged"}, res="inplace"),
    "ws0_none_sep_ragged": C(0, 3, 19, 21, 64, 64, NONE, {"ws<0> act=none", "ws<0> res=sep", "ws<0> ragged"}, res="sep"),
    "ws0_lrelu_nobias_cout128": C(0, 2, 24, 40, 64, 128, LRELU, {
        "ws<0> act=lrelu", "ws<0> bias=None", "ws<0> cout=128", "ws<0> res=sep"}, bias=False, res="sep"),
    "ws0_tanh_cout512": C(0, 2, 19, 21, 64, 512, TANH24, {"ws<0> act=tanh24", "ws<0> cout=512", "ws<0> res=none"}),
    "ws0_sigmoid_full_tiles": C(0, 4, 32, 32, 64, 64, SIGMOID, {"ws<0> act=sigmoid", "ws<0> res=none"}),
    "ws0_none_tiles_gt_grid": C(0, 18, 64, 64, 64, 64, NONE, {"ws<0> act=none", "ws<0> res=none", "ws<0> tiles>grid"}),
    # conv3x3_ws_kernel<1>
    "ws1_relu_tiles_gt_grid": C(1, 540, 8, 8, 64, 64, RELU, {"ws<1> act=relu", "ws<1> tiles>grid", "ws<1> wg below image"}),
    "ws1_none_ragged_cout128": C(1, 3, 19, 21, 64, 128, NONE, {
        "ws<1> act=none", "ws<1> ragged", "ws<1> wg below image", "ws<1> cout=128"}),
    "ws1_lrelu_tiny": C(1, 2, 5, 6, 64, 64, LRELU, {"ws<1> act=lrelu", "ws<1> ragged"}),
    "ws1_tanh": C(1, 2, 16, 16, 64, 64, TANH24, {"ws<1> act=tanh24"}),
    "ws1_sigmoid": C(1, 2, 9, 12, 64, 64, SIGMOID, {"ws<1> act=sigmoid", "ws<1> ragged"}),
    # conv3x3_wgmma_kernel<64>
    "wgmma064_resident_res": C(0, 2, 19, 21, 128, 64, RELU, {"wgmma<64> resident+res"}, res="sep"),
    "wgmma064_streamed_res": C(0, 1, 16, 24, 192, 128, NONE, {"wgmma<64> streamed+res", "wgmma<64> nsplit>1"},
                               res="inplace"),
    "wgmma064_out_f32": C(0, 2, 17, 20, 64, 64, RELU, {"wgmma<64> out_f32 nblk=1"}, y=False, f32c=64, res_f32=True,
                          post=(0.5, 0.25)),
    # conv3x3_wgmma_kernel<32>
    "wgmma032_resident": C(0, 2, 16, 16, 256, 96, LRELU, {"wgmma<32> resident", "wgmma<32> nsplit>1"}),
    "wgmma032_streamed": C(0, 2, 13, 11, 320, 32, NONE, {"wgmma<32> streamed", "wgmma<32> res=sep"}, res="sep"),
    # conv3x3_wgmma_kernel<16>
    "wgmma016_output_stage": C(0, 2, 40, 24, 64, 16, NONE, {"wgmma<16> output stage"}, y=False, f32c=3, res_f32=True,
                               post=(2.0, -1.0)),
    "wgmma016_fnet_head": C(0, 2, 17, 25, 64, 16, TANH24, {"wgmma<16> fnet head"}, y=False, f32c=2),
    "wgmma016_y_and_f32": C(0, 2, 19, 13, 128, 48, RELU, {"wgmma<16> y+out_f32", "wgmma<16> out_f32_c spans splits"},
                            f32c=48, res_f32=True, post=(0.5, 0.25)),
    "wgmma016_f32c_two_splits": C(0, 2, 21, 19, 64, 48, NONE, {"wgmma<16> out_f32_c spans splits"}, y=False, f32c=20,
                                  res_f32=True),
    "wgmma016_sigmoid_f32": C(0, 2, 16, 24, 64, 16, SIGMOID, {"wgmma<16> act=sigmoid", "wgmma<16> out_f32"}, y=False,
                              f32c=16, shift=-10.0),
    "wgmma016_inplace_res": C(0, 2, 19, 21, 64, 16, RELU, {"wgmma<16> res=inplace"}, res="inplace"),
}

REQUIRED = (
    {"ws<0> act=%s" % a for a in ACT_NAMES} | {"ws<1> act=%s" % a for a in ACT_NAMES} |
    {"ws<0> res=none", "ws<0> res=sep", "ws<0> res=inplace", "ws<0> bias=None", "ws<0> cout=128", "ws<0> cout=512",
     "ws<0> ragged", "ws<0> smaller than a tile", "ws<0> tiles>grid",
     "ws<1> ragged", "ws<1> wg below image", "ws<1> tiles>grid", "ws<1> cout=128",
     "wgmma<64> resident+res", "wgmma<64> streamed+res", "wgmma<64> out_f32 nblk=1",
     "wgmma<32> resident", "wgmma<32> streamed",
     "wgmma<16> output stage", "wgmma<16> fnet head", "wgmma<16> y+out_f32", "wgmma<16> out_f32_c spans splits",
     "wgmma<16> res=inplace"})

# teco_conv3x3_lin_tc: 32x32 images and trunk-shaped plans (the only ones it takes), with (input buffer, output buffer,
# residual buffer or -1, activation) per layer.  LeakyReLU only on a last layer: 0.2 v leaves the grid the next layer needs.
LIN_CASES = {
    "linear": (3, 32, [(0, 1, -1, NONE)]),
    "lrelu_into_b": (4, 32, [(0, 1, -1, RELU), (1, 2, -1, LRELU)]),
    "inplace_res_lrelu_on_b": (5, 32, [(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, -1, RELU), (1, 2, 2, LRELU)]),
    "res_block": (2, 32, [(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, 1, NONE)]),
    "images_gt_sms": (150, 32, [(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, 1, NONE), (1, 2, -1, RELU), (2, 1, 1, NONE)]),
    "nine_layers_weight_ring": (7, 32, [(0, 1, -1, RELU)] + [(1, 2, -1, RELU), (2, 1, 1, NONE)] * 4),
    # even L: a cluster's later clips start on the same ring parity as its first (odd L above alternates it)
    "three_clips_even_layers": (140, 32, [(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, 1, NONE), (1, 2, -1, RELU)]),
}
LIN_REQUIRED = {"lin L=1", "lin L=9", "lin weight ring wraps", "lin clips>clusters", "lin res=inplace on buffer 1",
                "lin res=inplace on buffer 2", "lin last output in buffer 2", "lin act=none", "lin act=relu", "lin act=lrelu",
                "lin three clips per cluster, L odd", "lin three clips per cluster, L even"}

# teco_conv3x3_wgrad_tc: the shapes of test_gpu_kernels.py::test_conv3x3_wgrad_tc_matches_autograd_on_bf16_operands
WGRAD_CASES = [(1, 8, 16, 64, 64), (4, 32, 32, 64, 64), (2, 19, 21, 51, 64), (3, 16, 24, 128, 32), (2, 32, 32, 32, 256),
               (2, 9, 40, 256, 64), (2, 13, 21, 64, 4), (3, 5, 7, 32, 64)]
WGRAD_REQUIRED = {"wgrad ragged", "wgrad cout=4", "wgrad padded channels", "wgrad several tiles"}


def _case_features(c):
    return features(c.mode, c.n, c.h, c.w, c.cin, c.cout, c.act, c.bias, c.res, c.y, c.f32c, c.res_f32, c.post)


def test_case_tables_reach_every_required_path():
    """Host restatement of the dispatch (tests/conv_paths.py): each case reaches the paths it claims, and together the
    tables reach every kernel instance of teco_conv3x3_tc with each epilogue feature listed in REQUIRED, the chain's
    weight-ring wrap, in-place residuals on either buffer, more clips than clusters and clusters running three clips at
    an odd and an even layer count (on plans its entry takes), and the
    weight gradient's ragged and narrow shapes.  Mode 1 runs on conv3x3_ws_kernel<1> only, and route() refuses it for
    exactly four conditions, each of which mode 0 takes."""
    from tecogan_b200 import kernels as K
    seen = set()
    for name, c in CASES.items():
        got = _case_features(c)
        assert c.reaches <= got, (name, sorted(c.reaches - got))
        if c.act in (TANH24, SIGMOID):      # the bound-based comparison does not model a residual or the post transform
            assert not c.res and not c.res_f32 and c.post == (1.0, 0.0), name
        if c.act == LRELU:                  # the two-candidate comparison is bf16-only
            assert not c.f32c, name
        seen |= got
    assert REQUIRED <= seen, sorted(REQUIRED - seen)
    kernels = {route(c.mode, c.cin, c.cout, bool(c.res), c.res == "inplace", c.f32c > 0, c.y).kernel for c in CASES.values()}
    assert kernels == {"ws<0>", "ws<1>", "wgmma<64>", "wgmma<32>", "wgmma<16>"}
    assert route(0, 128, 64).resident and not route(0, 192, 64).resident
    assert route(0, 256, 32).resident and not route(0, 320, 32).resident
    assert route(0, 512, 16).resident
    assert route(1, 64, 64).kernel == route(1, 64, 128).kernel == "ws<1>"
    for cin, cout, res, out_f32 in ((128, 64, False, False), (64, 32, False, False), (64, 48, False, False),
                                    (64, 64, True, False), (64, 64, False, True)):
        assert route(1, cin, cout, res=res, out_f32=out_f32).kernel == "refused", (cin, cout, res, out_f32)
        assert route(0, cin, cout, res=res, out_f32=out_f32).kernel != "refused", (cin, cout, res, out_f32)
    lin = set().union(*(lin_features(*v) for v in LIN_CASES.values()))
    assert LIN_REQUIRED <= lin, sorted(LIN_REQUIRED - lin)
    for n, h, plan in LIN_CASES.values():
        assert all(act != LRELU for _, _, _, act in plan[:-1])
        assert K.conv3x3_lin_in_smem(n, h, 32, plan), plan
    wg = set().union(*(wgrad_features(*s) for s in WGRAD_CASES))
    assert WGRAD_REQUIRED <= wg, sorted(WGRAD_REQUIRED - wg)


# ------------------------------------------------------------------------------------------------------ grids and guard
def _grid(rng, shape, unit, kmax):
    """Integers in [-kmax, kmax] times unit, float64 (+0.0 turns -0 into +0, as the kernels' bias add does)."""
    return torch.from_numpy(rng.randint(-kmax, kmax + 1, size=shape) * unit + 0.0)


def _bf16_grid(rng, shape):
    """bf16 values on the 2^-11 grid with magnitude <= 2: rounding a 2^-11-grid value to bf16 keeps it on that grid."""
    v = _grid(rng, shape, 2.0 ** -11, 4096).to(torch.bfloat16).double() + 0.0
    assert bool((v * 2048 == torch.round(v * 2048)).all())
    return v


def _lsb(a):
    """Largest power of two that divides every non-zero element of a (float64); inf for an all-zero tensor."""
    a = a.abs().flatten().numpy()
    a = a[a != 0]
    if a.size == 0:
        return float("inf")
    m, e = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    return float(((mi & -mi).astype(np.float64) * np.exp2(e - 53.0)).min())


def _assert_exact_regime(what, x, w, s_terms, *addends):
    """The exactness condition: every product x w is a multiple of g = lsb(x) lsb(w), so is every addend (bias, residual),
    and sum|terms| <= 2^22 g for every output."""
    g = _lsb(x) * _lsb(w)
    for a in addends:
        assert _lsb(a) >= g, "%s: an addend is off the %g grid" % (what, g)
    assert s_terms.max().item() <= EXACT_SPAN * g, "%s: sum|terms| %.4g > 2^22 g = %.4g" % (
        what, s_terms.max().item(), EXACT_SPAN * g)


def _is_f32(v):
    return bool(torch.equal(v.float().double(), v))


# ------------------------------------------------------------------------------------------------ epilogue reference
def _lrelu_f32(z):
    """v >= 0 ? v : 0.2f * v in fp32 (z exact in fp32)."""
    z32 = z.float()
    return torch.where(z32 >= 0, z32, torch.tensor(0.2, dtype=torch.float32) * z32).double()


def _exact_candidates(act, z, r):
    """Pre-rounding fp32 values (float64 tensors) the epilogue may produce from the exact z = conv + bias: one for none /
    ReLU, and for LeakyReLU followed by a residual the separately rounded multiply and add and the FMA."""
    if act == NONE:
        a = [z]
    elif act == RELU:
        a = [z.clamp_min(0.0)]
    else:
        a = [_lrelu_f32(z)]
    if r is None:
        return a
    out = [(a[0].float() + r.float()).double()]
    if act == LRELU:    # fma(0.2f, v, r): 0.2f v + r is exact in float64 (at most 47 significant bits), rounded once
        fma = (torch.tensor(np.float32(0.2), dtype=torch.float64) * z + r).float().double()
        out.append(torch.where(z >= 0, out[0], fma))
    return out


def _approx_ref(act, z):
    return torch.tanh(z) * 24.0 if act == TANH24 else 1.0 / (1.0 + torch.exp(-z))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _bf16_step(e, up):
    """The bf16 neighbour of e (bf16, non-zero) towards +inf (up) or -inf, as float64."""
    b = e.view(torch.int16).int()
    away = (e > 0) == up                 # towards larger magnitude
    nb = torch.where(away, b + 1, b - 1).to(torch.int16)
    return nb.view(torch.bfloat16).double()


def _check_bf16(got, cands, what, approx=None):
    """got (bf16) against the bf16 roundings of the candidates (exact), or, with approx = (ref64, bound), against the bf16
    rounding of ref64 and its neighbour where ref64 +- bound straddles the midpoint between them."""
    gb = _bits(got)
    if approx is None:
        ok = torch.zeros_like(gb, dtype=torch.bool)
        for c in cands:
            ok |= gb == _bits(c.float().to(torch.bfloat16))
        exp = cands[0].float().to(torch.bfloat16)
    else:
        ref, bound = approx
        exp = ref.float().to(torch.bfloat16)
        e64 = exp.double()
        ok = gb == _bits(exp)
        for up in (True, False):
            nb = _bf16_step(exp, up)
            mid = (e64 + nb) / 2
            allowed = ((ref - mid).abs() <= bound) & (e64 != 0)
            ok |= allowed & (gb == _bits(nb.to(torch.bfloat16)))
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(int(v) for v in bad[0])
        raise AssertionError("%s: %d / %d elements differ, first at %s: got %r, expected %r" % (
            what, bad.shape[0], ok.numel(), i, float(got[i]), float(exp[i])))


def _check_f32(got, exp, what, bound=None):
    if bound is None:
        bad = _bits(got) != _bits(exp.float())
    else:
        bad = ~((got.double() - exp).abs() <= bound)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: %d / %d elements differ, first at %s: got %r, expected %r" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(exp[i])))


def _midpoints(v):
    """Elements of v (float64, exact in fp32) that lie exactly halfway between two bf16 values."""
    return int(((_bits(v.float()) & 0xFFFF) == 0x8000).sum()) if v.numel() else 0


# ------------------------------------------------------------------------------------------------------ teco_conv3x3_tc
def _operands(name):
    c = CASES[name]
    rng = np.random.RandomState(1 + sorted(CASES).index(name))
    s = 2 if c.mode == 1 else 1
    x = _grid(rng, (c.n, c.h, c.w, c.cin), 2.0 ** -4, 16)
    wshape = (3, 3, c.cin, c.cout) if c.mode == 0 else (3, 3, c.cout, c.cin)
    wt = _grid(rng, wshape, 2.0 ** -7, 16)
    b = _grid(rng, (c.cout,), 2.0 ** -11, 2048) + c.shift if c.bias else torch.zeros(c.cout, dtype=torch.float64)
    oshape = (c.n, s * c.h, s * c.w)
    r = _bf16_grid(rng, oshape + (c.cout,)) if c.res else None
    rf = _grid(rng, oshape + (c.f32c,), 2.0 ** -11, 4096) if c.res_f32 else None
    return c, x, wt, b, r, rf


def _launch(c, x, wt, b, r, rf, device="cuda"):
    """One teco_conv3x3_tc launch into sentinel-filled outputs with one guard image after the last; returns (y, f32) on
    the host, guard image included."""
    from tecogan_b200 import kernels as K
    s = 2 if c.mode == 1 else 1
    oshape = (c.n + 1, s * c.h, s * c.w)
    wpk = K.packed_weight(wt.float().to(device), c.cin, c.cout, transpose_layout=c.mode == 1)
    y = torch.full(oshape + (c.cout,), SENT_BF16, dtype=torch.bfloat16, device=device) if c.y else None
    res = None
    if c.res == "inplace":
        y[:c.n] = r.to(torch.bfloat16).to(device)
        res = y[:c.n]
    elif c.res:
        res = r.to(torch.bfloat16).to(device)
    f32 = torch.full(oshape + (c.f32c,), SENT_F32, device=device) if c.f32c else None
    K.conv3x3_tc(x.to(torch.bfloat16).to(device), wpk, b.float().to(device) if c.bias else None,
                 y[:c.n] if c.y else None, cout=c.cout, act=c.act, res=res, mode=c.mode,
                 out_f32=f32[:c.n] if c.f32c else None, res_f32=rf.float().to(device) if c.res_f32 else None, post=c.post)
    torch.cuda.synchronize()
    return (y.cpu() if c.y else None), (f32.cpu() if c.f32c else None)


def _check_guard_image(t, sentinel, what):
    assert bool((_bits(t[-1]) == _bits(torch.tensor(sentinel, dtype=t.dtype))).all()), what + ": wrote past the last image"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conv3x3_tc_matches_float64_reference_bit_for_bit(name):
    """One launch per case on grid operands: the bf16 output equals the bf16 rounding of the float64 epilogue bit for bit
    (or one of the two LeakyReLU + residual candidates, or a tie-neighbour within the tanh / sigmoid bound), the fp32
    output equals the float64 value exactly (within the bound for tanh / sigmoid), no pixel keeps the sentinel, and the
    guard image after the last one is untouched."""
    c, x, wt, b, r, rf = _operands(name)
    op = O.conv2d if c.mode == 0 else O.conv2d_transpose
    z = op(x, wt) + b
    s_conv = op(x.abs(), wt.abs()) + b.abs()
    _assert_exact_regime(name + " y", x, wt, s_conv + (r.abs() if r is not None else 0.0), b, *([r] if r is not None else []))
    if c.f32c:
        _assert_exact_regime(name + " out_f32", x, wt, s_conv[..., :c.f32c] + (rf.abs() if rf is not None else 0.0), b,
                             *([rf] if rf is not None else []))
    assert _is_f32(z)

    y, f32 = _launch(c, x, wt, b, r, rf)
    approx = c.act in (TANH24, SIGMOID)
    if c.y:
        _check_guard_image(y, SENT_BF16, name + " y")
        got = y[:-1]
        if approx:
            ref = _approx_ref(c.act, z)
            _check_bf16(got, None, name + " y", approx=(ref, REL_BOUND * ref.abs()))
        else:
            cands = _exact_candidates(c.act, z, r)
            for v in cands:
                assert _is_f32(v), name + ": pre-rounding value not exact in fp32"
            _check_bf16(got, cands, name + " y")
            if c.act in (NONE, RELU):
                assert _midpoints(cands[0]) > 0, name + ": no output on a bf16 rounding midpoint"
    if c.f32c:
        _check_guard_image(f32, SENT_F32, name + " out_f32")
        got = f32[:-1]
        zc = z[..., :c.f32c]
        if approx:
            ref = _approx_ref(c.act, zc)
            _check_f32(got, ref, name + " out_f32", bound=REL_BOUND * ref.abs())
        else:
            v = zc.clamp_min(0.0) if c.act == RELU else zc
            v = (v + (rf if rf is not None else 0.0)) * c.post[0] + c.post[1]
            assert _is_f32(v), name + ": fp32 output not exact in fp32"
            _check_f32(got, v, name + " out_f32")


_KERNEL_RE = re.compile(r"conv3x3_(ws|wgmma)_kernel<([^>]*)>")

# Runs fn of module once, then again in one profiler session, and prints the names of the CUDA kernels of that session
# in launch order as JSON.  Repeated profiler sessions in one process can leave later sessions with no events, so the
# suite's own process never profiles here: _profiled_conv_kernels runs this in a child process.
_PROFILE = """
import json, sys, torch
sys.path.insert(0, %r)
from torch.profiler import ProfilerActivity, profile
from %s import %s as fn
fn()                                  # module load and the packing, outside the profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
ev = sorted((e.time_range.start, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
print(json.dumps([name for _, name in ev]))
"""


def _profiled_conv_kernels(module, fn):
    """The teco_conv3x3_tc kernel instances ('ws<1>', 'wgmma<64>', ...) that fn of module launches, in order, recorded
    by the profiler in a child process."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    flags = ["-I"] if sys.flags.isolated else (["-s"] if sys.flags.no_user_site else [])
    script = _PROFILE % (root, module, fn)
    out = subprocess.run([sys.executable] + flags + ["-c", script], cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    kernels = json.loads(out.stdout.strip().splitlines()[-1])
    if not kernels:
        pytest.skip("the profiler recorded no CUDA kernel")
    got = []
    for k in kernels:
        m = _KERNEL_RE.search(k)
        if m:
            got.append("%s<%s>" % (m.group(1), ",".join(re.findall(r"\d+", m.group(2)))))
    return got


def _zero_launch(c):
    s = 2 if c.mode == 1 else 1
    zeros = lambda *shape: torch.zeros(*shape, dtype=torch.float64)
    wt = zeros(3, 3, c.cin, c.cout) if c.mode == 0 else zeros(3, 3, c.cout, c.cin)
    _launch(c, zeros(c.n, c.h, c.w, c.cin), wt, zeros(c.cout), zeros(c.n, s * c.h, s * c.w, c.cout) if c.res else None,
            zeros(c.n, s * c.h, s * c.w, c.f32c) if c.res_f32 else None)


def _zero_launches():
    for c in CASES.values():
        _zero_launch(c)


@pytest.mark.gpu
def test_conv3x3_tc_runs_the_kernels_conv_paths_names():
    """The kernel instance of each case's launch, as the profiler records it, is the one tests/conv_paths.py::route
    restates, so the case table reaches the paths the CPU test says it does."""
    got = _profiled_conv_kernels("tests.test_gpu_conv_exact", "_zero_launches")
    want = [route(c.mode, c.cin, c.cout, bool(c.res), c.res == "inplace", c.f32c > 0, c.y).kernel for c in CASES.values()]
    assert len(got) == len(want), (got, want)
    bad = [(name, g, w) for name, g, w in zip(CASES, got, want) if g != w]
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0])
def test_ws_and_wgmma_kernels_agree_bit_for_bit_on_continuous_operands(mode):
    """DESIGN 4.1: conv3x3_ws_kernel<0> runs the products of conv3x3_wgmma_kernel in the same tap and K order with the
    same epilogue, so their bf16 outputs are bit-identical on any operands.  Asking for an fp32 output as well moves the
    same 64 -> 64 launch onto conv3x3_wgmma_kernel<64>, which writes the bf16 output in the same launch.  Mode 1 has
    one kernel; tools/ab_conv.py compares it between two builds."""
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(5 + mode)
    n, h, w = 3, 37, 45
    x = (torch.rand(n, h, w, 64, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    wt = (torch.rand(3, 3, 64, 64, generator=g) * 2 - 1) * (3.0 / 576) ** 0.5
    b = (torch.rand(64, generator=g) - 0.5).cuda()
    wpk = K.packed_weight(wt.cuda(), 64, 64, transpose_layout=mode == 1)
    s = 2 if mode == 1 else 1
    for act in range(5):
        ws = K.conv3x3_tc(x, wpk, b, cout=64, act=act, mode=mode)
        wg = torch.empty_like(ws)
        f32 = torch.empty(n, s * h, s * w, 64, device="cuda")
        K.conv3x3_tc(x, wpk, b, wg, cout=64, act=act, mode=mode, out_f32=f32)
        torch.cuda.synchronize()
        assert torch.equal(_bits(ws), _bits(wg)), (mode, ACT_NAMES[act], int((_bits(ws) != _bits(wg)).sum()))
        assert torch.equal(_bits(ws), _bits(f32.to(torch.bfloat16))), (mode, ACT_NAMES[act])


# --------------------------------------------------------------------------------------------------- teco_conv3x3_lin_tc
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LIN_CASES))
def test_conv3x3_lin_chain_matches_float64_reference_bit_for_bit(name):
    """The multi-layer chain layer by layer.  Layer 0 runs x = k/16 against weights m/128, so its products and outputs sit
    on the 2^-11 grid, and a bf16 rounding of a 2^-11-grid value stays on it.  Later layers use sparse weights in
    {-1, 0, 1} (three non-zero per output on average), so their products stay on that grid too and every layer is in the
    exact regime; the guard checks it per layer.  Both buffers end equal to the reference bit for bit and their guard
    images are untouched."""
    from tecogan_b200 import kernels as K
    n, h, plan = LIN_CASES[name]
    rng = np.random.RandomState(200 + sorted(LIN_CASES).index(name))
    L = len(plan)
    x = _grid(rng, (n, h, 32, 64), 2.0 ** -4, 16)
    ext = _bf16_grid(rng, (n, h, 32, 64))
    layers = [(_grid(rng, (3, 3, 64, 64), 2.0 ** -7, 16), _grid(rng, (64,), 2.0 ** -11, 2048))]
    for _ in range(1, L):
        sparse = rng.rand(3, 3, 64, 64) < 3.0 / 576
        layers.append((torch.from_numpy(sparse * rng.choice([-1.0, 1.0], size=sparse.shape) + 0.0),
                       _grid(rng, (64,), 2.0 ** -11, 2048)))

    bufs = {0: x, 1: torch.zeros_like(x), 2: ext}
    cands, ties = None, 0
    for l, ((wt, b), (i, o, ri, act)) in enumerate(zip(layers, plan)):
        z = O.conv2d(bufs[i], wt) + b
        r = bufs[ri] if ri >= 0 else None
        s_terms = O.conv2d(bufs[i].abs(), wt.abs()) + b.abs() + (r.abs() if r is not None else 0.0)
        _assert_exact_regime("%s layer %d" % (name, l), bufs[i], wt, s_terms, b, *([r] if r is not None else []))
        cands = _exact_candidates(act, z, r)
        assert all(_is_f32(v) for v in cands), (name, l)
        if act != LRELU:
            ties += _midpoints(cands[0])
        bufs[o] = cands[0].float().to(torch.bfloat16).double()
    assert ties > 0 or all(act == LRELU for *_, act in plan), name + ": no output on a bf16 rounding midpoint"

    def dev_buf(v):
        t = torch.full((n + 1, h, 32, 64), SENT_BF16, dtype=torch.bfloat16, device="cuda")
        t[:n] = v.to(torch.bfloat16).cuda()
        return t
    a, bb = dev_buf(torch.zeros_like(x)), dev_buf(ext)
    wall = torch.cat([K.packed_weight(wt.float().cuda(), 64, 64) for wt, _ in layers]).contiguous()
    ball = torch.cat([b.float().cuda() for _, b in layers]).contiguous()
    K.conv3x3_lin_chain(x.to(torch.bfloat16).cuda(), a[:n], bb[:n], wall, ball, plan)
    torch.cuda.synchronize()
    final = plan[-1][1]
    for idx, t in ((1, a.cpu()), (2, bb.cpu())):
        _check_guard_image(t, SENT_BF16, "%s buffer %d" % (name, idx))
        if idx == final:
            _check_bf16(t[:-1], cands, "%s buffer %d (last layer)" % (name, idx))
        else:
            _check_bf16(t[:-1], [bufs[idx]], "%s buffer %d" % (name, idx))


# ------------------------------------------------------------------------------------------------- teco_conv3x3_wgrad_tc
def _wgrad_ref(x, dz):
    """dw[ky, kx, ci, co] = sum over pixels p of x[p + (ky - 1, kx - 1), ci] dz[p, co], SAME zero padding, float64."""
    n, h, w, _ = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.stack([torch.stack([torch.einsum("nhwc,nhwd->cd", xp[:, ky:ky + h, kx:kx + w], dz) for kx in range(3)])
                        for ky in range(3)])


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,cin,cout", WGRAD_CASES)
def test_conv3x3_wgrad_tc_matches_float64_reference_bit_for_bit(n, h, w, cin, cout):
    """x = k/16 and dz = m/128: every per-tile partial dw and every fp32 atomicAdd of one into dw is exact, so dw equals
    the float64 sum bit for bit whatever order the tiles' atomics land in; also accumulated onto a 2^-11-grid dw.
    Nothing is written past dw."""
    from tecogan_b200 import kernels as K
    rng = np.random.RandomState(300 + n * 1000 + h * 10 + w + cin + cout)
    x = _grid(rng, (n, h, w, cin), 2.0 ** -4, 16)
    dz = _grid(rng, (n, h, w, cout), 2.0 ** -7, 16)
    dw0 = _grid(rng, (3, 3, cin, cout), 2.0 ** -11, 8192)
    ref, s_terms = _wgrad_ref(x, dz), _wgrad_ref(x.abs(), dz.abs())
    _assert_exact_regime("wgrad", x, dz, s_terms + dw0.abs(), dw0)

    def padded(t):
        c = t.shape[-1]
        out = torch.zeros(t.shape[:-1] + ((c + 63) // 64 * 64,), dtype=torch.bfloat16, device="cuda")
        out[..., :c] = t.to(torch.bfloat16).cuda()
        return out
    xb, dzb = padded(x), padded(dz)
    m = 9 * cin * cout
    for accumulate in (False, True):
        buf = torch.full((m + 64,), SENT_F32, device="cuda")
        if accumulate:
            buf[:m] = dw0.flatten().float().cuda()
        K.conv3x3_wgrad_tc(xb, dzb, buf[:m].view(3, 3, cin, cout), cin, cout, accumulate=accumulate)
        torch.cuda.synchronize()
        got = buf.cpu()
        assert bool((got[m:] == SENT_F32).all()), "wgrad wrote past dw"
        exp = ref + dw0 if accumulate else ref
        assert _is_f32(exp)
        _check_f32(got[:m].view(3, 3, cin, cout), exp + 0.0, "wgrad accumulate=%s" % accumulate)
