"""teco_conv3x3_im2col_tc (conv3x3_im2col_kernel): the 3x3 SAME convolution on 128-pixel tiles in flat N*H*W order, which
FNet runs on its levels smaller than a 16 x 8 tile.

  * against a float64 reference bit for bit, on the exactly representable operands of test_gpu_conv_exact.py (its grids,
    host guard and epilogue restatement), over small, ragged and tile-sized images, Cin / Cout 64 / 128 / 256, pixel
    counts that are not a multiple of 128, tiles that straddle images and more tiles than the persistent grid; nothing is
    written after the last pixel;
  * byte for byte against teco_conv3x3_tc on continuous operands, at FNet's shapes for 264 frame pairs;
  * a whole FNetPlan.run against the launch sequence that runs every layer on teco_conv3x3_tc."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.test_gpu_conv_exact import (LRELU, NONE, RELU, SENT_BF16, _assert_exact_regime, _bits, _check_bf16,
                                       _check_guard_image, _exact_candidates, _grid, _is_f32, _midpoints)

# name: (n, h, w, cin, cout, act, bias)
CASES = {
    "4x4_c256_c256_lrelu_67_images": (67, 4, 4, 256, 256, LRELU, True),      # 1072 pixels: 8 full tiles + 48
    "8x8_c128_c128_relu_ragged_count": (5, 8, 8, 128, 128, RELU, True),      # 320 pixels
    "16x16_c64_c64_none": (3, 16, 16, 64, 64, NONE, True),
    "5x7_c128_c256_none_straddling": (11, 5, 7, 128, 256, NONE, True),      # 35-pixel images, 385 pixels
    "3x9_c256_c64_relu_nobias": (9, 3, 9, 256, 64, RELU, False),            # 243 pixels
    "4x4_c64_c128_relu_one_image": (1, 4, 4, 64, 128, RELU, True),          # one image, one eighth of a tile
    "8x8_c64_c128_lrelu_tiles_gt_grid": (700, 8, 8, 64, 128, LRELU, True),  # 350 tiles x 2 Cout slices
}


def _launch(n, h, w, cin, cout, act, x, wt, b):
    """One teco_conv3x3_im2col_tc launch into a sentinel-filled output with one guard image after the last; returns the
    output on the host, guard image included."""
    from tecogan_b200 import kernels as K
    wpk = K.packed_weight(wt.float().cuda(), cin, cout)
    y = torch.full((n + 1, h, w, cout), SENT_BF16, dtype=torch.bfloat16, device="cuda")
    K.conv3x3_im2col_tc(x.to(torch.bfloat16).cuda(), wpk, b.float().cuda() if b is not None else None, y[:n], cout=cout,
                        act=act)
    torch.cuda.synchronize()
    return y.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conv3x3_im2col_tc_matches_float64_reference_bit_for_bit(name):
    """x = k/16, weights m/128, bias on 2^-11: every partial sum is exact in fp32 (the host guard checks it per output), so
    the bf16 output equals the bf16 rounding of the float64 epilogue bit for bit; none / ReLU cases hit rounding
    midpoints.  The guard image after the last one keeps its sentinel."""
    n, h, w, cin, cout, act, has_bias = CASES[name]
    rng = np.random.RandomState(400 + sorted(CASES).index(name))
    x = _grid(rng, (n, h, w, cin), 2.0 ** -4, 16)
    wt = _grid(rng, (3, 3, cin, cout), 2.0 ** -7, 16)
    b = _grid(rng, (cout,), 2.0 ** -11, 2048) if has_bias else torch.zeros(cout, dtype=torch.float64)
    z = O.conv2d(x, wt) + b
    _assert_exact_regime(name, x, wt, O.conv2d(x.abs(), wt.abs()) + b.abs(), b)
    assert _is_f32(z)
    y = _launch(n, h, w, cin, cout, act, x, wt, b if has_bias else None)
    _check_guard_image(y, SENT_BF16, name)
    cands = _exact_candidates(act, z, None)
    assert _is_f32(cands[0])
    _check_bf16(y[:-1], cands, name)
    if act in (NONE, RELU):
        assert _midpoints(cands[0]) > 0, name + ": no output on a bf16 rounding midpoint"


def test_im2col_case_table_covers_the_tile_walk():
    """The table reaches what the kernel's flat tile walk has to get right: pixel counts that are not a multiple of the
    128-pixel tile, tiles that start inside an image or straddle several, more tiles than one CTA per SM per Cout slice,
    and each Cin, Cout and activation FNet and the tests use."""
    pix = [n * h * w for n, h, w, *_ in CASES.values()]
    assert any(p % 128 for p in pix)
    assert any((h * w) % 128 and n * h * w > 128 for n, h, w, *_ in CASES.values())
    assert any(-(-n * h * w // 128) * (cout // 64) > 2 * 132 for n, h, w, _, cout, _, _ in CASES.values())
    assert {c[3] for c in CASES.values()} >= {64, 128, 256} and {c[4] for c in CASES.values()} >= {64, 128, 256}
    assert {c[5] for c in CASES.values()} == {NONE, RELU, LRELU}
    assert {(h, w) for _, h, w, *_ in CASES.values()} >= {(4, 4), (8, 8), (16, 16), (5, 7), (3, 9)}


# FNet's layers on 8 x 8 and 4 x 4 inputs at 32 x 32 LR, and decoder_3's first layer at 16 x 16: (h, cin, cout)
FNET_SHAPES = [(8, 64, 128), (8, 128, 128), (4, 128, 256), (4, 256, 256), (8, 256, 128), (16, 128, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("h,cin,cout", FNET_SHAPES)
def test_conv3x3_im2col_tc_equals_conv3x3_tc_on_fnet_shapes(h, cin, cout):
    """The same products in the same (K block, tap, K-step) order and the same epilogue as the layer's teco_conv3x3_tc
    kernel: byte-identical outputs on continuous operands, 264 frame pairs, LeakyReLU as in FNet."""
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(h * 1000 + cin + cout)
    x = (torch.rand(264, h, h, cin, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    wt = (torch.rand(3, 3, cin, cout, generator=g) * 2 - 1) * (3.0 / (9 * cin)) ** 0.5
    b = (torch.rand(cout, generator=g) - 0.5).cuda()
    wpk = K.packed_weight(wt.cuda(), cin, cout)
    want = K.conv3x3_tc(x, wpk, b, cout=cout, act=K.ACT_LRELU02)
    got = K.conv3x3_im2col_tc(x, wpk, b, cout=cout, act=K.ACT_LRELU02)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())


def _fnet_on_conv3x3_tc(plan):
    """FNetPlan.run with every convolution on teco_conv3x3_tc (the launch sequence before the small levels moved)."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import ACT_LRELU02, ACT_TANH24, call, ptr, stream_ptr
    x, n, bf16 = plan.x_in, plan.n, torch.bfloat16
    for i, ((c1, c2), (t1, t2, t3)) in enumerate(zip(plan.layers, plan.bufs)):
        K.conv3x3_tc(x, c1.wpk, c1.bias, t1, cout=c1.cout_pad, act=ACT_LRELU02)
        K.conv3x3_tc(t1, c2.wpk, c2.bias, t2, cout=c2.cout_pad, act=ACT_LRELU02)
        _, hh, ww, cc = t2.shape
        kern = "teco_maxpool2_bf16" if i < 3 else "teco_resize2x_bf16"
        call(kern, ptr(t2, bf16), ptr(t3, bf16), n, hh, ww, cc, stream_ptr())
        x = t3
    K.conv3x3_tc(x, plan.l_o1.wpk, plan.l_o1.bias, plan.o1, cout=64, act=ACT_LRELU02)
    flow = torch.empty_like(plan.flow)
    K.conv3x3_tc(plan.o1, plan.l_o2.wpk, plan.l_o2.bias, None, cout=16, act=ACT_TANH24, out_f32=flow)
    return flow


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 67, 264])
def test_fnet_plan_flow_is_byte_identical_to_the_conv3x3_tc_sequence(n):
    """FNetPlan.run on 32 x 32 pairs (its 8 x 8 and 4 x 4 levels on teco_conv3x3_im2col_tc) returns the same flow bytes
    as the same plan run with every layer on teco_conv3x3_tc."""
    from tecogan_b200 import config, tc_nets, variables as V
    from tecogan_b200.init_params import xavier_params
    prec, store = config.precision(), V.default_store()
    try:
        config.set_precision("bf16")
        V.set_default_store(V.VariableStore()).load(xavier_params(1234, 16))
        with V.variable_scope("fnet"), V.variable_scope("autoencode_unit") as fs:
            tc_nets._ensure_vars_fnet()
            plan = tc_nets.FNetPlan(fs, n, 32, 32, "cuda")
        g = torch.Generator().manual_seed(n)
        plan.x_in[..., :6].copy_((torch.rand(n, 32, 32, 6, generator=g)).to(torch.bfloat16))
        got = plan.run().clone()
        want = _fnet_on_conv3x3_tc(plan)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
        assert bool(got.abs().max() > 0)
    finally:
        config.set_precision(prec)
        V.set_default_store(store)
