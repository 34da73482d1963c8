"""teco_conv3x3_f32out_tc (conv3x3_f32out_kernel): the fp32 output stage of teco_conv3x3_tc -- the generator's 64 -> 3
output conv and FNet's 64 -> 2 flow head -- on its pipelined kernel.

  * against a float64 reference bit for bit, on the exactly representable operands of test_gpu_conv_exact.py (its grids,
    host guard and epilogue restatement), and byte for byte against teco_conv3x3_tc on the same launch: C = 3 with an
    fp32 residual and post (2, -1), C = 2 with tanh * 24, ReLU / none / sigmoid, ragged images, images smaller than a
    tile, more tiles than the persistent grid; the guard image and the guard words around the output keep their sentinel;
  * byte for byte against teco_conv3x3_tc on continuous operands at the generator's output-stage shapes (264 clips at
    128 x 128, one frame at 512 x 512 and 1024 x 1024) and the flow head of 264 frame pairs at 32 x 32;
  * GeneratorPlan.run and FNetPlan.run against the same plans with the teco_conv3x3_tc launch put back;
  * rejection of every descriptor the entry does not take."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.test_gpu_conv_exact import (NONE, RELU, REL_BOUND, SENT_F32, SIGMOID, TANH24, _approx_ref,
                                       _assert_exact_regime, _bits, _check_f32, _grid, _is_f32)

GUARD = 4                      # fp32 words of sentinel before the output (16 bytes keep it aligned) and after the guard image

# name: (n, h, w, C, act, residual, post, bias shift)
CASES = {
    "c3_res_post_output_stage": (2, 40, 24, 3, NONE, True, (2.0, -1.0), 0.0),
    "c2_tanh_flow_head": (2, 17, 26, 2, TANH24, False, (1.0, 0.0), 0.0),
    "c3_relu_res_ragged": (3, 19, 20, 3, RELU, True, (0.5, 0.25), 0.0),
    "c2_none_ragged_nores": (2, 21, 14, 2, NONE, False, (1.0, 0.0), 0.0),
    "c2_sigmoid": (2, 16, 24, 2, SIGMOID, False, (1.0, 0.0), -10.0),
    "c3_none_smaller_than_a_tile": (5, 5, 4, 3, NONE, True, (2.0, -1.0), 0.0),
    "c2_relu_tiles_gt_grid": (40, 32, 32, 2, RELU, False, (1.0, 0.0), 0.0),      # 320 tiles
    "c3_none_tiles_gt_grid_res": (20, 48, 36, 3, NONE, True, (2.0, -1.0), 0.0),  # 20 x 3 x 5 = 300 tiles, ragged W
}


def _operands(name):
    n, h, w, C, act, res, post, shift = CASES[name]
    rng = np.random.RandomState(700 + sorted(CASES).index(name))
    x = _grid(rng, (n, h, w, 64), 2.0 ** -4, 16)
    wt = _grid(rng, (3, 3, 64, C), 2.0 ** -7, 16)
    b = _grid(rng, (C,), 2.0 ** -11, 2048) + shift
    rf = _grid(rng, (n, h, w, C), 2.0 ** -11, 4096) if res else None
    return x, wt, b, rf


def _launch(conv, n, h, w, C, act, post, x, wt, b, rf):
    """One launch of conv (kernels.conv3x3_f32out_tc or conv3x3_tc) into a sentinel-filled buffer: GUARD words, the
    output, one guard image, GUARD words.  Returns the whole buffer on the host."""
    from tecogan_b200 import kernels as K
    wpk = K.packed_weight(wt.float().cuda(), 64, 16)
    flat = torch.full((GUARD + (n + 1) * h * w * C + GUARD,), SENT_F32, device="cuda")
    out = flat[GUARD:GUARD + n * h * w * C].view(n, h, w, C)
    conv(x.to(torch.bfloat16).cuda(), wpk, K.pad_bias(b.float().cuda(), 16), None, cout=16, act=act, out_f32=out,
         res_f32=rf.float().cuda() if rf is not None else None, post=post)
    torch.cuda.synchronize()
    return flat.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conv3x3_f32out_tc_matches_float64_reference_bit_for_bit(name):
    """x = k/16, weights m/128, bias and residual on 2^-11: every partial sum is exact in fp32 (the host guard checks it
    per output), so the fp32 output equals the float64 epilogue exactly (within the bound for tanh / sigmoid); the words
    before the output, the guard image and the words after it keep their sentinel; and the bytes equal those of the
    same teco_conv3x3_tc launch."""
    from tecogan_b200 import kernels as K
    n, h, w, C, act, res, post, _ = CASES[name]
    x, wt, b, rf = _operands(name)
    z = O.conv2d(x, wt) + b
    _assert_exact_regime(name, x, wt, O.conv2d(x.abs(), wt.abs()) + b.abs() + (rf.abs() if rf is not None else 0.0), b,
                         *([rf] if rf is not None else []))
    assert _is_f32(z)
    assert K.conv3x3_f32out_fits(w, C)
    flat = _launch(K.conv3x3_f32out_tc, n, h, w, C, act, post, x, wt, b, rf)
    npix = n * h * w * C
    sent = _bits(torch.tensor(SENT_F32))
    assert bool((_bits(flat[:GUARD]) == sent).all()), name + ": wrote before the output"
    assert bool((_bits(flat[GUARD + npix:]) == sent).all()), name + ": wrote past the last image"
    got = flat[GUARD:GUARD + npix].view(n, h, w, C)
    if act in (TANH24, SIGMOID):
        ref = _approx_ref(act, z)
        _check_f32(got, ref, name, bound=REL_BOUND * ref.abs())
    else:
        v = z.clamp_min(0.0) if act == RELU else z
        v = (v + (rf if rf is not None else 0.0)) * post[0] + post[1]
        assert _is_f32(v), name + ": fp32 output not exact in fp32"
        _check_f32(got, v, name)
    want = _launch(K.conv3x3_tc, n, h, w, C, act, post, x, wt, b, rf)
    assert torch.equal(_bits(flat), _bits(want)), name + ": differs from teco_conv3x3_tc"


def test_f32out_case_table_covers_the_tile_walk():
    """The table reaches both output widths with and without a residual, every activation the networks use plus the
    sigmoid, images whose H or W is not a multiple of the 16 x 8 tile, an image smaller than a tile, and more tiles than
    the persistent grid of a 132-SM H100 (two CTAs per SM)."""
    vals = list(CASES.values())
    assert {(c[3], c[5]) for c in vals} >= {(3, True), (2, False)}
    assert {c[4] for c in vals} >= {NONE, RELU, TANH24, SIGMOID}
    assert any(h % 16 for _, h, *_ in vals) and any(w % 8 for _, _, w, *_ in vals)
    assert any(h < 16 and w < 8 for _, h, w, *_ in vals)
    assert sum(n * -(-h // 16) * -(-w // 8) > 2 * 132 for n, h, w, *_ in vals) >= 2


def test_f32out_fits_rule():
    """kernels.conv3x3_f32out_fits: 2 or 3 channels, and a whole number of 16-byte units per fp32 row."""
    from tecogan_b200 import kernels as K
    assert K.conv3x3_f32out_fits(128, 3) and K.conv3x3_f32out_fits(4096, 3) and K.conv3x3_f32out_fits(32, 2)
    assert K.conv3x3_f32out_fits(4, 3) and K.conv3x3_f32out_fits(2, 2)
    assert not K.conv3x3_f32out_fits(126, 3) and not K.conv3x3_f32out_fits(33, 2)
    assert not K.conv3x3_f32out_fits(128, 1) and not K.conv3x3_f32out_fits(128, 4) and not K.conv3x3_f32out_fits(128, 16)


# (n, h, w, C, act, residual + post): the generator's output stage and FNet's flow head at the shapes the benchmark runs
SHAPES = [(264, 128, 128, 3, NONE, True), (1, 512, 512, 3, NONE, True), (1, 1024, 1024, 3, NONE, True),
          (264, 32, 32, 2, TANH24, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,C,act,res", SHAPES)
def test_conv3x3_f32out_tc_equals_conv3x3_tc_at_network_shapes(n, h, w, C, act, res):
    """The same products in the same order and the same epilogue as teco_conv3x3_tc: byte-identical outputs on
    continuous operands."""
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(n * 7 + h + C)
    x = (torch.rand(n, h, w, 64, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    wt = (torch.rand(3, 3, 64, C, generator=g) * 2 - 1) * (3.0 / (9 * 64)) ** 0.5
    b = K.pad_bias((torch.rand(C, generator=g) - 0.5).cuda(), 16)
    rf = torch.rand(n, h, w, C, generator=g).cuda() if res else None
    post = (2.0, -1.0) if res else (1.0, 0.0)
    wpk = K.packed_weight(wt.cuda(), 64, 16)
    want = torch.empty(n, h, w, C, device="cuda")
    got = torch.empty(n, h, w, C, device="cuda")
    K.conv3x3_tc(x, wpk, b, cout=16, act=act, out_f32=want, res_f32=rf, post=post)
    K.conv3x3_f32out_tc(x, wpk, b, cout=16, act=act, out_f32=got, res_f32=rf, post=post)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
    assert bool(got.abs().max() > 0)


def _with_store(fn):
    from tecogan_b200 import config, variables as V
    from tecogan_b200.init_params import xavier_params
    prec, store = config.precision(), V.default_store()
    try:
        config.set_precision("bf16")
        V.set_default_store(V.VariableStore()).load(xavier_params(1234, 16))
        return fn()
    finally:
        config.set_precision(prec)
        V.set_default_store(store)


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,w", [(2, 32, 32), (264, 32, 32), (1, 128, 128)])
def test_generator_plan_output_is_byte_identical_to_the_conv3x3_tc_launch(B, h, w):
    """GeneratorPlan.run with its output stage on teco_conv3x3_f32out_tc returns the same bytes as the same plan with
    that launch on teco_conv3x3_tc."""
    from tecogan_b200 import kernels as K, tc_nets, variables as V

    def run():
        with V.variable_scope("generator"), V.variable_scope("generator_unit") as gs:
            tc_nets._ensure_vars_generator(16)
            plan = tc_nets.GeneratorPlan(gs, B, h, w, 16, "cuda")
        assert plan.out_conv is K.conv3x3_f32out_tc
        g = torch.Generator().manual_seed(B + h)
        plan.x_in[..., :51].copy_(torch.rand(B, h, w, 51, generator=g).to(torch.bfloat16))
        lr = torch.rand(B, h, w, 3, generator=g).cuda()
        got = plan.run(lr).clone()
        plan.out_conv = K.conv3x3_tc
        want = plan.run(lr).clone()
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
        assert bool(got.abs().max() > 0)
    _with_store(run)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 67, 264])
def test_fnet_plan_flow_is_byte_identical_to_the_conv3x3_tc_launch(n):
    """FNetPlan.run with its flow head on teco_conv3x3_f32out_tc returns the same flow bytes as the same plan with that
    launch on teco_conv3x3_tc."""
    from tecogan_b200 import kernels as K, tc_nets, variables as V

    def run():
        with V.variable_scope("fnet"), V.variable_scope("autoencode_unit") as fs:
            tc_nets._ensure_vars_fnet()
            plan = tc_nets.FNetPlan(fs, n, 32, 32, "cuda")
        assert plan.head_conv is K.conv3x3_f32out_tc
        g = torch.Generator().manual_seed(n)
        plan.x_in[..., :6].copy_(torch.rand(n, 32, 32, 6, generator=g).to(torch.bfloat16))
        got = plan.run().clone()
        plan.head_conv = K.conv3x3_tc
        want = plan.run().clone()
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
        assert bool(got.abs().max() > 0)
    _with_store(run)


@pytest.mark.gpu
def test_conv3x3_f32out_tc_rejects_what_it_does_not_take():
    """Every descriptor outside the entry's contract returns TECO_E_INVALID (ValueError) before anything runs; the
    buffers are real and large enough, so nothing is read or written out of bounds either way."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import TcDesc, call, ptr, stream_ptr
    bf16 = torch.bfloat16
    x = torch.zeros(2, 16, 16, 128, device="cuda", dtype=bf16)
    wpk = torch.zeros(9 * 128 * 64, device="cuda", dtype=bf16)
    bias = torch.zeros(64, device="cuda")
    big = torch.zeros(2 * 16 * 16 * 64 + 4, device="cuda")
    out = big[:2 * 16 * 16 * 3]
    ybf = torch.zeros(2, 16, 16, 16, device="cuda", dtype=bf16)

    def desc(**kw):
        d = dict(N=2, H=16, W=16, Cin=64, Cout=16, act=0, mode=0, out_f32_c=3, post_scale=1.0, post_shift=0.0)
        d.update(kw)
        return TcDesc(**d)

    def launch(d, x_=x, y=None, res=None, out_=out, res_f32=None):
        call("teco_conv3x3_f32out_tc", d, ptr(x_), ptr(wpk), ptr(bias), ptr(res), ptr(y), ptr(res_f32), ptr(out_),
             stream_ptr())

    launch(desc())                                    # the descriptor the others start from is taken
    torch.cuda.synchronize()
    bad = {
        "Cin 128": dict(d=desc(Cin=128)),
        "Cout 32": dict(d=desc(Cout=32)),
        "Cout 64": dict(d=desc(Cout=64)),
        "mode 1": dict(d=desc(mode=1)),
        "a bf16 output": dict(d=desc(), y=ybf),
        "a bf16 residual": dict(d=desc(), res=ybf),
        "C = 1": dict(d=desc(out_f32_c=1)),
        "C = 4": dict(d=desc(out_f32_c=4)),
        "C = 16": dict(d=desc(out_f32_c=16)),
        "W * C * 4 not a multiple of 16": dict(d=desc(W=15, out_f32_c=3)),
        "odd W at C = 2": dict(d=desc(W=15, out_f32_c=2)),
        "unknown activation": dict(d=desc(act=5)),
        "no output": dict(d=desc(), out_=None),
        "misaligned output": dict(d=desc(), out_=big[1:1 + 2 * 16 * 16 * 3]),
        "misaligned residual": dict(d=desc(), res_f32=big[1:1 + 2 * 16 * 16 * 3]),
        "empty batch": dict(d=desc(N=0)),
    }
    for what, kw in bad.items():
        with pytest.raises(ValueError, match="teco_conv3x3_f32out_tc"):
            launch(**kw)
    for C, W in ((3, 15), (2, 15), (1, 16), (4, 16), (16, 16)):   # the shape rule the plans select by, on the same cases
        assert not K.conv3x3_f32out_fits(W, C), (W, C)
