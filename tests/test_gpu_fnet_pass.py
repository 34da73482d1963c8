"""FNet's single pass per clip batch and the two launch-level changes behind it:

  * teco_conv3x3_tc with pool = 1 (the 2x2 max-pool in conv3x3_ws_kernel<0>'s epilogue) equals the same launch followed by
    teco_maxpool2_bf16, byte for byte, at FNet's levels and batch sizes and at odd sizes, and writes nothing past the
    last pooled image;
  * k_live (only the K-steps that carry input channels) equals the full-K launch byte for byte on inputs whose channels
    from 16 k_live on are zero, on conv3x3_ws_kernel<0> and conv3x3_f32out_kernel at FNet's shapes;
  * ClipEngine's one FNet pass over all B (T - 1) pairs gives the flows of one-pair passes that run every layer unfused
    and over the full K."""
import pytest
import torch

from tests.test_gpu_conv_exact import SENT_BF16, _bits, _check_guard_image

bf16 = torch.bfloat16


def _operands(seed, n, h, w, live=64, zero_images=0):
    """Continuous bf16 activations in [-1, 1) with channels >= live zero (the first zero_images images all zero), FNet-like
    3x3 64 -> 64 weights and a bias with some exact zeros."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, h, w, 64, generator=g) * 2 - 1
    x[..., live:] = 0
    x[:zero_images] = 0
    wt = (torch.rand(3, 3, 64, 64, generator=g) * 2 - 1) * (3.0 / (9 * max(live, 16))) ** 0.5
    b = torch.rand(64, generator=g) - 0.5
    b[::4] = 0
    return x.to(bf16).cuda(), wt.cuda(), b.cuda()


# (n, h, w, k_live): FNet's encoder_1 / encoder_2 conv_2 levels at 32 x 32 LR for one pair, 67 and 264 x 9 pairs; its
# 8 x 8 level on the same kernel; the odd levels of a 144 x 180 LR frame (36 x 45, 18 x 22) and a ragged odd one
POOL_CASES = [(1, 32, 32, 2), (67, 32, 32, 2), (2376, 32, 32, 2), (1, 16, 16, 0), (67, 16, 16, 0), (2376, 16, 16, 0),
              (1, 8, 8, 0), (67, 8, 8, 0), (3, 36, 45, 2), (5, 18, 22, 0), (2, 37, 23, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,k_live", POOL_CASES)
def test_pooled_epilogue_equals_conv_then_maxpool(n, h, w, k_live):
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import ACT_LRELU02
    live = 16 * k_live if k_live else 64
    x, wt, b = _operands(n * 7 + h + w, n, h, w, live)
    wpk = K.packed_weight(wt, 64, 64)
    full = K.conv3x3_tc(x, wpk, b, cout=64, act=ACT_LRELU02)
    want = K.maxpool2_bf16(full)
    got = torch.full((n + 1, h // 2, w // 2, 64), SENT_BF16, dtype=bf16, device="cuda")
    K.conv3x3_tc(x, wpk, b, got[:n], cout=64, act=ACT_LRELU02, k_live=k_live, pool=True)
    torch.cuda.synchronize()
    _check_guard_image(got.cpu(), SENT_BF16, "pooled conv3x3_tc")
    assert torch.equal(_bits(got[:n]), _bits(want)), int((_bits(got[:n]) != _bits(want)).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 3])
def test_pooled_epilogue_takes_every_activation(act):
    """none, ReLU and tanh * 24 as well as FNet's LeakyReLU: the pool follows the same bias -> activation -> bf16 steps."""
    from tecogan_b200 import kernels as K
    x, wt, b = _operands(90 + act, 6, 24, 40)
    wpk = K.packed_weight(wt, 64, 64)
    want = K.maxpool2_bf16(K.conv3x3_tc(x, wpk, b, cout=64, act=act))
    got = K.conv3x3_tc(x, wpk, b, cout=64, act=act, pool=True)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want))


@pytest.mark.gpu
def test_pool_and_k_live_are_refused_where_no_kernel_honours_them():
    from tecogan_b200 import kernels as K
    x, wt, b = _operands(1, 2, 16, 16)
    x128 = torch.zeros(2, 16, 16, 128, dtype=bf16, device="cuda")
    wpk, wpk128 = K.packed_weight(wt, 64, 64), K.packed_weight(torch.zeros(3, 3, 128, 64, device="cuda"), 128, 64)
    with pytest.raises(ValueError):
        K.conv3x3_tc(x128, wpk128, b, cout=64, pool=True)                 # two K blocks: conv3x3_wgmma_kernel
    with pytest.raises(ValueError):
        K.conv3x3_tc(x, wpk, b, cout=64, pool=True, res=x)
    with pytest.raises(ValueError):
        K.conv3x3_tc(x128, wpk128, b, cout=64, k_live=2)
    with pytest.raises(ValueError):
        K.conv3x3_tc(x, wpk, b, cout=64, k_live=3)


# (n, h, k_live): encoder_1/conv_1 (6 live channels), encoder_1/conv_2 and encoder_2/conv_1 (32 live) at 264 pairs
LIVE_CASES = [(264, 32, 1), (264, 32, 2), (264, 16, 2), (2, 45, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,k_live", LIVE_CASES)
def test_live_k_equals_full_k_on_the_ws_kernel(n, h, k_live):
    """Dead channels are exact zeros: skipping their K-steps leaves every output bit as it is, also on an all-zero image
    with zero biases (signed zeros)."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import ACT_LRELU02
    live = 6 if k_live == 1 else 32
    x, wt, b = _operands(n + h + k_live, n, h, h, live, zero_images=1)
    wpk = K.packed_weight(wt[:, :, :live], 64, 64)
    for act in (ACT_LRELU02, 0):
        want = K.conv3x3_tc(x, wpk, b, cout=64, act=act)
        got = K.conv3x3_tc(x, wpk, b, cout=64, act=act, k_live=k_live)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), (act, int((_bits(got) != _bits(want)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("n,h", [(264, 32), (2376, 32), (3, 36)])
def test_live_k_equals_full_k_on_the_flow_head(n, h):
    """FNet's flow head (32 live channels of o1, 64 -> 2 packed as 16, tanh * 24) on conv3x3_f32out_kernel with two
    K-steps per tap equals the full-K launch of that kernel and of teco_conv3x3_tc."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import ACT_TANH24
    g = torch.Generator().manual_seed(n + h)
    x = torch.rand(n, h, h, 64, generator=g) * 2 - 1
    x[..., 32:] = 0
    x[0] = 0
    x = x.to(bf16).cuda()
    wt = ((torch.rand(3, 3, 32, 2, generator=g) * 2 - 1) * (3.0 / 288) ** 0.5).cuda()
    b = K.pad_bias(torch.tensor([0.0, 0.1]).cuda(), 16)
    wpk = K.packed_weight(wt, 64, 16)
    outs = []
    for conv, k_live in ((K.conv3x3_f32out_tc, 2), (K.conv3x3_f32out_tc, 0), (K.conv3x3_tc, 0), (K.conv3x3_tc, 2)):
        o = torch.empty(n, h, h, 2, device="cuda")
        conv(x, wpk, b, None, cout=16, act=ACT_TANH24, out_f32=o, k_live=k_live)
        outs.append(o)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(_bits(outs[0]), _bits(o)), int((_bits(outs[0]) != _bits(o)).sum())


def _fnet_unfused(plan, x_in):
    """One FNet pass of `plan` on x_in with every layer on teco_conv3x3_tc over the full K, the max-pools as launches."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import ACT_LRELU02, ACT_TANH24
    x = x_in
    for i, ((c1, c2), (t1, t2, t3)) in enumerate(zip(plan.layers, plan.bufs)):
        t1 = K.conv3x3_tc(x, c1.wpk, c1.bias, cout=c1.cout_pad, act=ACT_LRELU02)
        t2 = K.conv3x3_tc(t1, c2.wpk, c2.bias, cout=c2.cout_pad, act=ACT_LRELU02)
        x = K.maxpool2_bf16(t2) if i < 3 else K.resize2x_bf16(t2)
    o1 = K.conv3x3_tc(x, plan.l_o1.wpk, plan.l_o1.bias, cout=64, act=ACT_LRELU02)
    flow = torch.empty((x_in.shape[0], plan.fh, plan.fw, 2), device="cuda")
    K.conv3x3_tc(o1, plan.l_o2.wpk, plan.l_o2.bias, None, cout=16, act=ACT_TANH24, out_f32=flow)
    return flow


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 264])
def test_clip_engine_flows_equal_one_pair_passes(B):
    from tecogan_b200 import config, variables as V
    from tecogan_b200.engine import ClipEngine
    from tecogan_b200.init_params import xavier_params
    from tecogan_b200.tc_nets import _f32_slice_to_bf16
    prec, store = config.precision(), V.default_store()
    T = 10
    try:
        config.set_precision("bf16")
        V.set_default_store(V.VariableStore()).load(xavier_params(1234, 16))
        eng = ClipEngine(32, 32, T, 16, batch=B)
        assert eng.fnet.n == B * (T - 1)
        assert eng.fnet.fused_pool == [True, True, False, False, False, False]
        g = torch.Generator().manual_seed(B)
        clips = torch.rand(T, B, 32, 32, 3, generator=g).cuda()
        eng.run(clips)
        torch.cuda.synchronize()
        x_in = torch.zeros(B, 32, 32, 64, dtype=bf16, device="cuda")
        for t in range(1, T):
            _f32_slice_to_bf16(clips[t - 1], 0, 3, x_in, 0)
            _f32_slice_to_bf16(clips[t], 0, 3, x_in, 3)
            want = _fnet_unfused(eng.fnet, x_in)
            torch.cuda.synchronize()
            assert torch.equal(_bits(eng.flows[t - 1]), _bits(want)), (t, int((_bits(eng.flows[t - 1]) != _bits(want)).sum()))
        assert bool(eng.flows.abs().max() > 0)
    finally:
        config.set_precision(prec)
        V.set_default_store(store)
