"""The discriminator's 4x4 stride-2 convolutions on the tensor cores (kernels._Conv4x4S2TC: teco_f32_to_bf16_s2d2,
teco_pack_conv4x4s2_bf16, teco_conv4x4s2_tc, teco_conv4x4s2_dgrad_tc, teco_bf16_d2s2_to_f32 and the 3x3 weight gradient).

Forward, input gradient and weight gradient are compared with float64 bit for bit on exactly representable operands, under
the grid argument of test_gpu_conv_exact.py: x and dz = k/16, w = m/128 with |k|, |m| <= 16, so products lie on 2^-11
(forward, input gradient) or 2^-8 (weight gradient); while the sum of the magnitudes of an output's terms stays within
2^22 grid units every fp32 partial sum is exact, whatever the MMA order or atomic order.  _assert_exact_regime checks that
per output before comparing.  Then only the epilogue rounds: bf16 for y and dx (round to nearest even), none for dw."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import teco_oracle as O
from tests.test_disc_tc_host import _d2s, _direct, _s2d, _w_prime
from tests.test_gpu_train import Flags, _case, _fresh_store, _load, _t

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE, RELU, LRELU = 0, 1, 2


def _dyadic(shape, den, g):
    return torch.randint(-16, 17, shape, generator=g).double() / den


def _assert_exact_regime(span, unit):
    assert span.max().item() <= 2.0 ** 22 * unit, "operands leave the exact regime: %g > 2^22 * %g" % (span.max().item(), unit)


def _bf16(t):
    return t.float().bfloat16().float()


# (N, H, W, Cin, Cout): the four D layer shapes at the 128 x 128 crop (64^2, 32^2, 16^2, 8^2 outputs), N = 3 at the 8^2
# and 16^2 outputs leaving a partial last 128-pixel tile, and two ragged maps, one per 3x3 kernel the launch routes to.
SHAPES = [(2, 128, 128, 64, 64), (2, 64, 64, 64, 64), (3, 32, 32, 64, 128), (3, 16, 16, 128, 256),
          (2, 20, 12, 64, 128), (1, 36, 20, 128, 64), (5, 4, 4, 64, 64)]


@pytest.mark.parametrize("N,H,W,Cin,Cout", SHAPES)
def test_conv4x4s2_matches_float64_bit_for_bit(N, H, W, Cin, Cout):
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(N * H + W * Cin + Cout)
    x, w, dz = _dyadic((N, H, W, Cin), 16, g), _dyadic((4, 4, Cin, Cout), 128, g), _dyadic((N, H // 2, W // 2, Cout), 16, g)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y_ref = _direct(xr, wr)
    dx_ref, dw_ref = torch.autograd.grad(y_ref, (xr, wr), dz)
    _assert_exact_regime(_direct(x.abs(), w.abs()), 2.0 ** -11)
    _assert_exact_regime(_d2s(Fn.conv2d(dz.abs().permute(0, 3, 1, 2),
                                        torch.flip(_w_prime(w.abs()), (0, 1)).permute(2, 3, 0, 1), padding=1)
                              .permute(0, 2, 3, 1), Cin), 2.0 ** -11)
    _assert_exact_regime(torch.autograd.grad(_direct(xr.detach().abs(), wr), (wr,), dz.abs())[0], 2.0 ** -8)

    xg, wg = x.float().cuda().requires_grad_(True), w.float().cuda().requires_grad_(True)
    K.tc_cache_clear()
    y = K.conv4x4s2_train_tc(xg, wg)
    dx, dw = torch.autograd.grad(y, (xg, wg), dz.float().cuda())
    assert torch.equal(y.cpu(), _bf16(y_ref.detach()))
    assert torch.equal(dx.cpu(), _bf16(dx_ref))
    assert torch.equal(dw.cpu(), dw_ref.float())


@pytest.mark.parametrize("act", [RELU, LRELU])
def test_conv4x4s2_bias_and_activation_epilogue_bit_for_bit(act):
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(7 + act)
    x, w, b = _dyadic((3, 16, 16, 64), 16, g), _dyadic((4, 4, 64, 128), 128, g), _dyadic((128,), 2048, g)
    v = (_direct(x, w) + b).float()                   # exact in fp32 (the regime above)
    ref = torch.relu(v) if act == RELU else torch.where(v > 0, v, v * np.float32(0.2))
    K.tc_cache_clear()
    with torch.no_grad():
        y = K.conv4x4s2_train_tc(x.float().cuda(), w.float().cuda(), b.float().cuda(), act)
    assert torch.equal(y.cpu(), _bf16(ref))


@pytest.mark.parametrize("Cin,Cout", [(64, 64), (128, 256)])
def test_packed_weights_are_the_zero_scattered_3x3_weights(Cin, Cout):
    """teco_pack_conv4x4s2_bf16 writes what teco_pack_conv3x3_bf16 writes for W' (forward) and for W' with its flag 3
    (input gradient), byte for byte."""
    from tecogan_b200 import kernels as K
    w = torch.randn(4, 4, Cin, Cout, generator=torch.Generator().manual_seed(Cin + Cout))
    wp = _w_prime(w).cuda()
    wc = w.cuda()
    K.tc_cache_clear()
    assert torch.equal(K._c4s2_packed(wc, 0).view(torch.int16), K.packed_weight(wp, 4 * Cin, Cout, 0).view(torch.int16))
    assert torch.equal(K._c4s2_packed(wc, 1).view(torch.int16), K.packed_weight(wp, Cout, 4 * Cin, 3).view(torch.int16))


def test_space_to_depth_conversions_bit_for_bit():
    from tecogan_b200._ffi import call, ptr, stream_ptr
    x = torch.randn(3, 10, 6, 64, generator=torch.Generator().manual_seed(3)) * 100
    xs = torch.empty((3, 5, 3, 256), device="cuda", dtype=torch.bfloat16)
    call("teco_f32_to_bf16_s2d2", ptr(x.cuda()), ptr(xs), 3, 10, 6, 64, stream_ptr())
    assert torch.equal(xs.cpu(), _s2d(x).bfloat16())
    dx = torch.empty((3, 10, 6, 64), device="cuda")
    call("teco_bf16_d2s2_to_f32", ptr(xs), ptr(dx), 3, 10, 6, 64, stream_ptr())
    assert torch.equal(dx.cpu(), x.bfloat16().float())
    with pytest.raises(ValueError):
        call("teco_f32_to_bf16_s2d2", ptr(x.cuda()), ptr(xs), 3, 9, 6, 64, stream_ptr())


def test_entry_points_reject_shapes_they_do_not_take():
    from tecogan_b200._ffi import call, ptr, stream_ptr
    a = torch.zeros(1 << 20, device="cuda")
    for N, H, W, Cin, Cout in [(1, 15, 16, 64, 64), (1, 16, 15, 64, 64), (1, 16, 16, 32, 64), (1, 16, 16, 192, 64),
                               (1, 16, 16, 64, 96)]:
        with pytest.raises(ValueError):
            call("teco_conv4x4s2_tc", N, H, W, Cin, Cout, 0, ptr(a), ptr(a), ptr(None), ptr(a), stream_ptr())
        with pytest.raises(ValueError):
            call("teco_conv4x4s2_dgrad_tc", N, H, W, Cin, Cout, ptr(a), ptr(a), ptr(a), stream_ptr())


def test_graph_replay_repacks_updated_weights():
    """Packing runs inside a captured step (after tc_cache_clear), so a replay after an in-place weight update computes
    with the new weights: it matches an eager run on them bit for bit (dw is compared at fp32-atomic tolerance)."""
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(11)
    x = torch.randn(4, 32, 32, 64, generator=g).cuda().requires_grad_(True)
    w = (torch.randn(4, 4, 64, 128, generator=g) * 0.05).cuda().requires_grad_(True)
    dz = torch.randn(4, 16, 16, 128, generator=g).cuda()

    def step():
        K.tc_cache_clear()
        y = K.conv4x4s2_train_tc(x, w)
        return (y,) + torch.autograd.grad(y, (x, w), dz)

    step()                                          # eager first: module load, the slot index on the device
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    with torch.no_grad():
        w.mul_(-1.5).add_(0.01)
    graph.replay()
    want = step()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], want[0]) and torch.equal(outs[1], want[1])
    torch.testing.assert_close(outs[2], want[2], rtol=1e-5, atol=1e-5)


def test_bf16_discriminator_close_to_reference_golden():
    """discriminator_F of the bf16 training graph (all four disblocks on the tensor cores) against the reference's golden
    at the bf16 tolerances of the training-step tests."""
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import discriminator_F
    from tecogan_b200.variables import variable_scope
    g = _load("discriminator")
    _fresh_store(O.init_discriminator(seed=int(g["seed"]), bias_std=float(g["bias_std"])))
    config.set_train_precision("bf16")
    try:
        with variable_scope('tdiscriminator'):
            prob, layers = discriminator_F(_t(g["inputs"]).requires_grad_(True), FLAGS=Flags())
    finally:
        config.set_train_precision("fp32")
    np.testing.assert_allclose(prob.detach().cpu().numpy(), g["prob"], rtol=4e-2, atol=2e-3)
    for i, l in enumerate(layers):
        want = torch.from_numpy(g["layer%d" % i]).reshape(-1)
        got = l.detach().cpu().reshape(-1)
        assert float((got * want).sum() / (got.norm() * want.norm())) > 0.999, i


# Records, in a child process (repeated profiler sessions in one process can leave later ones empty), the CUDA kernels of
# one forward and backward of discriminator_F in the bf16 training graph, and prints their names as JSON.
_PROFILE_D = """
import json, torch
from torch.profiler import ProfilerActivity, profile
from oracle import teco_oracle as O
from tecogan_b200 import config
from tecogan_b200.lib.Teco import discriminator_F
from tecogan_b200.variables import variable_scope
from tecogan_b200 import kernels as K
from tests.test_gpu_train import Flags, _fresh_store
st = _fresh_store(O.init_discriminator(seed=5, bias_std=0.05))
for v in st.values():
    v.requires_grad_(True)
config.set_train_precision("bf16")
x = torch.rand(2, 32, 32, 27, device="cuda", requires_grad=True)
def run():
    K.tc_cache_clear()
    with variable_scope("tdiscriminator"):
        prob, _ = discriminator_F(x, FLAGS=Flags())
    prob.sum().backward()
run()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run()
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_bf16_discriminator_launches_no_fp32_4x4_convolution():
    """In the bf16 training graph the only fp32 convolution launches of discriminator_F are its dense layer's (a 1x1
    conv: forward, input gradient, weight gradient); the four disblocks run the space-to-depth tensor-core path."""
    flags = ["-I"] if sys.flags.isolated else (["-s"] if sys.flags.no_user_site else [])
    script = "import sys\nsys.path.insert(0, %r)\n" % ROOT + _PROFILE_D
    out = subprocess.run([sys.executable] + flags + ["-c", script], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().splitlines()[-1])
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel")
    count = lambda s: sum(s in n for n in names)
    assert count("conv2d_f32_kernel") == 2, [n for n in names if "conv2d" in n]
    assert count("conv2d_wgrad_f32_kernel") == 1
    assert count("f32_to_bf16_s2d2_kernel") == 4 and count("bf16_d2s2_to_f32_kernel") == 4
    assert count("pack_conv4x4s2_kernel") == 8


def test_bf16_tecogan_step_with_tensor_core_discriminator_close_to_fp32_oracle(monkeypatch):
    """One bf16 TecoGAN step with the disblocks on the tensor cores: losses at the bf16 step tolerances, and the
    discriminator's weight gradient in the direction of the fp32 oracle's.  The bound on its cosine is looser than the
    generator's 0.99 in the FRVSR step test: every discriminator gradient also carries the bf16 rounding of the generator
    output it is taken at, through four batch norms of small batches (0.981 measured on an H100)."""
    from tecogan_b200 import config, kernels as K
    from tecogan_b200.lib.Teco import TecoGAN
    calls = []
    tc = K.conv4x4s2_train_tc
    monkeypatch.setattr(K, "conv4x4s2_train_tc", lambda *a: calls.append(a[0].shape) or tc(*a))
    g, FL, P = _case("teco_pp")
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    tr = O.Trainer(P, FL, True)
    ref = tr.step(ri, rt)
    _fresh_store(P)
    config.set_train_precision("bf16")
    try:
        net = TecoGAN(ri.cuda(), rt.cuda(), FL)
        out = net.train()
    finally:
        config.set_train_precision("fp32")
    assert len(calls) >= 4 and len(calls) % 4 == 0, calls
    want = np.array([float(v) for v in ref["update_list"]])
    np.testing.assert_allclose(np.array(out["update_list"]), want, rtol=4e-2, atol=2e-3)
    st = net.train
    o = st.opt_g.n + st.opt_f.n
    got = st.bucket[o:o + st.opt_d.n].cpu()
    refg = torch.cat([ref["grads"][k].reshape(-1) for k in st.opt_d.names])
    assert refg.norm() > 0
    cos = float((got * refg).sum() / (got.norm() * refg.norm()))
    assert cos > 0.97, cos
