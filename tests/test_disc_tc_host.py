"""The space-to-depth-2 identity behind the discriminator's tensor-core 4x4 stride-2 convolutions (kernels._Conv4x4S2TC,
teco_conv4x4s2_tc), checked in float64 against a direct 4x4/2 SAME convolution and its two gradients, and the rule that
sends a conv2() there."""
import pytest
import torch
import torch.nn.functional as Fn

from tecogan_b200 import config, kernels as K, variables as V
from tecogan_b200.lib import ops
from tecogan_b200.variables import VariableStore, set_default_store, variable_scope

# discriminator_F's disblocks at the 128 x 128 TecoGAN crop: (input H = W, Cin, Cout)
D_SHAPES = [(128, 64, 64), (64, 64, 64), (32, 64, 128), (16, 128, 256)]


def _direct(x, w):
    """TF conv2d 4x4 stride 2 SAME, NHWC / HWIO: on even H, W one row / column of padding before and one after."""
    y = Fn.conv2d(Fn.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1)), w.permute(3, 2, 0, 1), stride=2)
    return y.permute(0, 2, 3, 1)


def _conv3x3_same(xs, wp):
    return Fn.conv2d(xs.permute(0, 3, 1, 2), wp.permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1)


def _s2d(x):
    N, H, W, C = x.shape
    return x.view(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H // 2, W // 2, 4 * C)


def _d2s(xs, C):
    N, h, w, _ = xs.shape
    return xs.view(N, h, w, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * h, 2 * w, C)


def _w_prime(w):
    """W' [3, 3, 4 Cin, Cout]: w scattered into the live (tap, phase) slots, zero elsewhere."""
    Cin, Cout = w.shape[2], w.shape[3]
    wp = torch.zeros((36, Cin, Cout), dtype=w.dtype)
    wp[K._c4s2_rows()] = w.reshape(16, Cin, Cout)
    return wp.view(3, 3, 4 * Cin, Cout)


def test_slot_map_is_ky_2ty_plus_py_minus_1():
    """The Python slot map and the rule the packing kernel uses (ky = 2 ty + py - 1, columns alike) are the same map:
    16 distinct live slots, each phase a whole block of Cin channels."""
    rows = K._c4s2_rows()
    assert len(set(rows)) == 16
    for ky in range(4):
        for kx in range(4):
            tap, ph = divmod(rows[ky * 4 + kx], 4)
            (ty, tx), (py, px) = divmod(tap, 3), divmod(ph, 2)
            assert (2 * ty + py - 1, 2 * tx + px - 1) == (ky, kx)
    assert [divmod(ky + 1, 2) for ky in range(4)] == [(0, 1), (1, 0), (1, 1), (2, 0)]


@pytest.mark.parametrize("H,Cin,Cout", D_SHAPES)
def test_space_to_depth_identity_forward_and_gradients_float64(H, Cin, Cout):
    g = torch.Generator().manual_seed(H + Cin + Cout)
    N = 1 if H == 128 else 2
    x = torch.randn(N, H, H, Cin, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(4, 4, Cin, Cout, generator=g, dtype=torch.float64, requires_grad=True)
    dz = torch.randn(N, H // 2, H // 2, Cout, generator=g, dtype=torch.float64)
    y = _direct(x, w)
    dx_ref, dw_ref = torch.autograd.grad(y, (x, w), dz)

    wp = _w_prime(w.detach())
    xs = _s2d(x.detach())
    torch.testing.assert_close(_conv3x3_same(xs, wp), y.detach(), rtol=1e-12, atol=1e-9)
    # input gradient: the flipped-tap transpose W'' of W' on dz, then depth-to-space
    wpp = torch.flip(wp, dims=(0, 1)).permute(0, 1, 3, 2)
    torch.testing.assert_close(_d2s(_conv3x3_same(dz, wpp), Cin), dx_ref, rtol=1e-12, atol=1e-9)
    # weight gradient: the 3x3 weight gradient of (xs, dz) at the 16 live slots
    wfree = torch.zeros_like(wp, requires_grad=True)
    (dwp,) = torch.autograd.grad(_conv3x3_same(xs, wfree), (wfree,), dz)
    dw = dwp.reshape(36, Cin, Cout)[K._c4s2_rows()].view(4, 4, Cin, Cout)
    torch.testing.assert_close(dw, dw_ref, rtol=1e-12, atol=1e-9)


def test_fits_rule():
    assert K.conv4x4s2_tc_fits(128, 128, 64, 64) and K.conv4x4s2_tc_fits(16, 16, 128, 256) and K.conv4x4s2_tc_fits(2, 6, 64, 512)
    assert not K.conv4x4s2_tc_fits(127, 128, 64, 64)      # odd H
    assert not K.conv4x4s2_tc_fits(128, 9, 64, 64)        # odd W
    assert not K.conv4x4s2_tc_fits(32, 32, 3, 64)         # Cin not a multiple of 64
    assert not K.conv4x4s2_tc_fits(32, 32, 256, 64)       # 4 Cin beyond the 3x3 kernel's 512 input channels
    assert not K.conv4x4s2_tc_fits(32, 32, 64, 48)        # Cout not a multiple of 64


@pytest.fixture
def dispatch(monkeypatch):
    """ops.conv2 on CPU tensors with both kernels replaced by recorders: returns conv(shape, ...) -> the kernel picked."""
    calls = []
    monkeypatch.setattr(K, "conv4x4s2_train_tc", lambda *a, **k: calls.append("tc"))
    monkeypatch.setattr(K, "conv2d", lambda *a, **k: calls.append("fp32"))
    monkeypatch.setattr(K, "conv3x3_train_tc", lambda *a, **k: calls.append("tc3x3"))
    monkeypatch.setitem(V._state, "store", V._state["store"])   # each call below installs its own CPU store
    prev = config.train_precision()
    config.set_train_precision("bf16")

    def conv(shape, kernel=4, stride=2, cout=64, grad=True, **kw):
        calls.clear()
        set_default_store(VariableStore(device="cpu"))
        with torch.set_grad_enabled(grad), variable_scope("disblock"):
            ops.conv2(torch.zeros(shape), kernel, cout, stride, use_bias=False, scope="conv1", **kw)
        return calls[0]

    yield conv
    config.set_train_precision(prev)


def test_dispatch_rule(dispatch):
    assert dispatch((2, 128, 128, 64)) == "tc"
    assert dispatch((2, 16, 16, 128), cout=256) == "tc"
    assert dispatch((2, 127, 128, 64)) == "fp32"          # odd sizes: TF's SAME padding is not one row before
    assert dispatch((2, 128, 63, 64)) == "fp32"
    assert dispatch((2, 32, 32, 3)) == "fp32"             # Cin not a multiple of 64
    assert dispatch((2, 32, 32, 64), cout=48) == "fp32"
    assert dispatch((2, 32, 32, 64), kernel=3, stride=2) == "fp32"
    assert dispatch((2, 32, 32, 64), kernel=4, stride=1) == "fp32"
    assert dispatch((2, 32, 32, 64), grad=False) == "fp32"   # inference
    with config.train_forward():
        assert dispatch((2, 32, 32, 64), grad=False) == "tc"  # the trainer's evaluate() runs the step's kernels
    config.set_train_precision("fp32")
    assert dispatch((2, 128, 128, 64)) == "fp32"
