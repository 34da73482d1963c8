"""The transposed convolution (teco_conv3x3_tc mode 1) against the oracle on bf16 operands, beyond the shapes of
test_gpu_kernels.py::test_conv_transpose_tc_matches_oracle_on_bf16_operands: the warp-specialised kernel's 16 x 16 output
boxes clipped at the 2H x 2W edges, idle warpgroups below the image, more tiles than the persistent grid and two
64-channel output slices.  The output is prefilled, so a pixel the kernel never writes fails the check.
conv3x3_ws_kernel<1> is the only mode-1 kernel: the launches it does not take (Cin other than 64, Cout not a multiple of
64, a residual, an fp32 output) are refused, with no kernel launched and nothing written."""
import pytest
import torch

from oracle import teco_oracle as O
from tests.test_gpu_conv_exact import _profiled_conv_kernels
from tests.test_gpu_kernels import _bf, assert_close, dev, rnd

pytestmark = pytest.mark.gpu

_ACTS = {0: lambda v: v, 1: torch.relu, 2: O.lrelu}
FILL = 7.0

# Mode-1 launches outside conv3x3_ws_kernel<1>'s rule: (n, h, w, cin, cout, residual, fp32 output), and the condition
# teco_conv3x3_tc names in refusing them
REFUSED = {
    "cout32": ((3, 19, 21, 64, 32, False, False), "Cout a multiple of 64"),
    "cout48": ((2, 24, 20, 64, 48, False, False), "Cout a multiple of 64"),
    "residual": ((2, 19, 21, 64, 64, True, False), "no residual"),
    "cin128": ((2, 9, 11, 128, 64, False, False), "Cin 64"),
    "f32_output": ((2, 19, 21, 64, 64, False, True), "no fp32 output"),
}


def _filled(n, h, w, c, dtype=torch.bfloat16):
    """An [n, 2h, 2w, c] output prefilled with FILL."""
    return torch.full((n, 2 * h, 2 * w, c), FILL, device="cuda", dtype=dtype)


def _launch(y, cin, act, res=False, out_f32=None):
    """One mode-1 launch into y on seeded bf16 operands; returns the operands (x, w, bias, residual) on the host."""
    from tecogan_b200 import kernels as K
    n, h, w, cout = y.shape[0], y.shape[1] // 2, y.shape[2] // 2, y.shape[3]
    x, wt, b = _bf(rnd(1, n, h, w, cin)), _bf(rnd(2, 3, 3, cout, cin) * 0.06), rnd(3, cout) * 0.1
    r = _bf(rnd(4, n, 2 * h, 2 * w, cout)) if res else None
    wpk = K.packed_weight(dev(wt), cin, cout, transpose_layout=True)
    K.conv3x3_tc(dev(x).to(torch.bfloat16), wpk, dev(b), y, cout=cout, act=act, mode=1,
                 res=dev(r).to(torch.bfloat16) if res else None, out_f32=out_f32)
    return x, wt, b, r


@pytest.mark.parametrize("n,h,w,cout,act,res", [
    (3, 19, 21, 64, 1, False),      # ragged: the 16 x 16 output boxes are clipped at 38 x 42
    (2, 5, 6, 64, 2, False),        # an image smaller than one tile
    (60, 24, 40, 64, 1, False),     # 600 tiles: the halo ring wraps, staging tiles are reused after idle lower warpgroups
    (2, 24, 40, 128, 2, False),     # two 64-channel output slices
    (1, 9, 8, 128, 0, False),       # one tile per slice; the lower warpgroup's only row is row 8
])
def test_conv_transpose_tc_shapes_and_paths(n, h, w, cout, act, res):
    y = _filled(n, h, w, cout)
    x, wt, b, r = _launch(y, 64, act, res)
    ref = _ACTS[act](O.conv2d_transpose(x, wt, b))
    if res:
        ref = ref + r
    assert_close(y, ref, 2e-3, 1.0 / 128, what="conv_transpose_tc")


@pytest.mark.parametrize("name", list(REFUSED))
def test_conv_transpose_tc_refuses_what_conv3x3_ws_kernel_1_does_not_take(name):
    """Mode 1 takes Cin 64, Cout a multiple of 64, a bf16 output and no residual.  Any other mode-1 launch raises
    ValueError naming the condition it fails, and y and the fp32 output keep their fill."""
    (n, h, w, cin, cout, res, f32), need = REFUSED[name]
    y = _filled(n, h, w, cout)
    out = _filled(n, h, w, cout, torch.float32) if f32 else None
    with pytest.raises(ValueError, match=need):
        _launch(y, cin, 1, res, out)
    torch.cuda.synchronize()
    assert bool((y == FILL).all()), name
    assert out is None or bool((out == FILL).all()), name


def _refused_then_accepted():
    for (n, h, w, cin, cout, res, f32), _ in REFUSED.values():
        with pytest.raises(ValueError):
            _launch(_filled(n, h, w, cout), cin, 1, res, _filled(n, h, w, cout, torch.float32) if f32 else None)
    _launch(_filled(1, 9, 8, 64), 64, 1)
    torch.cuda.synchronize()


def test_conv_transpose_tc_refusals_launch_no_convolution_kernel():
    """Recorded by the profiler: the refused launches run no convolution kernel, and the accepted launch after them runs
    conv3x3_ws_kernel<1>."""
    assert _profiled_conv_kernels("tests.test_gpu_conv_tail", "_refused_then_accepted") == ["ws<1>"]
