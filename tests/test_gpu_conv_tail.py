"""The transposed convolution (teco_conv3x3_tc mode 1) against the oracle on bf16 operands, beyond the shapes of
test_gpu_kernels.py::test_conv_transpose_tc_matches_oracle_on_bf16_operands: the warp-specialised kernel's 16 x 16 output
boxes clipped at the 2H x 2W edges, idle warpgroups below the image, more tiles than the persistent grid, two
64-channel output slices, and the inputs that stay on conv3x3_wgmma_kernel<1, NT> (Cout not a multiple of 64, a
residual).  The output is prefilled, so a pixel the kernel never writes fails the check."""
import pytest
import torch

from oracle import teco_oracle as O
from tests.test_gpu_kernels import _bf, assert_close, dev, rnd

pytestmark = pytest.mark.gpu

_ACTS = {0: lambda v: v, 1: torch.relu, 2: O.lrelu}


@pytest.mark.parametrize("n,h,w,cout,act,res", [
    (3, 19, 21, 64, 1, False),      # ragged: the 16 x 16 output boxes are clipped at 38 x 42
    (2, 5, 6, 64, 2, False),        # an image smaller than one tile
    (60, 24, 40, 64, 1, False),     # 600 tiles: the halo ring wraps, staging tiles are reused after idle lower warpgroups
    (2, 24, 40, 128, 2, False),     # two 64-channel output slices
    (1, 9, 8, 128, 0, False),       # one tile per slice; the lower warpgroup's only row is row 8
    (3, 19, 21, 32, 1, False),      # Cout = 32: conv3x3_wgmma_kernel<1, 32>
    (2, 24, 20, 48, 2, False),      # Cout = 48: conv3x3_wgmma_kernel<1, 16>, three output slices
    (2, 19, 21, 64, 0, True),       # a residual: conv3x3_wgmma_kernel<1, 32>
])
def test_conv_transpose_tc_shapes_and_paths(n, h, w, cout, act, res):
    from tecogan_b200 import kernels as K
    x, wt, b = _bf(rnd(1, n, h, w, 64)), _bf(rnd(2, 3, 3, cout, 64) * 0.06), rnd(3, cout) * 0.1
    r = _bf(rnd(4, n, 2 * h, 2 * w, cout)) if res else None
    wpk = K.packed_weight(dev(wt), 64, cout, transpose_layout=True)
    y = torch.full((n, 2 * h, 2 * w, cout), 7.0, device="cuda", dtype=torch.bfloat16)
    K.conv3x3_tc(dev(x).to(torch.bfloat16), wpk, dev(b), y, cout=cout, act=act, mode=1,
                 res=dev(r).to(torch.bfloat16) if res else None)
    ref = _ACTS[act](O.conv2d_transpose(x, wt, b))
    if res:
        ref = ref + r
    assert_close(y, ref, 2e-3, 1.0 / 128, what="conv_transpose_tc")
