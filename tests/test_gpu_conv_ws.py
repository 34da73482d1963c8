"""The warp-specialised 64-input-channel path of teco_conv3x3_tc (conv3x3_ws_kernel): in-place residuals on the persistent
grid, ragged and tiny images, and more than one 64-channel output slice, against the oracle on bf16 operands."""
import pytest
import torch

from oracle import teco_oracle as O

pytestmark = pytest.mark.gpu


def _rnd(seed, *shape):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape, generator=g) * 2.0 - 1.0


def _bf(t):
    return t.to(torch.bfloat16).to(torch.float32)


def _check(got, ref, what):
    # fp32 accumulation of 576 bf16 products, one bf16 rounding of the output: the bound of the other conv3x3_tc tests
    err = (got.float().cpu() - ref).abs()
    bound = 2e-3 + ref.abs() / 128
    assert bool((err <= bound).all()), "%s: max err %.3e" % (what, err.max().item())


@pytest.mark.parametrize("n,h,w,act", [
    (150, 32, 32, 0),    # 1200 tiles: every CTA walks several tiles and the halo ring wraps
    (3, 19, 21, 2),      # ragged rows and columns: the TMA store clips, the lower warpgroup of the last tile row is idle
    (2, 5, 6, 1),        # an image smaller than one tile
    (1, 128, 128, 0),    # fewer tiles than SMs
])
def test_conv3x3_ws_inplace_residual(n, h, w, act):
    """res == y (the generator's residual blocks) gives the same bits as a separate residual tensor."""
    from tecogan_b200 import kernels as K
    x, wt, b = _bf(_rnd(1, n, h, w, 64)), _bf(_rnd(2, 3, 3, 64, 64) * (2.0 / 24.0)), _rnd(3, 64) * 0.1
    r = _bf(_rnd(4, n, h, w, 64))
    wpk = K.packed_weight(wt.cuda(), 64, 64)
    xb, rb = x.cuda().to(torch.bfloat16), r.cuda().to(torch.bfloat16)
    sep = K.conv3x3_tc(xb, wpk, b.cuda(), cout=64, act=act, res=rb)
    inplace = rb.clone()
    K.conv3x3_tc(xb, wpk, b.cuda(), inplace, cout=64, act=act, res=inplace)
    torch.cuda.synchronize()
    assert torch.equal(sep.view(torch.int16), inplace.view(torch.int16))
    acts = {0: lambda v: v, 1: torch.relu, 2: O.lrelu}
    _check(inplace, acts[act](O.conv2d(x, wt, b)) + r, "in-place residual")


def test_conv3x3_ws_staging_reuse_after_idle_tiles():
    """H = 24: the lower warpgroup has no rows in the image on the second tile row, so it stores nothing there.  W = 40
    (5 tiles per row) on the 132-CTA persistent grid gives each CTA tile rows in the order 0 0 0 1 1 0 0 0 1 1 ...: after
    two idle tiles the newest store is the one that last used the staging tile about to be rewritten, so the kernel must
    wait for that store itself to have read it, not only for the older ones.  Checked with and without a residual."""
    from tecogan_b200 import kernels as K
    n, h, w = 300, 24, 40
    x, wt, b = _bf(_rnd(11, n, h, w, 64)), _bf(_rnd(12, 3, 3, 64, 64) * (2.0 / 24.0)), _rnd(13, 64) * 0.1
    r = _bf(_rnd(14, n, h, w, 64))
    wpk = K.packed_weight(wt.cuda(), 64, 64)
    xb = x.cuda().to(torch.bfloat16)
    got = K.conv3x3_tc(xb, wpk, b.cuda(), cout=64, act=K.ACT_RELU)
    inplace = r.cuda().to(torch.bfloat16)
    K.conv3x3_tc(xb, wpk, b.cuda(), inplace, cout=64, res=inplace)
    torch.cuda.synchronize()
    z = O.conv2d(x, wt, b)
    _check(got, torch.relu(z), "no residual")
    _check(inplace, z + r, "in-place residual")


@pytest.mark.parametrize("cout", [128, 192])
def test_conv3x3_ws_output_slices(cout):
    """Cout > 64: one 64-channel slice per grid row, each with its own weights, bias, residual and output box."""
    from tecogan_b200 import kernels as K
    n, h, w = 5, 24, 40
    x, wt, b = _bf(_rnd(5, n, h, w, 64)), _bf(_rnd(6, 3, 3, 64, cout) * (2.0 / 24.0)), _rnd(7, cout) * 0.1
    r = _bf(_rnd(8, n, h, w, cout))
    wpk = K.packed_weight(wt.cuda(), 64, cout)
    got = K.conv3x3_tc(x.cuda().to(torch.bfloat16), wpk, b.cuda(), cout=cout, act=K.ACT_LRELU02)
    got_res = K.conv3x3_tc(x.cuda().to(torch.bfloat16), wpk, None, cout=cout, res=r.cuda().to(torch.bfloat16))
    torch.cuda.synchronize()
    _check(got, O.lrelu(O.conv2d(x, wt, b)), "lrelu")
    _check(got_res, O.conv2d(x, wt, torch.zeros(cout)) + r, "no bias + residual")
