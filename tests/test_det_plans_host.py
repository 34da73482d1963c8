"""Host: the workspace sizes the fixed-order entry points ask for (their *_plan_bytes calls, which need no device) are the
ones tests/det_plans.py restates from the shapes alone, so the partitions behind them take no device property."""
import itertools

import pytest

from tests import det_plans as DP


def _lib_plan(name, *args):
    from tecogan_b200 import kernels as K
    return K.plan_bytes(name, *args)


@pytest.mark.parametrize("N,H,W,cin,cout", [(1, 8, 16, 64, 64), (40, 32, 32, 64, 64), (3, 13, 29, 64, 4),
                                            (4, 64, 64, 256, 64), (2, 8, 8, 512, 256), (9, 37, 11, 192, 128),
                                            (200, 64, 64, 64, 64)])
def test_wgrad_tc_partition(N, H, W, cin, cout):
    assert _lib_plan("teco_conv3x3_wgrad_tc_det", N, H, W, cin, cout) == DP.wgrad_tc_bytes(N, H, W, cin, cout)
    splits, tpc = DP.wgrad_tc(N, H, W, cin, cout)
    tiles = N * DP.cdiv(W, 16) * DP.cdiv(H, 8)
    assert (splits - 1) * tpc < tiles <= splits * tpc


@pytest.mark.parametrize("N,H,W,Cin,Cout,K,with_bias", [(1, 5, 7, 3, 64, 3, 1), (4, 32, 32, 64, 64, 3, 1),
                                                         (2, 33, 17, 20, 3, 3, 0), (4, 64, 64, 256, 128, 4, 1),
                                                         (1, 1, 1, 1, 1, 1, 1), (40, 128, 128, 64, 3, 3, 1)])
def test_wgrad_f32_partition(N, H, W, Cin, Cout, K, with_bias):
    from tecogan_b200._ffi import ConvDesc
    d = ConvDesc(N=N, H=H, W=W, Cin=Cin, OH=H, OW=W, Cout=Cout, KH=K, KW=K, stride=1, pad_t=K // 2, pad_l=K // 2,
                 out_H=H, out_W=W, out_sy=1, out_oy=0, out_sx=1, out_ox=0, in_cpitch=Cin, out_cpitch=Cout, act=0,
                 post_scale=1.0, post_shift=0.0)
    assert _lib_plan("teco_conv2d_wgrad_f32_det", d, with_bias) == DP.wgrad_f32_bytes(N * H * W, K, K, Cin, Cout, with_bias)


@pytest.mark.parametrize("npix,C", list(itertools.product([1, 7, 1000, 1025, 70000, 5_000_000], [1, 3, 64, 100, 256])))
def test_bias_bn_loss_partitions(npix, C):
    assert _lib_plan("teco_bias_grad_f32_det", npix, C) == DP.bias(npix, C)[0] * C * 4
    assert _lib_plan("teco_bn_det", npix, C) == DP.bn(npix)[0] * 2 * C * 4
    assert _lib_plan("teco_loss_det", npix, C) == DP.loss_bytes(npix, C)


@pytest.mark.parametrize("N,H,W", [(1, 2, 2), (3, 17, 31), (40, 128, 128)])
def test_warp_partition(N, H, W):
    assert _lib_plan("teco_warp_bwd_f32_det", N, H, W) == DP.warp_bytes(N, H, W)


def test_plans_reject_bad_shapes():
    with pytest.raises(ValueError):
        _lib_plan("teco_bias_grad_f32_det", 10, 257)
    with pytest.raises(ValueError):
        _lib_plan("teco_bn_det", 0, 3)
    with pytest.raises(ValueError):
        _lib_plan("teco_warp_bwd_f32_det", 1, 1, 5)
    with pytest.raises(ValueError):
        _lib_plan("teco_conv3x3_wgrad_tc_det", 1, 8, 8, 0, 64)
