"""CPU checks of tests/conv_simt_cases.py: the case tables reach every edge of the fp32 convolution and its weight gradient,
every layer the networks launch has a case, the exactness guard holds for every case, and the float64 restatements agree
with the oracle, with torch float64 autograd, and (through kernels._phase_taps and the weight slicing of
kernels.conv_transpose2x_raw) with the direct transposed convolution and the stride-2 input gradient."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import teco_oracle as O
from tests import conv_simt_cases as T


def test_case_tables_reach_every_required_edge():
    for family, (cases, f) in T.FAMILIES.items():
        seen = set().union(*(f(name, 132) for name in cases))
        assert T.REQUIRED[family] <= seen, (family, sorted(T.REQUIRED[family] - seen))


def test_every_layer_key_has_a_case():
    have = {T.launch_key(c) for c in T.LAYER_CASES.values()}
    for run, ks in T.LAYERS.items():
        assert ks, run
        assert ks <= have, (run, sorted(ks - have))
    assert len(have) == len(T.LAYER_CASES)
    for name, c in T.LAYER_CASES.items():
        assert (name in T.FWD_CASES) == isinstance(c, T.Fwd) and (name in T.WGRAD_CASES) == isinstance(c, T.Wg)


def test_layer_table_spot_checks():
    """Spot checks of the table against the networks' layer lists: LPIPS conv1, the transposed conv's four phases, the
    4x4 stride-2 input gradient's phases, the dense layer in the bf16 step."""
    fwd_keys = {k for ks in T.LAYERS.values() for k in ks if k[0] == "fwd"}
    assert ("fwd", 11, 11, 4, 2, 2, 3, 64, 3, 64, (1, 0, 1, 0), T.RELU, True, False, (1.0, 0.0), 0, False) in fwd_keys
    tconv = {(k[1], k[2], k[4], k[5], k[10]) for k in fwd_keys if k[10][0] == 2 and k[6] == 64 and k[12]}
    assert tconv == {(2, 2, 1, 1, (2, 0, 2, 0)), (2, 1, 1, 0, (2, 0, 2, 1)), (1, 2, 0, 1, (2, 1, 2, 0)),
                     (1, 1, 0, 0, (2, 1, 2, 1))}
    d4 = {(k[1], k[2], k[4], k[5], k[10]) for k in fwd_keys if k[10][0] == 2 and not k[12]}
    assert d4 == {(2, 2, 1, 1, (2, 0, 2, 0)), (2, 2, 1, 0, (2, 0, 2, 1)), (2, 2, 0, 1, (2, 1, 2, 0)),
                  (2, 2, 0, 0, (2, 1, 2, 1))}
    assert {k[0] for k in T.LAYERS["bf16 TecoGAN step"]} == {"fwd", "wgrad"}


@pytest.mark.parametrize("name", sorted(T.FWD_CASES))
def test_forward_guard_holds(name):
    T.fwd_guard(name)


@pytest.mark.parametrize("name", sorted(T.WGRAD_CASES))
def test_wgrad_guard_holds(name):
    T.wgrad_guard(name)


def test_epilogue_candidates():
    """None / ReLU give one candidate; LeakyReLU + residual and post != (1, 0) add the contracted rounding, which differs
    from the separately rounded one somewhere in those cases (so the second candidate is not vacuous)."""
    for name in ("lrelu_res_post", "cout100_cin36_pitch38_res", "none_nobias_post_half"):
        c = T.FWD_CASES[name]
        x, w, b, res = T.fwd_inputs(name)
        cands = T.epilogue(c, T.fwd_ref(c, x, w, b, res)[0], res)
        assert len(cands) == {"lrelu_res_post": 4, "cout100_cin36_pitch38_res": 1, "none_nobias_post_half": 2}[name]
        if name == "lrelu_res_post":
            assert any((a.view(np.int32) != cands[0].view(np.int32)).any() for a in cands[1:])


# ------------------------------------------------------------------------------------------------ restatement checks
def _apply(c, x, w, b=None, out=None):
    """z = conv + bias of one launch (float64), scattered through its output map into `out` (zeros if None)."""
    if out is None:
        out = np.zeros((c.N, c.out_H, c.out_W, c.out_cp))
    T._mapped(c, out)[...] = T.fwd_ref(c, x, w, b, None)[0]
    return out


def _phase_weights(w_oi, kys, kxs):
    """The [ty, tx, ci, co] slice kernels.conv_transpose2x_raw stacks for one phase."""
    return np.stack([np.stack([w_oi[ky, kx] for kx in kxs], 0) for ky in kys], 0).transpose(0, 1, 3, 2)


def _transpose_by_phases(x, w_oi, pad, b=None):
    N, H, W, _ = x.shape
    K = w_oi.shape[0]
    out = np.zeros((N, 2 * H, 2 * W, w_oi.shape[2]))
    for c in T.transpose_phases(N, H, W, K, x.shape[3], w_oi.shape[2], pad, T.NONE, b is not None):
        kys, _ = T.phase_taps(K, pad, c.out_map[1])
        kxs, _ = T.phase_taps(K, pad, c.out_map[3])
        _apply(c, x, _phase_weights(w_oi, kys, kxs), b, out)
    return out


def _grid(r, shape, den, kmax=16):
    return r.randint(-kmax, kmax + 1, shape) / den


@pytest.mark.parametrize("K,stride,hw", [(3, 1, (7, 9)), (1, 1, (4, 5)), (4, 2, (8, 10)), (3, 2, (7, 8)),
                                         (5, 1, (6, 3))])
def test_forward_restatement_matches_oracle_conv2d(K, stride, hw):
    r = np.random.RandomState(K * 10 + stride)
    x, w, b = _grid(r, (2,) + hw + (5,), 16), _grid(r, (K, K, 5, 7), 128), _grid(r, (7,), 2048, 2048)
    c = T.fwd(2, hw[0], hw[1], K, K, 5, 7, stride=stride)
    want = O.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride).numpy()
    np.testing.assert_array_equal(_apply(c, x, w, b), want)


def test_forward_restatement_matches_torch_at_lpips_conv1():
    """11 x 11, stride 4, pad 2 on both sides (torch padding=2), taps past the bottom and right edges."""
    r = np.random.RandomState(3)
    x, w = _grid(r, (1, 35, 39, 3), 16), _grid(r, (11, 11, 3, 4), 128)
    c = T.fwd(1, 35, 39, 11, 11, 3, 4, stride=4, pad=(2, 2), OH=8, OW=9, bias=False)
    want = Fn.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(w).permute(3, 2, 0, 1), stride=4,
                     padding=2).permute(0, 2, 3, 1).numpy()
    np.testing.assert_array_equal(_apply(c, x, w), want)


@pytest.mark.parametrize("hw", [(1, 1), (1, 4), (3, 1), (4, 6), (5, 7)])
def test_transposed_conv_by_phases_matches_oracle(hw):
    r = np.random.RandomState(sum(hw))
    x, w, b = _grid(r, (2,) + hw + (6,), 16), _grid(r, (3, 3, 5, 6), 128), _grid(r, (5,), 2048, 2048)
    want = O.conv2d_transpose(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b)).numpy()
    np.testing.assert_array_equal(_transpose_by_phases(x, w, 0, b), want)


@pytest.mark.parametrize("hw", [(1, 1), (1, 3), (2, 1), (3, 4), (5, 6)])
def test_stride2_input_gradient_by_phases_matches_autograd(hw):
    """dx of the 4 x 4 stride-2 SAME conv on a 2h x 2w input (pad 1 before) from dz [h, w]."""
    r = np.random.RandomState(7 + sum(hw))
    h, w_ = hw
    x = torch.from_numpy(_grid(r, (2, 2 * h, 2 * w_, 5), 16)).requires_grad_(True)
    w = torch.from_numpy(_grid(r, (4, 4, 5, 6), 128))
    dz = _grid(r, (2, h, w_, 6), 16)
    y = O.conv2d(x, w, None, 2)
    assert y.shape == dz.shape
    (dx,) = torch.autograd.grad(y, x, torch.from_numpy(dz))
    np.testing.assert_array_equal(_transpose_by_phases(dz, w.numpy(), 1), dx.numpy())


def _conv_grads_by_restatement(x, w, b, dy, K, stride):
    """dx, dw, db of kernels._Conv2d.backward restated: the launches T.conv_launches lists, fed as the wrapper feeds them."""
    N, H, W, Cin = x.shape
    Cout = w.shape[3]
    cs = T.conv_launches(Cin, Cout, K=K, stride=stride, bias=b is not None, N=N, hw=(H, W))
    f, wgc = cs[0], cs[-1]
    if stride == 1:
        dx = _apply(cs[1], dy, np.flip(w, (0, 1)).transpose(0, 1, 3, 2))
    else:
        dx = _transpose_by_phases(dy, w, f.pad_t)
    dw, _, db, _ = T.wgrad_ref(wgc, x, dy, None, None)
    return _apply(f, x, w, b), dx, dw, db


@pytest.mark.parametrize("K,stride,hw,bias", [(3, 1, (6, 7), True), (1, 1, (3, 5), True), (4, 2, (8, 6), False),
                                              (4, 2, (2, 2), True), (3, 1, (1, 1), True)])
def test_conv_gradient_restatements_match_torch_autograd(K, stride, hw, bias):
    r = np.random.RandomState(K + 3 * stride + hw[0])
    x = _grid(r, (2,) + hw + (5,), 16)
    w = _grid(r, (K, K, 5, 6), 128)
    b = _grid(r, (6,), 2048, 2048) if bias else None
    xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True) if bias else None
    y = O.conv2d(xt, wt, bt, stride)
    dy = _grid(r, tuple(y.shape), 128)
    grads = torch.autograd.grad(y, [t for t in (xt, wt, bt) if t is not None], torch.from_numpy(dy))
    y_r, dx, dw, db = _conv_grads_by_restatement(x, w, b, dy, K, stride)
    np.testing.assert_array_equal(y_r, y.detach().numpy())
    np.testing.assert_array_equal(dx, grads[0].numpy())
    np.testing.assert_array_equal(dw, grads[1].numpy())
    if bias:
        np.testing.assert_array_equal(db, grads[2].numpy())


@pytest.mark.parametrize("hw", [(1, 1), (3, 4), (4, 5)])
def test_transposed_conv_gradient_restatements_match_torch_autograd(hw):
    """kernels._ConvTranspose2x.backward: dx is the 3 x 3 stride-2 pad-0 conv of dz with w as stored, dw the weight
    gradient with the roles of input and output gradient swapped (stride 2 onto x's grid), db the sum of dz."""
    r = np.random.RandomState(11 + sum(hw))
    H, W = hw
    x = _grid(r, (2, H, W, 6), 16)
    w = _grid(r, (3, 3, 5, 6), 128)
    b = _grid(r, (5,), 2048, 2048)
    xt, wt, bt = (torch.from_numpy(a).requires_grad_(True) for a in (x, w, b))
    y = O.conv2d_transpose(xt, wt, bt)
    dz = _grid(r, tuple(y.shape), 128)
    gx, gw, gb = torch.autograd.grad(y, (xt, wt, bt), torch.from_numpy(dz))
    cs = T.tconv_launches(6, 5, act=T.NONE, N=2, hw=hw)
    dgrad, wgc = cs[4], cs[5]
    np.testing.assert_array_equal(_transpose_by_phases(x, w, 0, b), y.detach().numpy())
    np.testing.assert_array_equal(_apply(dgrad, dz, w), gx.numpy())
    dw = T.wgrad_ref(wgc, dz, x, None, None)[0]
    np.testing.assert_array_equal(dw, gw.numpy())
    np.testing.assert_array_equal(dz.sum((0, 1, 2)), gb.numpy())


def test_wgrad_restatement_reads_through_the_output_map_and_accumulates():
    """A strided output map reads dy at (oy sy + oy0, ox sx + ox0) only; accumulate adds the prior dw and db."""
    c = T.WGRAD_CASES["strided_map_acc"]
    x, dy, dw0, db0 = T.wgrad_inputs("strided_map_acc")
    dw, _, db, _ = T.wgrad_ref(c, x, dy, dw0, db0)
    dense = dy[:, 1::2, 0::2, :c.Cout].astype(np.float64)
    assert np.isfinite(dense).all() and np.isnan(dy[:, 0::2]).all()
    np.testing.assert_array_equal(db, dense.sum((0, 1, 2)) + db0)
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_(False)
    wt = torch.zeros((2, 2, c.Cin, c.Cout), dtype=torch.float64, requires_grad=True)
    xp = Fn.pad(xt.permute(0, 3, 1, 2), (c.pad_l, 1, c.pad_t, 1))
    y = Fn.conv2d(xp, wt.permute(3, 2, 0, 1))[:, :, :c.OH, :c.OW].permute(0, 2, 3, 1)
    (gw,) = torch.autograd.grad(y, wt, torch.from_numpy(dense))
    np.testing.assert_array_equal(dw, gw.numpy() + dw0)


def test_maxpool3s2_restatement_matches_torch():
    r = np.random.RandomState(5)
    x = r.randint(-3, 4, (2, 9, 8, 3)).astype(np.float32)
    want = Fn.max_pool2d(torch.from_numpy(x).permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1).numpy()
    np.testing.assert_array_equal(T.maxpool3s2_ref(x), want)
    x[0, 0, 0, 0] = np.nan
    assert np.isnan(T.maxpool3s2_ref(x)[0, 0, 0, 0])
