"""Host checks of tests/train_nets_exact.py: with rounding off the restatement is the oracle's float64 autograd, its
guards hold on every case the GPU test runs, and the case tables reach every kernel path the issue of bit-exact training
tests has to cover."""
import pytest
import torch

from oracle import teco_oracle as O
from tests import nets_exact as E
from tests import train_nets_exact as T


def _leaves(p):
    return {k: v.clone().requires_grad_(True) for k, v in p.items()}


def _close(got, ref, what, rel=1e-12):
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= rel * scale, "%s: max error %.3g, scale %.3g" % (what, err, scale)


def _compare(outs_r, outs_o, dys, inputs, what):
    """Outputs equal, and the gradients of sum <out, dy> w.r.t. inputs (a list of (name, tensor, slice or None))."""
    for i, (a, b) in enumerate(zip(outs_r, outs_o)):
        _close(a, b, "%s output %d" % (what, i))
    gr = torch.autograd.grad(outs_r, [t for _, t, _ in inputs[0]], dys)
    go = torch.autograd.grad(outs_o, [t for _, t, _ in inputs[1]], dys)
    for (name, _, sl), a, b in zip(inputs[0], gr, go):
        if sl is not None:
            a, b = a[sl], b[sl]
        _close(a, b, "%s d/d %s" % (what, name))


def test_generator_restatement_without_rounding_is_the_oracle():
    """Inputs, weights and biases: every gradient equals O.generator_F's float64 autograd.  The LR channels 0:3 are left
    out of the input gradient: the oracle differentiates bicubic_four, the device (and the restatement) does not."""
    p, x = E.generator_operands(7, 2, 8, 12, 2)
    dy = T.grad_grid(8, (2, 32, 48, 3))
    pr, po = _leaves(p), _leaves(p)
    xr, xo = x.clone().requires_grad_(), x.clone().requires_grad_()
    out_r = T.generator_train_ref(pr, xr, 2, T.TrainRounding(on=False), O.bicubic_four(x[..., 0:3]))
    out_o = O.generator_F(po, xo, 2)
    sl = (Ellipsis, slice(3, 51))
    _compare([out_r], [out_o], [dy], ([("inputs", xr, sl)] + [(k, v, None) for k, v in pr.items()],
                                      [("inputs", xo, sl)] + [(k, v, None) for k, v in po.items()]), "generator")


@pytest.mark.parametrize("signed", [False, True], ids=["nonneg", "signed"])
def test_fnet_restatement_without_rounding_is_the_oracle(signed):
    p, x = E.fnet_operands(9, 2, 16, 24, signed)
    dy = T.grad_grid(10, (2, 16, 24, 2))
    pr, po = _leaves(p), _leaves(p)
    xr, xo = x.clone().requires_grad_(), x.clone().requires_grad_()
    out_r = T.fnet_train_ref(pr, xr, T.TrainRounding(on=False))
    out_o = O.fnet(po, xo)
    _compare([out_r], [out_o], [dy], ([("inputs", xr, None)] + [(k, v, None) for k, v in pr.items()],
                                      [("inputs", xo, None)] + [(k, v, None) for k, v in po.items()]), "fnet")


def test_vgg_restatement_without_rounding_is_the_oracle():
    """The four raw taps of O.vgg19_features (norm_flag=False) and the input gradient; the weights are frozen."""
    p, x = T.vgg_operands(11, 1, 32, 48)
    xr, xo = x.clone().requires_grad_(), x.clone().requires_grad_()
    out_r = T.vgg_train_ref(p, xr, T.TrainRounding(on=False))
    out_o = O.vgg19_features(p, xo, norm_flag=False)
    assert list(out_r) == list(out_o) == O.VGG_TAPS
    dys = [T.grad_grid(12 + i, out_o[k].shape) for i, k in enumerate(O.VGG_TAPS)]
    _compare([out_r[k] for k in O.VGG_TAPS], [out_o[k] for k in O.VGG_TAPS], dys,
             ([("inputs", xr, None)], [("inputs", xo, None)]), "vgg")


def _layer_record(layers):
    """(what, input shape, weight shape) as TrainRounding records them."""
    out = []
    for L in layers:
        cin = L.cin
        shape = (3, 3, L.cout, cin) if L.transpose else (3, 3, cin, L.cout)
        out.append((L.what, (L.n, L.h, L.w, cin), shape))
    return out


def _exact_bias(R, names):
    """Bias gradients held to bits: every bias interval of `names` is one point."""
    for k in names:
        lo, hi = R.bias[k]
        assert torch.equal(lo, hi), k + ": bias gradient not exact"


@pytest.mark.parametrize("name", list(T.GEN_CASES))
def test_guards_hold_on_every_generator_case(name):
    """The rounding-on restatement on the GPU test's operands passes every guard, walks the layers gen_layers lists, and
    every bias gradient is exact."""
    B, h, w, N, seed, density = T.GEN_CASES[name]
    p, x = E.generator_operands(seed, B, h, w, N)
    dy = T.sparse_grad(seed, (B, 4 * h, 4 * w, 3), density)
    R = T.TrainRounding(check=True)
    pl, xl = _leaves(p), x.clone().requires_grad_()
    out = T.generator_train_ref(pl, xl, N, R, R.f32(O.bicubic_four(x[..., 0:3])))
    torch.autograd.grad(out, [xl] + list(pl.values()), dy)
    assert R.layers == _layer_record(T.gen_layers(B, h, w, N))
    _exact_bias(R, [L.what for L in T.gen_layers(B, h, w, N)])


@pytest.mark.parametrize("signed", [False, True], ids=["nonneg", "signed"])
@pytest.mark.parametrize("name", list(T.FNET_CASES))
def test_forward_guards_hold_on_every_fnet_case(name, signed):
    """FNet's forward on the GPU test's operands passes every conv and resize guard and walks fnet_layers."""
    n, h, w = T.FNET_CASES[name]
    p, x = E.fnet_operands(T.fnet_seed(name, signed), n, h, w, signed)
    R = T.TrainRounding(check=True)
    T.fnet_train_ref(p, x, R)
    assert R.layers == _layer_record(T.fnet_layers(n, h, w))


@pytest.mark.parametrize("name", list(T.FNET_BWD_CASES))
def test_guards_hold_on_every_fnet_backward_case(name):
    """FNet forward and backward on the 'signed' operands with sparse upstream flow gradients: every guard passes (the
    head's two act_bwd candidates included, here on the host's flow), the layers are fnet_layers', the input gradient is
    not zero, and besides the head some layer's bias gradient sums a dz that is not bf16-exact (LeakyReLU's negative
    branch: its interval is wider than one point), and every parameter's gradient is non-zero."""
    c = T.FNET_BWD_CASES[name]
    p, x = E.fnet_operands(c.seed, c.n, c.h, c.w, True)
    dy = T.sparse_grad(c.seed, (c.n, c.h, c.w, 2), c.density)
    R = T.TrainRounding(check=True)
    pl, xl = _leaves(p), x.clone().requires_grad_()
    flow = T.fnet_train_ref(pl, xl, R)
    grads = torch.autograd.grad(flow, [xl] + list(pl.values()), dy)
    layers = T.fnet_layers(c.n, c.h, c.w, backward=True)
    assert R.layers == _layer_record(layers)
    assert bool((grads[0] != 0).any()), "the input gradient is zero"
    wide = [k for k, (lo, hi) in R.bias.items() if not torch.equal(lo, hi)]
    assert T.FNET + "output_stage/conv2/Conv" in wide and len(wide) > 1, wide
    assert all(bool((g != 0).any()) for g in grads[1:])


@pytest.mark.parametrize("name", list(T.VGG_CASES))
def test_guards_hold_on_every_vgg_case(name):
    n, h, w = T.VGG_CASES[name]
    p, x = T.vgg_operands(T.vgg_seed(name), n, h, w)
    R = T.TrainRounding(check=True)
    xl = x.clone().requires_grad_()
    out = T.vgg_train_ref(p, xl, R)
    dys = [T.grad_grid(T.vgg_seed(name) + i, out[k].shape) for i, k in enumerate(O.VGG_TAPS)]
    torch.autograd.grad([out[k] for k in O.VGG_TAPS], [xl], dys)
    assert R.layers == _layer_record(T.vgg_layers(n, h, w))
    assert not R.bias                                      # frozen: no weight or bias gradient


def test_case_tables_reach_every_required_feature():
    """The launches the GPU test checks over the case tables reach every key of REQUIRED.  Every channel count is padded
    to 64, so the training graph never reaches conv3x3_wgmma_kernel<32>."""
    seen, kernels = set(), set()
    for name, layers in T.case_layers().items():
        for L in layers:
            seen |= T.layer_features(L)
        kernels |= T.kernels_reached(layers)
    assert T.REQUIRED <= seen, sorted(T.REQUIRED - seen)
    assert kernels == {"ws<0>", "ws<1>", "wgmma<64>", "wgmma<16>"}, kernels
