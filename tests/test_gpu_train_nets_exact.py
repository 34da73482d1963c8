"""The bf16 training graph (train precision 'bf16': lib/frvsr.py generator_F and fnet, lib/Teco.py::_vgg_raw on
_Conv3x3TC and _ConvTranspose2xTC) against the float64 restatement of tests/train_nets_exact.py, which walks the
oracle's layers and rounds where the training kernels round, forward and backward.  On the operands built there every
sum is exact (host guards check each conv, gradient, resize and gradient sum before anything is compared), so:
  * generator_F: the HR output, the input gradient (all 51 channels: the LR ones carry the input conv's dx alone, the
    bicubic residual is not differentiated) and every weight gradient equal the reference bit for bit, and every bias
    gradient too (its interval is one point on these operands); also over two frames with reuse=True, under
    deterministic mode, and for the forward-only evaluation Network.train.evaluate runs;
  * _vgg_raw with frozen weights: the four tapped maps and the input gradient bit for bit, and no weight or bias
    gradient is computed;
  * fnet: the flow within the tanh bound of test_gpu_conv_exact.py on both operand sets; on the 'signed' set with
    sparse upstream flow gradients (train_nets_exact.FNET_BWD_CASES) also the input gradient and every weight gradient
    bit for bit, and every bias gradient bit for bit or, where its dz is not on one grid (the flow head, LeakyReLU's
    negative branch), within its interval; and once more under deterministic mode.
This pins the training graph's wiring: each layer's route, packed weights and dgrad packing, the bf16 rounding points,
the residual add and its gradient, LeakyReLU's and tanh24's backward, the narrow output stages' padded weight-gradient
columns, the bias gradient's fp32 operand, and the packed-weight cache across the recurrent loop, which the oracle tolerances of test_gpu_train.py miss."""
import types

import pytest
import torch

from oracle import teco_oracle as O
from tests import nets_exact as E
from tests import train_nets_exact as T
from tests.test_gpu_conv_exact import REL_BOUND, _bits, _check_f32, _is_f32


@pytest.fixture
def train_bf16():
    """Train precision 'bf16' (inference precision 'fp32', as the training step sets it); loads operands into a new
    default VariableStore.  Precisions, the deterministic flag and the store come back afterwards."""
    from tecogan_b200 import config, variables as V
    saved = (config.precision(), config.train_precision(), config.deterministic(), V.default_store())

    def load(p, trainable=True):
        st = V.set_default_store(V.VariableStore())
        st.load(p)
        for k in st:
            st[k].requires_grad_(trainable)
        return st
    config.set_precision("fp32")
    config.set_train_precision("bf16")
    yield load
    config.set_precision(saved[0])
    config.set_train_precision(saved[1])
    config.set_deterministic(saved[2])
    V.set_default_store(saved[3])


def _check_bias(got, bounds, what):
    """got within [lo, hi]; bit for bit where the interval is one point."""
    lo, hi = (b.cpu() for b in bounds)
    point = lo == hi
    assert _is_f32(lo[point]), what + ": an exact bias gradient is not an fp32 value"
    bad = (point & (_bits(got) != _bits(lo.float()))) | (~point & ((got.double() < lo) | (got.double() > hi)))
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d / %d elements outside [lo, hi], first at %d: got %r, expected [%r, %r]" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(lo[i]), float(hi[i])))


def _check_grads(names, got, ref, R, what):
    for k, g, r in zip(names, got, ref):
        if k.endswith("/biases"):
            _check_bias(g.cpu(), R.bias[k[:-len("/biases")]], "%s %s" % (what, k))
        else:
            assert _is_f32(r), "%s %s: the reference gradient is not an fp32 value" % (what, k)
            _check_f32(g.cpu(), r.cpu(), "%s %s" % (what, k))


def _generator(load, p, xs, dys, N):
    """generator_F on the device over the frames xs (reuse=True after the first) and the gradients of
    sum <out, dy>; the reference likewise.  Returns (outs, ref outs, names, grads, ref grads, R)."""
    from tecogan_b200 import kernels as K, variables as V
    from tecogan_b200.lib.frvsr import generator_F
    st = load(p)
    K.tc_cache_clear()
    names = list(p)
    flags = types.SimpleNamespace(num_resblock=N)
    xd = [x.cuda().float().requires_grad_() for x in xs]
    with V.variable_scope("generator"):
        outs = [generator_F(x, 3, reuse=i > 0, FLAGS=flags) for i, x in enumerate(xd)]
    grads = torch.autograd.grad(outs, xd + [st[k] for k in names], [dy.cuda().float() for dy in dys])
    torch.cuda.synchronize()
    R = T.TrainRounding(check=True)
    pl = {k: v.cuda().requires_grad_() for k, v in p.items()}
    xl = [x.cuda().requires_grad_() for x in xs]
    refs = [T.generator_train_ref(pl, x, N, R, K.bicubic4(xx[..., 0:3].detach().contiguous()).double())
            for x, xx in zip(xl, xd)]
    rgrads = torch.autograd.grad(refs, xl + [pl[k] for k in names], [dy.cuda() for dy in dys])
    return outs, refs, names, grads, rgrads, R


def _check_generator(res, nframes, what):
    outs, refs, names, grads, rgrads, R = res
    for i in range(nframes):
        _check_f32(outs[i].detach().cpu(), refs[i].detach().cpu(), "%s frame %d out" % (what, i))
        _check_f32(grads[i].cpu(), rgrads[i].cpu(), "%s frame %d d/d gen_inputs" % (what, i))
    _check_grads(names, grads[nframes:], rgrads[nframes:], R, what)


def _gen_case(name):
    B, h, w, N, seed, density = T.GEN_CASES[name]
    p, x = E.generator_operands(seed, B, h, w, N)
    return p, x, T.sparse_grad(seed, (B, 4 * h, 4 * w, 3), density), N


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(T.GEN_CASES))
def test_generator_F_training_graph_matches_float64_reference_bit_for_bit(name, train_bf16):
    p, x, dy, N = _gen_case(name)
    _check_generator(_generator(train_bf16, p, [x], [dy], N), 1, name)


@pytest.mark.gpu
def test_generator_F_recurrent_reuse_sums_both_frames_bit_for_bit(train_bf16):
    """Two frames through generator_F (reuse=True on the second) and one backward: each parameter's gradient, summed over
    the frames by autograd in fp32, equals the reference; the packed weights are cached across the two frames."""
    p, x, dy, N = _gen_case("1x13x19 N=3")
    seed = T.GEN_CASES["1x13x19 N=3"].seed + 100
    x2 = E.generator_operands(seed, 1, 13, 19, N)[1]
    dy2 = T.sparse_grad(seed, dy.shape)
    _check_generator(_generator(train_bf16, p, [x, x2], [dy, dy2], N), 2, "recurrent")


@pytest.mark.gpu
def test_generator_F_deterministic_mode_gives_the_same_bits(train_bf16):
    """config.set_deterministic(True): the fixed-order weight and bias gradient kernels give the reference's bits."""
    from tecogan_b200 import config
    config.set_deterministic(True)
    p, x, dy, N = _gen_case("2x32x32 N=3")
    _check_generator(_generator(train_bf16, p, [x], [dy], N), 1, "deterministic")


@pytest.mark.gpu
def test_generator_F_forward_without_grad_equals_the_training_forward(train_bf16):
    """Network.train.evaluate's validation forward: inference precision 'fp32', torch.no_grad() and
    config.train_forward() run the training kernels, so the output has the grad-enabled forward's bits."""
    from tecogan_b200 import config, kernels as K, variables as V
    from tecogan_b200.lib.frvsr import generator_F
    p, x, dy, N = _gen_case("1x13x19 N=3")
    outs, refs = _generator(train_bf16, p, [x], [dy], N)[:2]
    K.tc_cache_clear()
    with torch.no_grad(), config.train_forward(), V.variable_scope("generator"):
        out = generator_F(x.cuda().float(), 3, reuse=True, FLAGS=types.SimpleNamespace(num_resblock=N))
    torch.cuda.synchronize()
    assert torch.equal(_bits(out.cpu()), _bits(outs[0].detach().cpu())), "the forward-only output differs"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(T.VGG_CASES))
def test_vgg_trunk_training_graph_matches_float64_reference_bit_for_bit(name, train_bf16, monkeypatch):
    """_vgg_raw under train precision 'bf16' on frozen weights: the four taps and the input gradient for upstream
    gradients at the taps equal the reference; neither weight nor bias gradient kernel runs."""
    from tecogan_b200 import kernels as K
    from tecogan_b200.lib.Teco import _vgg_raw
    calls = []
    for fn in ("conv3x3_wgrad_tc", "bias_grad"):
        orig = getattr(K, fn)
        monkeypatch.setattr(K, fn, lambda *a, _f=orig, _n=fn, **k: (calls.append(_n), _f(*a, **k))[1])
    n, h, w = T.VGG_CASES[name]
    p, x = T.vgg_operands(T.vgg_seed(name), n, h, w)
    train_bf16(p, trainable=False)
    K.tc_cache_clear()
    xd = x.cuda().float().requires_grad_()
    out = _vgg_raw(xd)
    R = T.TrainRounding(check=True)
    xl = x.cuda().requires_grad_()
    ref = T.vgg_train_ref({k: v.cuda() for k, v in p.items()}, xl, R)
    dys = [T.grad_grid(T.vgg_seed(name) + i, ref[k].shape).cuda() for i, k in enumerate(O.VGG_TAPS)]
    (dx,) = torch.autograd.grad([out[k] for k in O.VGG_TAPS], [xd], [d.float() for d in dys])
    torch.cuda.synchronize()
    (rdx,) = torch.autograd.grad([ref[k] for k in O.VGG_TAPS], [xl], dys)
    for k in O.VGG_TAPS:
        _check_f32(out[k].detach().cpu(), ref[k].detach().cpu(), "%s %s" % (name, k))
    _check_f32(dx.cpu(), rdx.cpu(), name + " d/d input")
    assert not calls, calls


@pytest.mark.gpu
@pytest.mark.parametrize("signed", [False, True], ids=["nonneg", "signed"])
@pytest.mark.parametrize("name", list(T.FNET_CASES))
def test_fnet_training_forward_within_the_tanh_bound(name, signed, train_bf16):
    """fnet with gradients enabled (the training kernels), both operand sets: the flow lies within REL_BOUND of the
    reference's."""
    from tecogan_b200 import kernels as K, variables as V
    from tecogan_b200.lib.frvsr import fnet
    n, h, w = T.FNET_CASES[name]
    p, x = E.fnet_operands(T.fnet_seed(name, signed), n, h, w, signed)
    train_bf16(p)
    K.tc_cache_clear()
    with V.variable_scope("fnet"):
        flow = fnet(x.cuda().float().requires_grad_(), reuse=False)
    torch.cuda.synchronize()
    ref = T.fnet_train_ref({k: v.cuda() for k, v in p.items()}, x.cuda(), T.TrainRounding(check=True)).cpu()
    _check_f32(flow.detach().cpu(), ref, "%s %s flow" % (name, "signed" if signed else "nonneg"),
               bound=REL_BOUND * ref.abs())


def _check_fnet_backward(load, name):
    """fnet on the device and its gradients w.r.t. the frame pairs and every parameter for the case's sparse upstream
    flow gradient; the reference's, its head's backward started from the device's flow.  The flow lies within the tanh
    bound; the input gradient (the 6-channel first conv's dx) and every weight gradient are bit for bit; every bias
    gradient is bit for bit where its interval is one point and within it elsewhere (the head, and channels on
    LeakyReLU's negative branch)."""
    from tecogan_b200 import kernels as K, variables as V
    from tecogan_b200.lib.frvsr import fnet
    c = T.FNET_BWD_CASES[name]
    p, x = E.fnet_operands(c.seed, c.n, c.h, c.w, True)
    dy = T.sparse_grad(c.seed, (c.n, c.h, c.w, 2), c.density)
    st = load(p)
    K.tc_cache_clear()
    names = list(p)
    xd = x.cuda().float().requires_grad_()
    with V.variable_scope("fnet"):
        flow = fnet(xd, reuse=False)
    grads = torch.autograd.grad(flow, [xd] + [st[k] for k in names], dy.cuda().float())
    torch.cuda.synchronize()
    R = T.TrainRounding(check=True, flow=flow.detach().double())
    pl = {k: v.cuda().requires_grad_() for k, v in p.items()}
    xl = x.cuda().requires_grad_()
    ref = T.fnet_train_ref(pl, xl, R)
    rgrads = torch.autograd.grad(ref, [xl] + [pl[k] for k in names], dy.cuda())
    ref = ref.detach().cpu()
    _check_f32(flow.detach().cpu(), ref, name + " flow", bound=REL_BOUND * ref.abs())
    _check_f32(grads[0].cpu(), rgrads[0].cpu(), name + " d/d fnet_input")
    _check_grads(names, grads[1:], rgrads[1:], R, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(T.FNET_BWD_CASES))
def test_fnet_training_graph_matches_float64_reference_bit_for_bit(name, train_bf16):
    _check_fnet_backward(train_bf16, name)


@pytest.mark.gpu
def test_fnet_deterministic_mode_gives_the_same_bits(train_bf16):
    """config.set_deterministic(True) on FNet: the fixed-order weight and bias gradient kernels and the resize
    gradient's _det kernel give the reference's bits (and the bias sums stay within their intervals)."""
    from tecogan_b200 import config
    config.set_deterministic(True)
    _check_fnet_backward(train_bf16, "2x32x32")
