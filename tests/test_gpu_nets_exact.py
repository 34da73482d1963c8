"""GeneratorPlan and FNetPlan (tecogan_b200/tc_nets.py) end to end against the float64 reference of tests/nets_exact.py,
which walks the oracle's layers and rounds where the device rounds.  On the operands built there every accumulation is
exact (a host guard checks each conv and resize before anything is compared), so every bf16 buffer the plans expose --
the packed generator input, the trunk output and the last conv_1 output, both transposed-conv outputs, each FNet level's
conv outputs and pooled / resized map, the head's first conv -- must equal the reference bit for bit, channels past the
layer's width must be zero, the generator's fp32 output must equal it exactly and the flow (tanh * 24) must lie within
the bound of test_gpu_conv_exact.py.  This pins the plans' wiring: each layer's packed weights, bias, activation, residual
buffer, input channel order, live K-steps, fused pool and level path, which the plans' routes share and the oracle
tolerances can miss.  The API entries generator_F / fnet under bf16 precision add the fp32 -> bf16 slice copies, the
channel offsets of the packed input and the bicubic's read of the LR channels at a 51-channel pitch."""
import types

import pytest
import torch

from oracle import teco_oracle as O
from tests import nets_exact as E
from tests.test_gpu_conv_exact import REL_BOUND, _bits, _check_f32

bf16 = torch.bfloat16


@pytest.fixture
def fresh_store():
    """Loads operands into a new default VariableStore; the previous store and precision come back afterwards."""
    from tecogan_b200 import config, variables as V
    prec, store = config.precision(), V.default_store()

    def load(p):
        st = V.set_default_store(V.VariableStore())
        st.load(p)
        return st
    yield load
    config.set_precision(prec)
    V.set_default_store(store)


def _cuda(p):
    return {k: v.cuda() for k, v in p.items()}


def _check_bf16(got, ref, what):
    """got: bf16 device tensor of C >= ref's channels; its first channels equal bf16(ref) bit for bit, the rest are +0."""
    c = ref.shape[-1]
    g = _bits(got.cpu())
    want = _bits(ref.cpu().float().to(bf16))
    bad = g[..., :c] != want
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: %d / %d elements differ, first at %s: got %r, expected %r" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(ref[i])))
    assert bool((g[..., c:] == 0).all()), what + ": a channel past the layer's width is not zero"


def _check_generator(plan, ref, out, what):
    packed = torch.cat([ref["x_in"][..., 3:51], ref["x_in"][..., 0:3]], dim=-1)    # [0,48) space-to-depth, [48,51) LR
    _check_bf16(plan.x_in, packed, what + " x_in")
    for k in ("a", "b", "u1", "u2"):
        _check_bf16(getattr(plan, k), ref[k], "%s %s" % (what, k))
    _check_f32(out.cpu(), ref["out"].cpu(), what + " out")


def _check_fnet(plan, ref, flow, what):
    _check_bf16(plan.x_in, ref["x_in"], what + " x_in")
    for i, ((t1, t2, t3), (r1, r2, r3)) in enumerate(zip(plan.bufs, ref["levels"])):
        name = "%s %s" % (what, O.FNET_LAYERS[i][0])
        _check_bf16(t1, r1, name + " conv_1")
        if not plan.fused_pool[i]:                     # a fused level does not write its conv_2 output
            _check_bf16(t2, r2, name + " conv_2")
        _check_bf16(t3, r3, name + (" pooled" if i < 3 else " resized"))
    _check_bf16(plan.o1, ref["o1"], what + " output_stage/conv1")
    f = ref["flow"].cpu()
    _check_f32(flow.cpu(), f, what + " flow", bound=REL_BOUND * f.abs())


def _generator_plan(B, h, w, N):
    from tecogan_b200 import tc_nets, variables as V
    with V.variable_scope("generator"), V.variable_scope("generator_unit") as gs:
        return tc_nets.GeneratorPlan(gs, B, h, w, N, "cuda")


def _fnet_plan(n, h, w):
    from tecogan_b200 import tc_nets, variables as V
    with V.variable_scope("fnet"), V.variable_scope("autoencode_unit") as fs:
        return tc_nets.FNetPlan(fs, n, h, w, "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(E.GEN_CASES))
def test_generator_plan_matches_float64_reference_bit_for_bit(name, fresh_store):
    """GeneratorPlan.run on one case of E.GEN_CASES, its trunk on the route the case names (the one launch at one round
    of clusters and at clusters running three clips, or per layer), with the device's own bicubic residual."""
    from tecogan_b200 import kernels as K
    c = E.GEN_CASES[name]
    G = K.conv3x3_lin_clusters()
    B = E.gen_batch(c, G)
    p, x = E.generator_operands(E.gen_seed(name), B, c.h, c.w, c.N)
    fresh_store(p)
    plan = _generator_plan(B, c.h, c.w, c.N)
    if c.lin is not None:
        assert not c.lin or hasattr(plan, "trunk_plan"), name + ": the one-launch trunk does not take the shape"
        plan.lin = c.lin
    assert plan.lin == E.gen_lin(c, G)
    xd = x.cuda()
    plan.x_in.zero_()
    plan.x_in[..., 0:48] = xd[..., 3:51].to(bf16)
    plan.x_in[..., 48:51] = xd[..., 0:3].to(bf16)
    out = plan.run(xd[..., 0:3].float().contiguous())
    torch.cuda.synchronize()
    ref = E.generator_ref(_cuda(p), xd, c.N, E.Rounding(check=E.nets_check), bic=plan.bic.double())
    _check_generator(plan, ref, out, name)


@pytest.mark.gpu
@pytest.mark.parametrize("signed", [False, True], ids=["nonneg", "signed"])
@pytest.mark.parametrize("shape", list(E.FNET_SHAPES))
def test_fnet_plan_matches_float64_reference_bit_for_bit(shape, signed, fresh_store):
    """FNetPlan.run on one shape of E.FNET_SHAPES under one operand set; the plan's level paths and fused pools are the
    ones nets_exact restates (and the case table is checked against on the host)."""
    n, h, w = E.FNET_SHAPES[shape]
    p, x = E.fnet_operands(E.fnet_seed(shape, signed), n, h, w, signed)
    fresh_store(p)
    plan = _fnet_plan(n, h, w)
    assert plan.small == E.fnet_small(h, w) and plan.fused_pool == E.fnet_fused(h, w)
    xd = x.cuda()
    plan.x_in[..., :6] = xd.to(bf16)
    flow = plan.run()
    torch.cuda.synchronize()
    ref = E.fnet_ref(_cuda(p), xd, E.Rounding(check=E.nets_check))
    _check_fnet(plan, ref, flow, "%s %s" % (shape, "signed" if signed else "nonneg"))


def _only_plan(kind, store):
    from tecogan_b200 import tc_nets
    plans = [pl for k, pl in tc_nets._plans.items() if k[0] == kind and k[1] == store.uid]
    assert len(plans) == 1, len(plans)
    return plans[0]


@pytest.mark.gpu
def test_generator_F_api_entry_matches_float64_reference_bit_for_bit(fresh_store):
    """generator_F under bf16 precision on fp32 [B, h, w, 51] inputs: the packed input holds the space-to-depth channels
    at 0 and the LR channels at 48, the bicubic residual equals teco_bicubic4_f32 on the LR channels alone, and every
    buffer and the returned output equal the reference."""
    from tecogan_b200 import config, variables as V
    from tecogan_b200._ffi import call, ptr, stream_ptr
    from tecogan_b200.lib.frvsr import generator_F
    B, h, w, N = 2, 20, 28, 4
    p, x = E.generator_operands(3000, B, h, w, N)
    st = fresh_store(p)
    config.set_precision("bf16")
    xd = x.cuda()
    with torch.no_grad(), V.variable_scope("generator"):
        out = generator_F(xd.float(), 3, reuse=False, FLAGS=types.SimpleNamespace(num_resblock=N))
    plan = _only_plan("gen", st)
    lr = xd[..., 0:3].float().contiguous()
    bic = torch.empty(B, 4 * h, 4 * w, 3, device="cuda")
    call("teco_bicubic4_f32", ptr(lr, torch.float32), ptr(bic, torch.float32), B, h, w, 3, 3, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(_bits(plan.bic), _bits(bic)), "the bicubic residual did not read the LR channels"
    ref = E.generator_ref(_cuda(p), xd, N, E.Rounding(check=E.nets_check), bic=bic.double())
    _check_generator(plan, ref, out, "generator_F")


@pytest.mark.gpu
def test_fnet_api_entry_matches_float64_reference_bit_for_bit(fresh_store):
    """fnet under bf16 precision on fp32 [n, h, w, 6] frame pairs (signed operands): the packed input and every buffer
    and the returned flow equal the reference."""
    from tecogan_b200 import config, variables as V
    from tecogan_b200.lib.frvsr import fnet
    n, h, w = 3, 24, 40
    p, x = E.fnet_operands(3001, n, h, w, signed=True)
    st = fresh_store(p)
    config.set_precision("bf16")
    xd = x.cuda()
    with torch.no_grad(), V.variable_scope("fnet"):
        flow = fnet(xd.float(), reuse=False)
    torch.cuda.synchronize()
    ref = E.fnet_ref(_cuda(p), xd, E.Rounding(check=E.nets_check))
    _check_fnet(_only_plan("fnet", st), ref, flow, "fnet")
