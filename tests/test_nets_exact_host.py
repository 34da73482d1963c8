"""Host checks of tests/nets_exact.py, the float64 restatement of the bf16 generator and FNet plans that
tests/test_gpu_nets_exact.py compares them with: its structure against the oracle, its operands against their guards,
and its case tables against the plan features they must reach."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests import nets_exact as E

HOST_IMAGES = 2          # images of a large batch the host guards (image i does not depend on the batch size)


def test_reference_without_rounding_is_the_oracle_bit_for_bit():
    """Rounding off and continuous float64 parameters: the reference's generator output and flow equal O.generator_F
    and O.fnet bit for bit, so its layer order, parameter names, activations, pools and resizes are the oracle's."""
    N = 3
    pg = O.damp_generator(O.init_generator(seed=3, num_resblock=N, bias_std=0.05, dtype=torch.float64))
    pf = O.init_fnet(seed=4, bias_std=0.05, dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 10, 12, 51, generator=g, dtype=torch.float64)
    got = E.generator_ref(pg, x, N, E.Rounding(on=False))["out"]
    assert torch.equal(got, O.generator_F(pg, x, N))
    f = torch.rand(2, 24, 40, 6, generator=g, dtype=torch.float64)
    got = E.fnet_ref(pf, f, E.Rounding(on=False))
    want = O.fnet(pf, f)
    assert torch.equal(got["flow"], want)
    assert got["flow"].abs().max() > 0.1
    # the restatement is not vacuous: rounding on moves the result
    assert not torch.equal(E.fnet_ref(pf, f, E.Rounding())["flow"], want)


def _gen_case(name, images=HOST_IMAGES):
    c = E.GEN_CASES[name]
    B = min(E.gen_batch(c, E.MAX_CLUSTERS), images)
    return c, E.generator_operands(E.gen_seed(name), B, c.h, c.w, c.N)


def _fnet_case(shape, signed, images=HOST_IMAGES):
    n, h, w = E.FNET_SHAPES[shape]
    return E.fnet_operands(E.fnet_seed(shape, signed), min(n, images), h, w, signed)


@pytest.mark.parametrize("name", list(E.GEN_CASES))
def test_generator_operands_pass_the_guard_at_every_layer(name):
    c, (p, x) = _gen_case(name)
    seen = []
    E.generator_ref(p, x, c.N, E.Rounding(check=lambda kind, what, *a: (seen.append(what), E.nets_check(kind, what, *a))),
                    bic=torch.zeros(x.shape[0], 4 * c.h, 4 * c.w, 3, dtype=torch.float64))
    assert len(seen) == 2 * c.N + 4


@pytest.mark.parametrize("signed", [False, True], ids=["nonneg", "signed"])
@pytest.mark.parametrize("shape", list(E.FNET_SHAPES))
def test_fnet_operands_pass_the_guard_at_every_layer(shape, signed):
    """Every conv and resize of both operand sets is in its exact regime; the signed set runs LeakyReLU's negative branch
    on every layer and the non-negative set never does; no level is constant."""
    p, x = _fnet_case(shape, signed)
    seen = []
    ref = E.fnet_ref(p, x, E.Rounding(check=lambda kind, what, *a: (seen.append(what), E.nets_check(kind, what, *a))))
    assert len(seen) == 14 + 3
    for i, (t1, t2, t3) in enumerate(ref["levels"]):
        for t in (t1, t2):
            assert bool((t < 0).any()) == signed, (i, signed)
            assert t.unique().numel() > 8, i
    assert ref["flow"].abs().max() < 23.9 and ref["flow"].std() > 0.1    # tanh not saturated: the head is informative


def test_guards_fail_operands_off_their_grid():
    """Moving one operand off its grid, or past what fp32 holds, makes the guard of that layer fail."""
    c, (p, x) = _gen_case("36x45", images=1)
    p = dict(p)
    w = p[E.GEN + "input_stage/conv/Conv/weights"].clone()
    w[1, 1, 5, 7] += 2.0 ** -20
    p[E.GEN + "input_stage/conv/Conv/weights"] = w
    with pytest.raises(AssertionError, match="input_stage"):
        E.generator_ref(p, x, c.N, E.Rounding(check=E.nets_check))

    p, x = _fnet_case("3x40x56", signed=False, images=1)
    name = E.FNET + "encoder_2/conv_2/Conv/biases"
    p[name] = p[name].clone()
    p[name][3] += 2.0 ** -30
    with pytest.raises(AssertionError, match="encoder_2/conv_2"):
        E.fnet_ref(p, x, E.Rounding(check=E.nets_check))

    p, x = _fnet_case("3x40x56", signed=True, images=1)
    for bad in ("two weights", "not a power of two"):
        q = dict(p)
        name = E.FNET + "decoder_1/conv_1/Conv/weights"
        w = q[name].clone()
        k = int(np.flatnonzero(w[..., 0].flatten().numpy())[0])
        if bad == "two weights":
            w.view(-1, w.shape[-1])[(k + 1) % (w.numel() // w.shape[-1]), 0] = 2.0 ** -20
        else:
            w.view(-1, w.shape[-1])[k, 0] *= 1.5
        q[name] = w
        with pytest.raises(AssertionError, match="decoder_1/conv_1"):
            E.fnet_ref(q, x, E.Rounding(check=E.nets_check))

    t = torch.full((1, 2, 2, 8), 1.0, dtype=torch.float64)
    t[0, 0, 1, 3] = 2.0 ** -30                 # 1 - 2^-30 is not an fp32 value
    with pytest.raises(AssertionError, match="resize"):
        E.resize_check("resize", t)
    E.resize_check("resize", torch.full((1, 2, 2, 8), 1.0, dtype=torch.float64))


def test_case_tables_reach_every_required_plan_feature():
    """Host restatement of the plans' choices: the generator cases run the trunk as one launch (one round, and clusters
    running three clips) and layer by layer, N = 16 and 10, ragged LR and HR tiles and a 180-wide output; the FNet shapes
    put every level on conv3x3_tc and on the im2col kernel, fuse the pool of encoder_1 / encoder_2 and pool every encoder
    separately (encoder_3 after conv3x3_tc), run odd level sizes, a 1 x 1 bottom level and more tiles than the grid."""
    gen = set().union(*(E.gen_features(c) for c in E.GEN_CASES.values()))
    assert E.GEN_REQUIRED <= gen, sorted(E.GEN_REQUIRED - gen)
    fn = set().union(*(E.fnet_features(*s) for s in E.FNET_SHAPES.values()))
    assert E.FNET_REQUIRED <= fn, sorted(E.FNET_REQUIRED - fn)
    assert E.fnet_level_sizes(40, 56)[3] == (5, 7) and E.fnet_level_sizes(8, 8)[3] == (1, 1)
    assert not E.gen_lin(E.GEN_CASES["B=2G+1 lin"]._replace(lin=None), E.MAX_CLUSTERS)   # forced: the plan would not
