"""The generator trunk as one launch with its activations in shared memory (teco_conv3x3_lin_tc on 32x32 images,
conv3x3_trunk_cluster_kernel): which plans take it, and that it computes byte for byte what one conv3x3_ws_kernel<0>
launch per layer computes -- on continuous operands, against a float64 reference in the exact regime, and end to end in
the clip engine."""
import numpy as np
import pytest
import torch

from oracle import teco_oracle as O

NONE, RELU, LRELU, TANH24 = 0, 1, 2, 3
TRUNK = [(0, 1, -1, RELU)] + [(1, 2, -1, RELU), (2, 1, 1, NONE)] * 16      # input conv + 16 residual blocks


def test_dispatch_takes_exactly_the_trunk_shaped_plans_on_32x32():
    from tecogan_b200 import kernels as K
    ok = lambda plan, n=4, h=32, w=32: K.conv3x3_lin_in_smem(n, h, w, plan)
    assert ok(TRUNK) and ok(TRUNK, n=1) and ok(TRUNK, n=264)
    assert ok([(0, 1, -1, NONE)])                                             # one layer
    assert ok([(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, 1, NONE)])         # one residual block
    assert ok([(0, 1, -1, RELU), (1, 2, -1, LRELU)])                         # the last output in buffer 2
    assert ok([(0, 1, -1, RELU), (1, 2, -1, RELU), (2, 1, -1, RELU), (1, 2, 2, NONE)])   # in place on b, written before
    assert not ok(TRUNK, h=28) and not ok(TRUNK, h=64) and not ok(TRUNK, w=40)
    assert not ok([(0, 1, 2, LRELU)])                                         # residual on layer 0
    assert not ok([(0, 2, -1, RELU)])                                         # layer 0 must write buffer 1
    assert not ok([(0, 1, -1, RELU), (1, 2, 2, NONE)])                        # buffer 2 not yet written by the chain
    assert not ok([(0, 1, -1, RELU), (0, 2, -1, RELU)])                       # a later layer reading x_in
    assert not ok([(0, 1, -1, RELU), (1, 2, 1, NONE)])                        # residual other than the output
    assert not ok([(0, 1, -1, RELU), (1, 2, -1, RELU), (1, 2, -1, RELU)])     # not the previous layer's output
    assert not ok([(0, 1, -1, TANH24)])
    assert ok(TRUNK + [(1, 2, -1, RELU), (2, 1, -1, RELU)] * 3 + [(1, 2, -1, RELU)])   # 40 layers
    assert not ok(TRUNK + [(1, 2, -1, RELU), (2, 1, -1, RELU)] * 4)          # 41
    assert not ok(TRUNK, n=0)
    from tecogan_b200.tc_nets import LIN_TRUNK_MIN_FILL
    assert 0.0 < LIN_TRUNK_MIN_FILL <= 1.0


def _trunk_operands(B, seed):
    from tecogan_b200 import kernels as K
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 32, 32, 64, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    ws = [((torch.rand(3, 3, 64, 64, generator=g) * 2 - 1) * (3.0 / 576) ** 0.5).cuda() for _ in TRUNK]
    bs = [((torch.rand(64, generator=g) - 0.5) * 0.2).cuda() for _ in TRUNK]
    return x, [K.packed_weight(w, 64, 64) for w in ws], bs


@pytest.mark.gpu
def test_trunk_matches_per_layer_launches_byte_for_byte():
    """33 layers on continuous operands at 1, 2, G + 1 (one clip more than one round of clusters) and 264 clips: buffers
    a and b equal those of 33 teco_conv3x3_tc launches bit for bit, and the guard image after the last clip is untouched."""
    from tecogan_b200 import kernels as K
    from tecogan_b200._ffi import lib
    G = lib().teco_conv3x3_lin_clusters()
    assert G > 0
    sent = -1.0e30
    for B in sorted({1, 2, G + 1, 264}):
        assert K.conv3x3_lin_in_smem(B, 32, 32, TRUNK)
        x, wpk, bs = _trunk_operands(B, seed=B)
        wall, ball = torch.cat(wpk).contiguous(), torch.cat(bs).contiguous()
        a = torch.full((B + 1, 32, 32, 64), sent, dtype=torch.bfloat16, device="cuda")
        b = torch.full_like(a, sent)
        K.conv3x3_lin_chain(x, a[:B], b[:B], wall, ball, TRUNK)
        ref = {0: x, 1: torch.zeros_like(x), 2: torch.zeros_like(x)}
        for l, (i, o, r, act) in enumerate(TRUNK):
            K.conv3x3_tc(ref[i], wpk[l], bs[l], ref[o], cout=64, act=act, res=ref[r] if r >= 0 else None)
        torch.cuda.synchronize()
        for name, got, exp in (("a", a, ref[1]), ("b", b, ref[2])):
            bits = got.view(torch.int16)
            assert torch.equal(bits[:B], exp.view(torch.int16)), (B, name, int((bits[:B] != exp.view(torch.int16)).sum()))
            assert bool((bits[B] == torch.tensor(sent, dtype=torch.bfloat16).view(torch.int16).cuda()).all()), (B, name)


@pytest.mark.gpu
def test_trunk_matches_float64_reference_bit_for_bit():
    """The full 33-layer plan at H = 32 in the exact regime of test_gpu_conv_exact.py: layer 0 on x = k/16 and weights
    m/128, later layers on sparse weights in {-1, 0, 1} (about one non-zero per output), so every layer's sums are exact
    in fp32 and each output is the bf16 rounding of the float64 value; the guard checks that per layer."""
    from tecogan_b200 import kernels as K
    from tests.test_gpu_conv_exact import (SENT_BF16, _assert_exact_regime, _bf16_grid, _check_bf16, _check_guard_image,
                                           _exact_candidates, _grid, _is_f32, _midpoints)
    n, plan = 3, TRUNK
    rng = np.random.RandomState(400)
    x = _grid(rng, (n, 32, 32, 64), 2.0 ** -4, 16)
    ext = _bf16_grid(rng, (n, 32, 32, 64))
    layers = [(_grid(rng, (3, 3, 64, 64), 2.0 ** -7, 16), _grid(rng, (64,), 2.0 ** -11, 2048))]
    for _ in range(1, len(plan)):
        sparse = rng.rand(3, 3, 64, 64) < 1.0 / 576
        layers.append((torch.from_numpy(sparse * rng.choice([-1.0, 1.0], size=sparse.shape) + 0.0),
                       _grid(rng, (64,), 2.0 ** -11, 256)))
    bufs = {0: x, 1: torch.zeros_like(x), 2: ext}
    ties = 0
    for l, ((wt, b), (i, o, ri, act)) in enumerate(zip(layers, plan)):
        z = O.conv2d(bufs[i], wt) + b
        r = bufs[ri] if ri >= 0 else None
        s_terms = O.conv2d(bufs[i].abs(), wt.abs()) + b.abs() + (r.abs() if r is not None else 0.0)
        _assert_exact_regime("trunk layer %d" % l, bufs[i], wt, s_terms, b, *([r] if r is not None else []))
        cands = _exact_candidates(act, z, r)
        assert all(_is_f32(v) for v in cands), l
        ties += _midpoints(cands[0])
        bufs[o] = cands[0].float().to(torch.bfloat16).double()
    assert ties > 0

    def dev_buf(v):
        t = torch.full((n + 1, 32, 32, 64), SENT_BF16, dtype=torch.bfloat16, device="cuda")
        t[:n] = v.to(torch.bfloat16).cuda()
        return t
    a, bb = dev_buf(torch.zeros_like(x)), dev_buf(ext)
    wall = torch.cat([K.packed_weight(wt.float().cuda(), 64, 64) for wt, _ in layers]).contiguous()
    ball = torch.cat([b.float().cuda() for _, b in layers]).contiguous()
    assert K.conv3x3_lin_in_smem(n, 32, 32, plan)
    K.conv3x3_lin_chain(x.to(torch.bfloat16).cuda(), a[:n], bb[:n], wall, ball, plan)
    torch.cuda.synchronize()
    for idx, t in ((1, a.cpu()), (2, bb.cpu())):
        _check_guard_image(t, SENT_BF16, "trunk buffer %d" % idx)
        _check_bf16(t[:-1], [bufs[idx]], "trunk buffer %d" % idx)


@pytest.mark.gpu
def test_clip_engine_takes_the_one_launch_trunk_from_the_batch_and_matches_per_layer_frames():
    """A batch of G clips (one full round of clusters) runs the one-launch trunk and G + 1 (a second round almost empty)
    and 8 the per-layer launches; the frames of the former are byte-identical to an engine of the same batch put onto
    the per-layer launches."""
    from tecogan_b200 import config
    from tecogan_b200.engine import ClipEngine
    from tests.test_gpu_models import _fresh_store, _smooth_clips
    from tecogan_b200 import kernels as K
    T, N, B = 10, 16, K.conv3x3_lin_clusters()
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=N)), O.init_fnet(seed=4321)
    clips = _smooth_clips(T, B, 32, 32, seed=5)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    assert not ClipEngine(32, 32, T, N, batch=8).gen.lin
    assert not ClipEngine(32, 32, T, N, batch=B + 1).gen.lin
    eng = ClipEngine(32, 32, T, N, batch=B)
    assert eng.gen.lin
    u8 = eng.run(clips.cuda()).clone()
    per_layer = ClipEngine(32, 32, T, N, batch=B)
    per_layer.gen.lin = False                    # before the first replay captures the graph
    u8_pl = per_layer.run(clips.cuda())
    assert torch.equal(u8, u8_pl), int((u8 != u8_pl).sum())
