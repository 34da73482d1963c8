"""GPU parity at network level: the mirror of the reference interface (tecogan_b200/lib) against the golden
vectors produced by the reference's own code (tests/golden) and against the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu


class Flags:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _fresh_store(params):
    from tecogan_b200 import variables as V
    st = V.set_default_store(V.VariableStore())
    st.load(params)
    return st


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _psnr(a, b):
    return O.psnr(a.detach().float().cpu().numpy(), b.detach().float().cpu().numpy())


@pytest.mark.parametrize("n", [3, 16])
def test_generator_fp32_matches_reference_golden(n):
    from tecogan_b200 import config
    from tecogan_b200.lib.frvsr import generator_F
    from tecogan_b200.variables import variable_scope
    g = _load("generator_n%d" % n)
    _fresh_store(O.init_generator(seed=int(g["seed"]), num_resblock=n, bias_std=float(g["bias_std"])))
    config.set_precision("fp32")
    with torch.no_grad(), variable_scope('generator'):
        out = generator_F(torch.from_numpy(g["inputs"]).cuda(), 3, reuse=False, FLAGS=Flags(num_resblock=n))
    err = (out.cpu() - torch.from_numpy(g["out"])).abs().max().item()
    assert err < 1e-4, err      # fp32 tolerance of SURVEY 8(c)


def test_fnet_fp32_matches_reference_golden():
    from tecogan_b200 import config
    from tecogan_b200.lib.frvsr import fnet
    from tecogan_b200.variables import variable_scope
    g = _load("fnet")
    _fresh_store(O.init_fnet(seed=int(g["seed"]), bias_std=float(g["bias_std"])))
    config.set_precision("fp32")
    with torch.no_grad(), variable_scope('fnet'):
        out = fnet(torch.from_numpy(g["inputs"]).cuda(), reuse=False)
    err = (out.cpu() - torch.from_numpy(g["out"])).abs().max().item()
    assert err < 2e-4, err      # flow is in [-24,24] LR pixels


@pytest.mark.parametrize("n,hw", [(3, (12, 10)), (16, (12, 10)), (16, (64, 48))])
def test_generator_bf16_tensor_core_close_to_oracle(n, hw):
    from tecogan_b200 import config
    from tecogan_b200.lib.frvsr import generator_F
    from tecogan_b200.variables import variable_scope
    p = O.damp_generator(O.init_generator(seed=12, num_resblock=n, bias_std=0.05))
    _fresh_store(p)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, hw[0], hw[1], 51, generator=g)
    ref = O.generator_F(p, x, n)
    config.set_precision("bf16")
    with torch.no_grad(), variable_scope('generator'):
        out = generator_F(x.cuda(), 3, reuse=False, FLAGS=Flags(num_resblock=n))
    ps = O.psnr(out.cpu().numpy(), ref.numpy(), peak=2.0)
    assert ps > 45.0, ps        # bf16 tolerance of SURVEY 8(c): PSNR(out, oracle) > 45 dB on the [-1,1] range


def test_fnet_bf16_tensor_core_close_to_oracle():
    from tecogan_b200 import config
    from tecogan_b200.lib.frvsr import fnet
    from tecogan_b200.variables import variable_scope
    p = O.init_fnet(seed=31, bias_std=0.05)
    _fresh_store(p)
    g = torch.Generator().manual_seed(6)
    x = torch.rand(2, 40, 36, 6, generator=g)
    ref = O.fnet(p, x)
    config.set_precision("bf16")
    with torch.no_grad(), variable_scope('fnet'):
        out = fnet(x.cuda(), reuse=False)
    assert tuple(out.shape) == tuple(ref.shape) == (2, 40, 32, 2)
    err = (out.cpu() - ref).abs()
    assert err.max().item() < 0.35 and err.mean().item() < 0.03, (err.max().item(), err.mean().item())


def _calendar_frames(crop=None, n=10):
    g = _load("calendar_lr")
    fr = g["crop32_u8"] if crop else g["full_u8"]
    fr = fr[:n].astype(np.float32) / 255.0
    order = O.warmup_order(len(fr))                     # lib/dataloader.py:42-44
    return [torch.from_numpy(fr[i]) for i in order]


def test_config1_calendar_32x32_fp32_engine_matches_oracle():
    """BASELINE config 1: runGan.py case-1 inference on calendar 32x32x10 (+5 warm-up), N=16, seed 1234."""
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=16)), O.init_fnet(seed=4321)
    frames = _calendar_frames(crop=True)
    ref = O.inference_sequence(pg, pf, frames, 16)
    _fresh_store({**pg, **pf})
    config.set_precision("fp32")
    eng = InferenceEngine(32, 32, 16)
    outs = eng.run_sequence([f.cuda() for f in frames])
    worst = max((o[0].cpu() - r).abs().max().item() for o, r in zip(outs, ref))
    assert worst < 1e-4, worst  # after 15 recurrent frames (SURVEY 8c tolerance, on [0,1] outputs)


def test_config1_calendar_32x32_bf16_engine_psnr_and_graph_equivalence():
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=16)), O.init_fnet(seed=4321)
    frames = _calendar_frames(crop=True)
    ref = O.inference_sequence(pg, pf, frames, 16)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    outs_g = InferenceEngine(32, 32, 16, use_graph=True).run_sequence([f.cuda() for f in frames])
    outs_e = InferenceEngine(32, 32, 16, use_graph=False).run_sequence([f.cuda() for f in frames])
    for a, b in zip(outs_g, outs_e):
        assert torch.equal(a, b)                        # CUDA-graph replay == eager launches, bit for bit
    ps = [O.psnr(o[0].cpu().numpy(), r.numpy()) for o, r in zip(outs_g[5:], ref[5:])]
    assert min(ps) > 40.0, ps
    # Y-PSNR parity with the reference's metric (metrics.py:37-70) against a common stand-in target
    tgt = [O.save_img_u8(O.bicubic_four(f.unsqueeze(0))[0]) for f in frames[5:]]
    d = [abs(O.psnr_y(t, O.save_img_u8(o[0].cpu())) - O.psnr_y(t, O.save_img_u8(r))) for t, o, r in zip(tgt, outs_g[5:], ref[5:])]
    assert max(d) < 0.05, d


def test_full_frame_144x180_streaming_exercises_symmetric_pad():
    """W=180 is not a multiple of 8: fnet sees 144x176 and the flow is SYMMETRIC-padded back (main.py:188-190,212)."""
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    pg, pf = O.init_generator(seed=7, num_resblock=4), O.init_fnet(seed=8)
    g = _load("calendar_lr")
    frames = [torch.from_numpy(g["full_u8"][i].astype(np.float32) / 255.0) for i in range(4)]
    ref = O.inference_sequence(pg, pf, frames, 4)
    _fresh_store({**pg, **pf})
    config.set_precision("fp32")
    outs = InferenceEngine(144, 180, 4).run_sequence([f.cuda() for f in frames])
    worst = max((o[0].cpu() - r).abs().max().item() for o, r in zip(outs, ref))
    assert worst < 1e-4, worst
    config.set_precision("bf16")
    outs = InferenceEngine(144, 180, 4).run_sequence([f.cuda() for f in frames])
    ps = [O.psnr(o[0].cpu().numpy(), r.numpy()) for o, r in zip(outs, ref)]
    assert min(ps) > 40.0, ps


def test_batched_clips_are_independent():
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    pg, pf = O.init_generator(seed=1, num_resblock=2), O.init_fnet(seed=2)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    g = torch.Generator().manual_seed(3)
    clips = torch.rand(2, 3, 32, 48, 3, generator=g).cuda()
    both = InferenceEngine(32, 48, 2, batch=2).run_sequence([clips[:, t] for t in range(3)])
    one = InferenceEngine(32, 48, 2, batch=1).run_sequence([clips[1, t] for t in range(3)])
    for a, b in zip(both, one):
        assert torch.equal(a[1], b[0])


def test_fnet_lookahead_is_bit_identical_to_the_serial_recurrence():
    """fnet(LR_i ++ LR_{i+1}) depends on no HR output (reference main.py:211), so the engine may run it concurrently with
    generator_F of frame i; every mix of look-ahead / serial steps must reproduce the serial outputs bit for bit."""
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    pg, pf = O.damp_generator(O.init_generator(seed=5, num_resblock=3)), O.init_fnet(seed=6)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    g = torch.Generator().manual_seed(11)
    frames = [torch.rand(32, 48, 3, generator=g).cuda() for _ in range(7)]
    serial = InferenceEngine(32, 48, 3).run_sequence(frames, lookahead=False)
    for use_graph in (True, False):
        ahead = InferenceEngine(32, 48, 3, use_graph=use_graph).run_sequence(frames, lookahead=True)
        for a, b in zip(ahead, serial):
            assert torch.equal(a, b)
    # mixed: serial, serial, look-ahead primed mid-clip, look-ahead, tail (no next frame), serial again
    eng = InferenceEngine(32, 48, 3)
    plan = [None, None, 3, 4, None, None, None]
    for i, fr in enumerate(frames):
        out = eng.step(fr, next_lr=frames[plan[i]] if plan[i] is not None else None)
        assert torch.equal(out, serial[i]), i
    with pytest.raises(ValueError):
        eng.step(frames[0], next_lr=torch.zeros(8, 8, 3, device="cuda"))


# ------------------------------------------------------------------------------------------------------------------
# Parity at the BENCHMARKED shapes (bench.py): the metric config (lock-step batch of 10-frame 32x32 clips through
# ClipEngine), configs[1] (128x128 streaming with the look-ahead graph) and one config-5 batch (256x256 x b2).
def _smooth_clips(T, B, h, w, seed):
    import bench
    return bench.synthetic_clips(T, B, h, w, seed)


def _y_psnr_delta(frames_lr, ours01, ref01):
    """|Y-PSNR(target, ours) - Y-PSNR(target, oracle)| with the reference's metric (metrics.py:37-70) against a common
    stand-in target (bicubic_four of the LR frame; no HR ground truth is shipped)."""
    d = []
    for lr, o, r in zip(frames_lr, ours01, ref01):
        tgt = O.save_img_u8(O.bicubic_four(lr.unsqueeze(0))[0])
        d.append(abs(O.psnr_y(tgt, O.save_img_u8(o)) - O.psnr_y(tgt, O.save_img_u8(r))))
    return max(d)


@pytest.mark.parametrize("B", [6, 12])
def test_metric_config_clip_engine_matches_oracle_and_streaming_engine(B):
    """bench.py headline path: B clips x 10 frames 32x32 in lock-step, one CUDA graph, fnet for all pairs first.
    B = 12 takes the one-launch trunk (teco_conv3x3_lin_tc, batches of >= 8 clips), B = 6 one launch per layer."""
    from tecogan_b200 import config
    from tecogan_b200.engine import ClipEngine, InferenceEngine
    T, N = 10, 16
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=N)), O.init_fnet(seed=4321)
    clips = _smooth_clips(T, B, 32, 32, seed=3)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    prev_lin = config.lin_trunk()
    config.set_lin_trunk(True)                           # the one-launch chain at B >= 8; the per-layer kernels below
    eng = ClipEngine(32, 32, T, N, batch=B)
    assert eng.gen.lin == (B >= 8)
    u8 = eng.run(clips.cuda()).clone()
    u8_again = eng.run(clips.cuda()).clone()            # second replay of the captured graph: same bits
    assert torch.equal(u8, u8_again)
    eager = ClipEngine(32, 32, T, N, batch=B, use_graph=False).run(clips.cuda())
    assert torch.equal(u8, eager)
    # same kernels as the streaming engine at the same batch -> bit-identical frames
    stream = InferenceEngine(32, 32, N, batch=B).run_sequence([clips[t].cuda() for t in range(T)], out="u8")
    for t in range(T):
        assert torch.equal(u8[t], stream[t]), t
    # against the oracle, clip by clip (fp32 CPU restatement of main.py:253-268)
    worst_psnr, worst_dy = 1e9, 0.0
    for b in range(3):
        ref = O.inference_sequence(pg, pf, [clips[t, b] for t in range(T)], N)
        ours = [u8[t, b].cpu().float() / 255.0 for t in range(T)]
        refq = [O.save_img_u8(r).astype(np.float32) / 255.0 for r in ref]
        worst_psnr = min(worst_psnr, min(O.psnr(o.numpy(), r) for o, r in zip(ours, refq)))
        worst_dy = max(worst_dy, _y_psnr_delta([clips[t, b] for t in range(T)], ours, ref))
    assert worst_psnr > 40.0, worst_psnr
    assert worst_dy < 0.05, worst_dy
    if B >= 8:
        # the per-layer kernels on the same clips: same arithmetic up to the fp32 summation order inside a layer
        config.set_lin_trunk(False)
        try:
            per_layer = ClipEngine(32, 32, T, N, batch=B)
            assert not per_layer.gen.lin
            u8_pl = per_layer.run(clips.cuda())
        finally:
            config.set_lin_trunk(prev_lin)
        diff = (u8.float() - u8_pl.float()).abs()
        assert diff.max().item() <= 3 and diff.mean().item() < 0.05, (diff.max().item(), diff.mean().item())
    config.set_lin_trunk(prev_lin)


def test_configs1_128x128_lookahead_graph_32_frames_matches_oracle():
    """bench.py configs[1] path: bf16, 128x128 -> 512x512, look-ahead CUDA graph on two streams, 32 recurrent frames."""
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    T, N = 32, 16
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=N)), O.init_fnet(seed=4321)
    clip = _smooth_clips(T, 1, 128, 128, seed=0)[:, 0]
    frames = [clip[t] for t in range(T)]
    ref = O.inference_sequence(pg, pf, frames, N)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    outs = InferenceEngine(128, 128, N, use_graph=True).run_sequence([f.cuda() for f in frames], lookahead=True)
    ours = [o[0].cpu() for o in outs]
    ps = [O.psnr(o.numpy(), r.numpy()) for o, r in zip(ours, ref)]
    assert min(ps) > 40.0, ps
    assert _y_psnr_delta(frames, ours, ref) < 0.05


def test_config5_256x256_batch2_matches_oracle():
    """bench.py config-5 path: ClipEngine at 256x256 -> 1024x1024, two clips, three frames (persistent multi-tile convs)."""
    from tecogan_b200 import config
    from tecogan_b200.engine import ClipEngine
    T, B, N = 3, 2, 16
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=N)), O.init_fnet(seed=4321)
    clips = _smooth_clips(T, B, 256, 256, seed=5)
    _fresh_store({**pg, **pf})
    config.set_precision("bf16")
    u8 = ClipEngine(256, 256, T, N, batch=B).run(clips.cuda())
    ref = O.inference_sequence(pg, pf, [clips[t, 1] for t in range(T)], N)
    ours = [u8[t, 1].cpu().float() / 255.0 for t in range(T)]
    refq = [O.save_img_u8(r).astype(np.float32) / 255.0 for r in ref]
    ps = [O.psnr(o.numpy(), r) for o, r in zip(ours, refq)]
    assert min(ps) > 40.0, ps
    assert _y_psnr_delta([clips[t, 1] for t in range(T)], ours, ref) < 0.05
