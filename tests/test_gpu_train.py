"""GPU parity of the training path (SURVEY 8a rows a11-a16): discriminator, VGG, the TecoGAN/FRVSR loss graph against
the goldens produced by the reference's own lib/Teco.py, and gradients / the train step against the oracle's autograd."""
import ast
import os

import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _fresh_store(params):
    from tecogan_b200 import variables as V
    st = V.set_default_store(V.VariableStore())
    st.load(params)
    return st


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32)).cuda()


class Flags:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def test_discriminator_matches_reference_golden():
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import discriminator_F
    from tecogan_b200.variables import variable_scope
    g = _load("discriminator")
    _fresh_store(O.init_discriminator(seed=int(g["seed"]), bias_std=float(g["bias_std"])))
    config.set_precision("fp32")
    with torch.no_grad(), variable_scope('tdiscriminator'):
        prob, layers = discriminator_F(_t(g["inputs"]), FLAGS=Flags())
    assert (prob.cpu() - torch.from_numpy(g["prob"])).abs().max().item() < 1e-4
    for i, l in enumerate(layers):
        assert (l.cpu() - torch.from_numpy(g["layer%d" % i])).abs().max().item() < 2e-4, i


def test_vgg19_slim_matches_reference_golden():
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import VGG19_slim
    g = _load("vgg")
    _fresh_store(O.init_vgg19(seed=int(g["seed"])))
    config.set_precision("fp32")
    with torch.no_grad():
        feats = VGG19_slim(_t(g["inputs"]), reuse=False, deep_list=O.VGG_TAPS)
    for i, k in enumerate(O.VGG_TAPS):
        assert (feats[k].cpu() - torch.from_numpy(g["tap%d" % i])).abs().max().item() < 1e-4, k


def _case(name):
    g = _load(name)
    ci = int(g["ci"])
    FL = O.TrainFlags(**ast.literal_eval(str(g["flags"])))
    P = {}
    P.update(O.init_generator(seed=61 + ci, num_resblock=FL.num_resblock, bias_std=0.05))
    P.update(O.init_fnet(seed=71 + ci, bias_std=0.05))
    if bool(g["gan"]):
        P.update(O.init_discriminator(seed=81 + ci, bias_std=0.05))
    if FL.vgg_scaling > 0:
        P.update(O.init_vgg19(seed=91 + ci))
    return g, FL, P


@pytest.mark.parametrize("name", ["teco_pp", "teco_nopp", "frvsr"])
def test_tecogan_loss_graph_matches_reference_golden(name):
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import _Graph
    g, FL, P = _case(name)
    _fresh_store(P)
    config.set_precision("fp32")
    with torch.no_grad():
        gr = _Graph(_t(g["r_inputs"]), _t(g["r_targets"]), FL, bool(g["gan"]), 0)
    assert gr.update_list_name == [str(s) for s in g["update_list_name"]]
    got = np.array([float(v) for v in gr.update_list])
    np.testing.assert_allclose(got, g["update_list"], rtol=3e-4, atol=2e-5)
    np.testing.assert_allclose(gr.s_gen_output.cpu().numpy(), g["gen_output"], rtol=1e-3, atol=3e-4)


@pytest.mark.parametrize("name", ["teco_pp", "frvsr", "teco_nopp"])
def test_train_step_gradients_and_control_flow_match_oracle(name):
    """One Network.train() step: every gradient tensor (flat bucket before Adam), the loss scalars, and the
    with-D / without-D decision against the oracle Trainer (torch-CPU autograd of the restated graph)."""
    from tecogan_b200.lib.Teco import FRVSR, TecoGAN
    g, FL, P = _case(name)
    gan = bool(g["gan"])
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    tr = O.Trainer(P, FL, gan)
    ref = tr.step(ri, rt)
    _fresh_store(P)
    net = TecoGAN(ri.cuda(), rt.cuda(), FL) if gan else FRVSR(ri.cuda(), rt.cuda(), FL)
    out = net.train()
    st = net.train
    np.testing.assert_allclose(np.array(out["update_list"]), np.array([float(v) for v in ref["update_list"]]), rtol=3e-4, atol=2e-5)
    assert out["with_d"] == ref["with_d"]
    o = 0
    worst = 0.0
    for k in st.names:
        n = st.store[k].numel()
        got = st.bucket[o:o + n].cpu()
        want = ref["grads"][k].reshape(-1)
        scale = max(want.abs().max().item(), 1e-6)
        err = (got - want).abs().max().item() / scale
        worst = max(worst, err)
        assert err < 5e-3, (k, err, scale)
        o += n
    # parameters moved by Adam: |delta| <= lr_t bound and same sign as the oracle wherever the gradient is not ~0
    k0 = st.opt_g.names[0]
    d_got = (st.store[k0].cpu() - P[k0])
    d_ref = (tr.p[k0] - P[k0])
    big = ref["grads"][k0].abs() > 1e-3 * ref["grads"][k0].abs().max()
    assert torch.allclose(d_got[big], d_ref[big], atol=2e-6), (d_got[big] - d_ref[big]).abs().max()


def test_second_step_uses_updated_weights_and_ema():
    from tecogan_b200.lib.Teco import TecoGAN
    g, FL, P = _case("teco_pp")
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    tr = O.Trainer(P, FL, True)
    tr.step(ri, rt)
    ref2 = tr.step(ri, rt)
    _fresh_store(P)
    net = TecoGAN(ri.cuda(), rt.cuda(), FL)
    net.train()
    out2 = net.train()
    np.testing.assert_allclose(np.array(out2["update_list"]), np.array([float(v) for v in ref2["update_list"]]), rtol=2e-3, atol=1e-4)
    assert abs(net.train.tb_ema - tr.tb_ema) < 1e-5
    assert net.global_step() == 2


def test_gauss_down_loader_matches_oracle():
    from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader
    FL = O.TrainFlags(batch_size=2, crop_size=8, RNN_N=2)
    hr = torch.rand(2, 2, 40, 40, 3, generator=torch.Generator().manual_seed(1))
    lr, tgt = frvsr_gpu_data_loader(hr.cuda(), FL)
    ref_lr = O.gauss_down_by4(hr.reshape(4, 40, 40, 3)).reshape(2, 2, 8, 8, 3)
    assert (lr.cpu() - ref_lr).abs().max().item() < 1e-5
    assert (tgt.cpu() - (hr[:, :, 4:36, 4:36] * 2 - 1)).abs().max().item() < 1e-6


def test_bf16_tensor_core_training_step_close_to_fp32_oracle():
    """--precision bf16 for training: 3x3 convs run forward + input-gradient on wgmma (bf16 operands, fp32 accumulate,
    fp32 master weights).  Losses within 2e-2 relative of the fp32 oracle, gradient direction preserved (cosine > 0.99)."""
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import FRVSR
    g, FL, P = _case("frvsr")
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    tr = O.Trainer(P, FL, False)
    ref = tr.step(ri, rt)
    _fresh_store(P)
    config.set_train_precision("bf16")
    try:
        net = FRVSR(ri.cuda(), rt.cuda(), FL)
        out = net.train()
    finally:
        config.set_train_precision("fp32")
    want = np.array([float(v) for v in ref["update_list"]])
    np.testing.assert_allclose(np.array(out["update_list"]), want, rtol=2e-2, atol=1e-4)
    st = net.train
    got = st.bucket[:st.opt_g.n + st.opt_f.n].cpu()
    refg = torch.cat([ref["grads"][k].reshape(-1) for k in st.opt_g.names + st.opt_f.names])
    cos = float((got * refg).sum() / (got.norm() * refg.norm()))
    assert cos > 0.99, cos


def test_bf16_tensor_core_tecogan_step_with_vgg_close_to_fp32_oracle():
    """Same for the full TecoGAN graph: VGG19 (frozen, up to 512 channels) also runs on wgmma in bf16 mode."""
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import TecoGAN
    g, FL, P = _case("teco_pp")
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    tr = O.Trainer(P, FL, True)
    ref = tr.step(ri, rt)
    _fresh_store(P)
    config.set_train_precision("bf16")
    try:
        net = TecoGAN(ri.cuda(), rt.cuda(), FL)
        out = net.train()
    finally:
        config.set_train_precision("fp32")
    want = np.array([float(v) for v in ref["update_list"]])
    np.testing.assert_allclose(np.array(out["update_list"]), want, rtol=4e-2, atol=2e-3)
    assert out["with_d"] == ref["with_d"]


@pytest.mark.parametrize("fmt", ["tf", "pt"])
def test_checkpoint_resume_restores_everything(tmp_path, fmt):
    """Saver semantics (reference main.py:307,346-349,418-421): save after two steps, restore weights + Adam moments +
    step counters + EMAs into a fresh process state -- bit-exact state -- and the third step lands where the uninterrupted
    run does (the weight-gradient kernels accumulate with atomics, so two runs of one step agree to rounding, not bits),
    through the TensorFlow V2 bundle written by tecogan_b200/tf_bundle.py as well as through the .pt file."""
    import main as M
    from tecogan_b200.lib.Teco import TecoGAN
    g, FL, P = _case("teco_nopp")
    ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
    st = _fresh_store(P)
    net = TecoGAN(ri, rt, FL)
    net.train()
    net.train()
    M.save_checkpoint(st, str(tmp_path), net.global_step(), net.train)
    saved_state = net.train.state_tensors()
    saved_w = {k: v.detach().cpu().clone() for k, v in st.items()}
    net.train()
    want = {k: v.detach().cpu().clone() for k, v in st.items()}
    want_ema, want_tb = list(net.train.loss_ema), net.train.tb_ema

    from tecogan_b200 import variables as V
    st2 = V.set_default_store(V.VariableStore())
    spec = str(tmp_path / "model-2") + ("" if fmt == "tf" else ".pt")
    M.load_checkpoint(st2, spec, FL.num_resblock, need_d=True, need_vgg=FL.vgg_scaling > 0)
    if FL.vgg_scaling > 0:            # the frozen VGG weights are part of neither scope list of the reference's restore
        st2.load({k: v for k, v in P.items() if k.startswith("vgg_19/")})
    net2 = TecoGAN(ri, rt, FL)
    missing = M.restore_train_state(net2.train, spec)
    assert missing == [] and net2.global_step() == 2 and net2.train.opt_g.t == 2
    restored = net2.train.state_tensors()
    assert set(restored) == set(saved_state)
    for k, v in saved_state.items():                       # moments, counters, EMAs: exactly what was saved
        assert torch.equal(restored[k], v), k
    for k, v in saved_w.items():
        if k in st2:
            assert torch.equal(st2[k].detach().cpu(), v), k
    net2.train()
    assert net2.global_step() == 3
    lr = FL.learning_rate
    for k in want:
        if k in st2 and not k.startswith("vgg_19/"):
            d = (st2[k].detach().cpu() - want[k]).abs()
            # a lost moment would move (nearly) every element by ~lr; two runs of the same step differ only where an
            # atomically accumulated gradient is itself rounding noise (near-zero gradients divided by sqrt(v) + eps)
            assert d.max().item() < 2.0 * lr and (d < 0.05 * lr).float().mean().item() > 0.97, (k, d.max().item())
    assert abs(net2.train.tb_ema - want_tb) < 1e-6
    np.testing.assert_allclose(np.array(net2.train.loss_ema), np.array(want_ema), rtol=1e-4, atol=1e-7)


def _config3_case():
    """BASELINE configs[2] shape: FRVSR (runGan.py case 4), B=4 clips x RNN_N=10 frames, 32x32 LR crops, N=10 blocks."""
    FL = O.TrainFlags.frvsr(batch_size=4, crop_size=32, RNN_N=10, num_resblock=10)
    P = {}
    P.update(O.damp_generator(O.init_generator(seed=161, num_resblock=10, bias_std=0.02)))
    P.update(O.init_fnet(seed=171, bias_std=0.02))
    g = torch.Generator().manual_seed(5)
    ri = torch.rand(4, 10, 32, 32, 3, generator=g)
    rt = torch.rand(4, 10, 128, 128, 3, generator=g) * 2 - 1
    return FL, P, ri, rt


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_config3_shape_train_step_matches_oracle(precision):
    """The benchmarked training shape (bench.py train.config3_frvsr): loss scalars and every gradient of one step against
    the oracle Trainer.  fp32: loss rtol 1e-3, per-tensor gradient error <= 1e-2 of the tensor's max (10 recurrent frames
    of BPTT, atomically accumulated weight gradients).  bf16 tensor-core convolutions: loss rtol 3e-2, gradient cosine
    > 0.98 per network."""
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import FRVSR
    FL, P, ri, rt = _config3_case()
    tr = O.Trainer(P, FL, False)
    ref = tr.step(ri, rt)
    _fresh_store(P)
    config.set_train_precision(precision)
    try:
        net = FRVSR(ri.cuda(), rt.cuda(), FL)
        out = net.train()
    finally:
        config.set_train_precision("fp32")
    want = np.array([float(v) for v in ref["update_list"]])
    st = net.train
    if precision == "fp32":
        np.testing.assert_allclose(np.array(out["update_list"]), want, rtol=1e-3, atol=2e-5)
        o = 0
        for k in st.names:
            n = st.store[k].numel()
            got, w = st.bucket[o:o + n].cpu(), ref["grads"][k].reshape(-1)
            err = (got - w).abs().max().item() / max(w.abs().max().item(), 1e-6)
            assert err < 1e-2, (k, err)
            o += n
    else:
        np.testing.assert_allclose(np.array(out["update_list"]), want, rtol=3e-2, atol=1e-4)
        o = 0
        for names in (st.opt_g.names, st.opt_f.names):
            n = sum(st.store[k].numel() for k in names)
            got = st.bucket[o:o + n].cpu()
            refg = torch.cat([ref["grads"][k].reshape(-1) for k in names])
            cos = float((got * refg).sum() / (got.norm() * refg.norm()))
            assert cos > 0.98, (names[0], cos)
            o += n
