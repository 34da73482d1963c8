"""GPU: training monitoring -- Network.train.evaluate (the training graph's forward on a validation batch, reference
main.py:299-304,391-402) against the goldens, the oracle and the training step itself; evaluation leaves training
untouched; and main.py --mode train --summary_dir end to end (event file, logfile.txt, validation block, test-sequence
frames, and, with --deterministic, the same checkpoint bit for bit as a run without monitoring).

The loss and BatchNorm reductions and the weight gradients accumulate with fp32 atomics, so two executions of the same
forward agree to rounding, not necessarily to the bit: values a run COMPUTES are compared at rounding tolerances, while
the state evaluate() must not WRITE is compared bit for bit."""
import ast
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def _case(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
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


def _net(g, FL, P):
    from tecogan_b200 import variables as V
    from tecogan_b200.lib.Teco import FRVSR, TecoGAN
    V.set_default_store(V.VariableStore()).load(P)
    ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
    return TecoGAN(ri, rt, FL) if bool(g["gan"]) else FRVSR(ri, rt, FL)


def _other_batch(g, seed=3):
    """A second batch of the golden's shape: LR in [0,1], targets in [-1,1]."""
    gen = torch.Generator().manual_seed(seed)
    ri = torch.rand(g["r_inputs"].shape, generator=gen)
    rt = torch.rand(g["r_targets"].shape, generator=gen) * 2 - 1
    return ri, rt


class _TrainPrecision:
    def __init__(self, p):
        self.p = p

    def __enter__(self):
        from tecogan_b200 import config
        config.set_train_precision(self.p)

    def __exit__(self, *a):
        from tecogan_b200 import config
        config.set_train_precision("fp32")


def _uplen(net):
    return len(net.update_list)


@pytest.mark.parametrize("name", ["teco_pp", "teco_nopp", "frvsr"])
def test_evaluate_matches_reference_golden_and_first_step(name):
    g, FL, P = _case(name)
    net = _net(g, FL, P)
    ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
    ev = net.train.evaluate(ri, rt)
    assert list(ev) == [str(s) for s in g["update_list_name"]] == net.update_list_name[:_uplen(net)]
    got = np.array(list(ev.values()))
    np.testing.assert_allclose(got, g["update_list"], rtol=3e-4, atol=2e-5)
    out = net.train()
    # same kernels on the same weights and batch: the two passes differ at most by the order of atomic fp32 additions
    np.testing.assert_allclose(got, np.array(out["update_list"]), rtol=1e-5, atol=1e-7)
    print("%s: evaluate vs first train() update_list, max |diff| %.3g, bit-identical %s"
          % (name, np.abs(got - np.array(out["update_list"])).max(), bool((got == np.array(out["update_list"])).all())))


def _snapshot(net):
    st = net.train
    t = {"static_in": st.static_in, "static_tg": st.static_tg, "bucket": st.bucket}
    for tag, opt in (("g", st.opt_g), ("f", st.opt_f), ("d", st.opt_d)):
        if opt is not None:
            t.update({tag + "_flat": opt.flat, tag + "_m": opt.m, tag + "_v": opt.v})
    t.update({"store/" + k: v for k, v in st.store.items()})
    t = {k: v.detach().clone() for k, v in t.items()}
    host = (st.global_step, list(st.loss_ema or []), st.tb_ema, st.counter1, st.counter2,
            [o.t for o in (st.opt_g, st.opt_f, st.opt_d) if o is not None], dict(st.last or {}).get("with_d"))
    return t, host


def _assert_same_snapshot(a, b):
    assert a[1] == b[1]
    assert set(a[0]) == set(b[0])
    for k in a[0]:
        assert torch.equal(a[0][k], b[0][k]), k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["teco_pp", "frvsr"])
def test_evaluate_does_not_perturb_training(name, precision):
    """P: train x3.  Q: train, evaluate(other batch), train, evaluate, train -- with the captured evaluation graph.
    Every buffer and counter of the trainer is bit-identical before and after each evaluate(); P and Q then agree on the
    integer state and the with-D decisions exactly and on weights / EMAs / losses to rounding -- in bf16 a last-bit
    difference of an atomic sum can move an activation by one bf16 step, so the tolerance there is bf16's."""
    g, FL, P = _case(name)
    ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
    vi, vt = (x.cuda() for x in _other_batch(g))
    with _TrainPrecision(precision):
        netp = _net(g, FL, P)
        outs_p = [dict(netp.train(ri, rt)) for _ in range(3)]
        snap_p = _snapshot(netp)
        netq = _net(g, FL, P)
        outs_q = [dict(netq.train(ri, rt))]
        for _ in range(2):
            before = _snapshot(netq)
            netq.train.evaluate(vi, vt)
            torch.cuda.synchronize()
            _assert_same_snapshot(before, _snapshot(netq))
            outs_q.append(dict(netq.train(ri, rt)))
        assert netq.train.eval_graph is not None and netq.train.graph is not None
        snap_q = _snapshot(netq)
    assert [o["with_d"] for o in outs_p] == [o["with_d"] for o in outs_q]
    hp, hq = snap_p[1], snap_q[1]
    assert hp[0] == hq[0] == 3 and hp[3:6] == hq[3:6]
    rtol, atol = (1e-5, 1e-7) if precision == "fp32" else (1e-2, 1e-5)
    np.testing.assert_allclose(hp[1], hq[1], rtol=rtol, atol=atol)
    assert abs(hp[2] - hq[2]) < 100 * atol
    np.testing.assert_allclose(outs_p[2]["update_list"], outs_q[2]["update_list"], rtol=10 * rtol, atol=atol)
    lr = FL.learning_rate
    for k in snap_p[0]:
        if k.startswith("store/") and not k.startswith("store/vgg_19/"):
            d = (snap_p[0][k] - snap_q[0][k]).abs()
            assert d.max().item() < 6.0 * lr, (k, d.max().item())
            if precision == "fp32":
                assert (d < 0.05 * lr).float().mean().item() > 0.97, (k, d.max().item())
        elif k.startswith("store/vgg_19/"):
            assert torch.equal(snap_p[0][k], snap_q[0][k]), k
    bit = all(torch.equal(snap_p[0][k], snap_q[0][k]) for k in snap_p[0] if k.startswith("store/"))
    print("%s %s: P and Q weights bit-identical %s" % (name, precision, bit))


def test_evaluate_after_two_steps_matches_oracle_fp32():
    """The evaluation graph is captured BEFORE training and replayed after two steps: it must see the updated weights."""
    g, FL, P = _case("teco_pp")
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    vi, vt = _other_batch(g)
    tr = O.Trainer(P, FL, True)
    tr.step(ri, rt)
    tr.step(ri, rt)
    ref = O.tecogan_forward(tr.p, vi, vt, FL, True, global_step=2)
    net = _net(g, FL, P)
    net.train.evaluate(vi.cuda(), vt.cuda())                 # capture on the initial weights
    net.train()
    net.train()
    ev = net.train.evaluate(vi.cuda(), vt.cuda())
    assert list(ev) == list(ref["update_list_name"])
    want = np.array([float(v) for v in ref["update_list"]])
    np.testing.assert_allclose(np.array(list(ev.values())), want, rtol=2e-3, atol=1e-4)


@pytest.mark.parametrize("name", ["teco_pp", "frvsr"])
def test_evaluate_bf16_replays_current_packed_weights(name):
    """bf16: the captured evaluation replayed after two steps equals an uncaptured no_grad forward of the training graph
    on the live weights (same kernels, weights packed now).  A replay of packings from capture time (initial weights)
    would show the whole two-step loss change instead of rounding."""
    from tecogan_b200 import config
    from tecogan_b200.lib.Teco import _Graph
    g, FL, P = _case(name)
    vi, vt = (x.cuda() for x in _other_batch(g))
    with _TrainPrecision("bf16"):
        net = _net(g, FL, P)
        first = np.array(list(net.train.evaluate(vi, vt).values()))
        net.train()
        net.train()
        ev = np.array(list(net.train.evaluate(vi, vt).values()))
        from tecogan_b200 import kernels as K
        K.tc_cache_clear()          # the cache now holds the training graph's packings, made before the last Adam update
        config.set_precision("fp32")
        try:
            with torch.no_grad(), config.train_forward():
                gr = _Graph(vi, vt, FL, bool(g["gan"]), net.train.global_step)
        finally:
            config.set_precision("bf16")
        want = np.array([float(v) for v in gr.update_list[:len(ev)]])
    np.testing.assert_allclose(ev, want, rtol=1e-5, atol=1e-7)
    moved = np.abs(want - first) > 1e-5 + 1e-5 * np.abs(want)
    assert moved.any(), "two steps did not move any loss: the stale-weight check has no power here"


# ------------------------------------------------------------------------------------------ main.py end to end
def _write_calendar(root):
    import cv2
    d = np.load(os.path.join(GOLDEN, "calendar_lr.npz"))
    full = d["full_u8"]
    p = os.path.join(root, "LR", "calendar")
    os.makedirs(p)
    for i in range(10):             # frames 0001..0010; the fixture holds 7 distinct 144x180 frames
        cv2.imwrite(os.path.join(p, "%04d.png" % (i + 1)), full[min(i, 6)][:, :, ::-1])


def _main(cwd, *args):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(ROOT, "main.py")] + list(args)
    # main.py sets CUDA_VISIBLE_DEVICES from --cudaID (reference main.py:107): keep the device this test runs on
    cmd += ["--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")]
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_main_train_with_summary_dir_end_to_end(tmp_path):
    _write_calendar(str(tmp_path))
    # fixed-order reductions: a run's training is a function of its inputs alone, so monitoring must leave it bit for bit
    # as it is (in the default mode the fp32 atomics let two runs drift apart over the steps, monitored or not)
    common = ["--mode", "train", "--deterministic", "--synthetic_data", "--max_iter", "4", "--summary_freq", "2",
              "--save_freq", "4", "--display_freq", "2", "--crop_size", "16", "--batch_size", "1", "--RNN_N", "3",
              "--num_resblock", "2", "--output_ext", "png"]
    out1 = _main(str(tmp_path), *common, "--output_dir", "run1", "--summary_dir", "summ")
    out2 = _main(str(tmp_path), *common, "--output_dir", "run2")

    # event file: train scalars and val_* at steps 2 and 4
    sys.path.insert(0, os.path.dirname(__file__))
    from test_train_monitoring_host import read_events
    files = glob.glob(str(tmp_path / "summ" / "events.out.tfevents.*"))
    assert len(files) == 1
    ev = read_events(files[0])
    by_step = {}
    for e in ev[1:]:
        by_step.setdefault(e["step"], []).extend(t for t, _ in e["values"])
    assert sorted(by_step) == [2, 4]
    for s in (2, 4):
        tags = by_step[s]
        assert "learning_rate" in tags and "l2_content_loss" in tags and "t_balance" in tags and "withD_counter" in tags
        assert "val_l2_content_loss" in tags and "val_t_discrim_loss" in tags and "val_t_balance" not in tags

    # stdout and logfile.txt: the reference's blocks, in its order
    log = open(str(tmp_path / "summ" / "logfile.txt")).read()
    for text in (out1, log):
        assert text.count("Run and Recording summary!!") == 2
        assert text.count("-----------Validation data scalars-----------") == 2
        assert "val_l2_content_loss " in text
        i = text.index("Run and Recording summary!!")
        assert i < text.index("-----------Validation data scalars-----------") < text.index("progress  step 2")

    # test-sequence frames at step 0 and step 4, identical to a separate inference run on model-4.pt
    names = sorted(os.path.basename(p) for p in glob.glob(str(tmp_path / "run1" / "train" / "*")))
    assert len(names) == 20
    assert names[:10] == ["000000000_%04d.png" % i for i in range(1, 11)]
    assert names[10:] == ["000000004_%04d.png" % i for i in range(1, 11)]
    _main(str(tmp_path), "--mode", "inference", "--checkpoint", "run1/model-4.pt", "--num_resblock", "2",
          "--input_dir_LR", "./LR/calendar/", "--input_dir_len", "10", "--output_dir", "inf", "--output_name", "000000004",
          "--output_pre", "", "--output_ext", "png")
    for i in range(1, 11):
        a = open(str(tmp_path / "run1" / "train" / ("000000004_%04d.png" % i)), "rb").read()
        b = open(str(tmp_path / "inf" / ("000000004_%04d.png" % i)), "rb").read()
        assert a == b, i

    # without --summary_dir: no log, no events, no frames, no validation lines -- and the same training
    assert not os.path.exists(str(tmp_path / "run2" / "train"))
    assert "val_" not in out2 and "Run and Recording summary!!" not in out2
    assert sorted(os.listdir(str(tmp_path))) == ["LR", "inf", "run1", "run2", "summ"]
    assert not glob.glob(str(tmp_path / "run2" / "events.*")) and not glob.glob(str(tmp_path / "run2" / "logfile.txt"))
    m1 = torch.load(str(tmp_path / "run1" / "model-4.pt"))
    m2 = torch.load(str(tmp_path / "run2" / "model-4.pt"))
    assert set(m1) == set(m2)
    for k in m1:
        assert torch.equal(m1[k], m2[k]), k
