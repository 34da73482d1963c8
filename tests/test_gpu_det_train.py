"""GPU: deterministic training (config.set_deterministic / main.py --deterministic).  Two runs from one seed agree bit
for bit -- every variable, Adam moment, counter, loss EMA and tb_ema, the validation scalars and the test-sequence frames --
for FRVSR and TecoGAN (ping-pong, VGG, D and its layer loss), fp32 and bf16, on the CUDA-graph and the eager path, from
--synthetic_data and from PNG scenes through the device frame store.  The graph and the eager step give the same bits,
torch.use_deterministic_algorithms(True) finds nothing to object to, and k steps + save + restore (.pt and TF bundle) +
m steps equal k + m uninterrupted steps exactly."""
import glob
import os
import re
import subprocess
import sys

import pytest
import torch

from tests.conftest import ROOT
from tests.test_frame_store_host import _scenes
from tests.test_gpu_train_monitoring import _write_calendar

pytestmark = pytest.mark.gpu


def _main(cwd, *args):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(ROOT, "main.py")] + list(args)
    cmd += ["--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")]
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _val_lines(out):
    return [l for l in out.splitlines() if l.startswith("val_")]


def _same_checkpoints(a, b):
    m1, m2 = torch.load(a), torch.load(b)
    assert set(m1) == set(m2)
    for k in m1:
        assert torch.equal(m1[k], m2[k]), k
    return m1


CASES = {   # name: flags of one run (besides the shared ones)
    "frvsr_fp32_graph": ["--ratio", "-0.01", "--train_precision", "fp32"],
    "frvsr_bf16_eager": ["--ratio", "-0.01", "--train_precision", "bf16", "--Dt_ratio_add", "0.01"],
    "teco_fp32_eager": ["--ratio", "0.01", "--pingpang", "--vgg_scaling", "0.2", "--train_precision", "fp32",
                        "--Dt_ratio_add", "0.01"],
    "teco_bf16_graph": ["--ratio", "0.01", "--pingpang", "--vgg_scaling", "0.2", "--train_precision", "bf16"],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_two_deterministic_runs_are_bit_identical(tmp_path, case):
    _write_calendar(str(tmp_path))
    common = ["--mode", "train", "--deterministic", "--synthetic_data", "--max_iter", "4", "--summary_freq", "2",
              "--save_freq", "4", "--display_freq", "2", "--crop_size", "16", "--batch_size", "2", "--RNN_N", "3",
              "--num_resblock", "2", "--output_ext", "png", "--rand_seed", "5"] + CASES[case]
    outs = []
    for r in ("a", "b"):
        outs.append(_main(str(tmp_path), *common, "--output_dir", "run_" + r, "--summary_dir", "summ_" + r))
    m = _same_checkpoints(str(tmp_path / "run_a" / "model-4.pt"), str(tmp_path / "run_b" / "model-4.pt"))
    assert any(k.endswith("/Adam") for k in m) and any(k.startswith("teco_b200/") for k in m)
    va, vb = _val_lines(outs[0]), _val_lines(outs[1])
    assert va and va == vb
    frames = sorted(os.path.basename(p) for p in glob.glob(str(tmp_path / "run_a" / "train" / "*.png")))
    assert len(frames) == 20
    for f in frames:
        assert open(str(tmp_path / "run_a" / "train" / f), "rb").read() == \
            open(str(tmp_path / "run_b" / "train" / f), "rb").read(), f
    # the training log's loss lines (wall time stripped) agree too
    la = [re.sub(r"[0-9.]+ ?(sec|min|s)\b.*", "", l) for l in outs[0].splitlines() if "loss" in l]
    lb = [re.sub(r"[0-9.]+ ?(sec|min|s)\b.*", "", l) for l in outs[1].splitlines() if "loss" in l]
    assert la == lb


def test_two_deterministic_runs_from_png_scenes_are_bit_identical(tmp_path):
    data = str(tmp_path / "frames")
    _scenes(data, [(84, 96), (80, 80), (90, 101), (96, 84), (82, 88), (88, 90)], frames=10, seed=3)
    common = ["--mode", "train", "--deterministic", "--input_video_dir", data, "--str_dir", "2000", "--end_dir", "2003",
              "--end_dir_val", "2005", "--max_frm", "9", "--RNN_N", "3", "--batch_size", "2", "--crop_size", "16",
              "--num_resblock", "2", "--ratio", "0.01", "--vgg_scaling", "0.2", "--synthetic_data", "--max_iter", "4",
              "--summary_freq", "2", "--save_freq", "4", "--display_freq", "100", "--queue_thread", "2",
              "--train_precision", "bf16"]
    outs = [_main(str(tmp_path), *common, "--output_dir", "run_" + r, "--summary_dir", "summ_" + r) for r in "ab"]
    assert "training reads its clips from the frame store on the device" in outs[0]
    _same_checkpoints(str(tmp_path / "run_a" / "model-4.pt"), str(tmp_path / "run_b" / "model-4.pt"))
    assert _val_lines(outs[0]) and _val_lines(outs[0]) == _val_lines(outs[1])


_STEPS = r"""
import sys, torch
import main as M
from tests.test_gpu_train import _case, _fresh_store
from tests.test_gpu_train_monitoring import _snapshot
from tecogan_b200 import config
from tecogan_b200 import variables as V
from tecogan_b200.lib.Teco import FRVSR, TecoGAN
name, precision, graph, dalg, steps, load, save, out = sys.argv[1:9]
config.set_deterministic(True)
config.set_train_precision(precision)
g, FL, P = _case(name)
FL.train_cuda_graph = graph == "1"
ri, rt = torch.from_numpy(g["r_inputs"]).cuda(), torch.from_numpy(g["r_targets"]).cuda()
st = _fresh_store(P)
if load != "-":
    st = V.set_default_store(V.VariableStore())
    M.load_checkpoint(st, load, FL.num_resblock, need_d=True, need_vgg=FL.vgg_scaling > 0)
    if FL.vgg_scaling > 0:
        st.load({k: v for k, v in P.items() if k.startswith("vgg_19/")})
net = TecoGAN(ri, rt, FL) if name.startswith("teco") else FRVSR(ri, rt, FL)
if load != "-":
    assert M.restore_train_state(net.train, load) == []
torch.use_deterministic_algorithms(dalg == "1")
for _ in range(int(steps)):
    net.train()
ev = net.train.evaluate(ri, rt)
torch.use_deterministic_algorithms(False)
if save != "-":
    import os
    os.makedirs(save, exist_ok=True)
    M.save_checkpoint(st, save, net.global_step(), net.train)
t, host = _snapshot(net)
state = {k: v.detach().cpu() for k, v in net.train.state_tensors().items()}
torch.save({"t": {k: v.cpu() for k, v in t.items() if not k.startswith("static")}, "host": host, "eval": ev,
            "state": state}, out)
"""


def _steps(tmp_path, tag, name, precision, graph, steps, dalg=False, load="-", save="-"):
    """Train `steps` steps of the golden case `name` in a process of its own; returns its snapshot."""
    out = str(tmp_path / (tag + ".pt"))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _STEPS, name, precision, str(int(graph)),
                                                                        str(int(dalg)), str(steps), load, save, out]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return torch.load(out)


def _same_snap(a, b):
    assert a["host"] == b["host"]
    assert set(a["t"]) == set(b["t"])
    for k in a["t"]:
        assert torch.equal(a["t"][k], b["t"][k]), k
    for k in a["state"]:
        assert torch.equal(a["state"][k], b["state"][k]), k


@pytest.mark.parametrize("name,precision", [
    ("teco_pp", "fp32"), ("frvsr", "fp32"), ("frvsr", "bf16"),
    # bf16 TecoGAN: the graph runs and the eager runs each reproduce bit for bit, but the two paths differ from each other
    # (DESIGN section 4.3); this case records that gap and fails loudly once it is closed.
    pytest.param("teco_pp", "bf16", marks=pytest.mark.xfail(strict=True, reason="bf16 TecoGAN graph and eager steps differ")),
])
def test_graph_and_eager_steps_are_bit_identical(tmp_path, name, precision):
    """Three steps and a validation pass on the CUDA graph and eagerly under torch.use_deterministic_algorithms(True)."""
    graph = _steps(tmp_path, "graph", name, precision, True, 3)
    eager = _steps(tmp_path, "eager", name, precision, False, 3, dalg=True)
    _same_snap(graph, eager)
    assert graph["eval"] == eager["eval"]


@pytest.mark.parametrize("fmt", ["tf", "pt"])
def test_deterministic_resume_is_exact(tmp_path, fmt):
    """2 steps + save + restore + 3 steps == 5 uninterrupted steps, every tensor and EMA bit for bit."""
    whole = _steps(tmp_path, "whole", "teco_pp", "fp32", True, 5)
    _steps(tmp_path, "first", "teco_pp", "fp32", True, 2, save=str(tmp_path / "ck"))
    spec = str(tmp_path / "ck" / "model-2") + ("" if fmt == "tf" else ".pt")
    resumed = _steps(tmp_path, "resumed", "teco_pp", "fp32", True, 3, load=spec)
    assert resumed["host"][0] == 5
    _same_snap(whole, resumed)


def _rank_run(tmp_path, tag):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", "2",
           os.path.join(ROOT, "main.py"), "--mode", "train", "--deterministic", "--synthetic_data", "--max_iter", "3",
           "--save_freq", "3", "--display_freq", "100", "--crop_size", "16", "--batch_size", "2", "--RNN_N", "3",
           "--num_resblock", "2", "--ratio", "0.01", "--output_dir", tag]
    r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_runs_are_bit_identical(tmp_path):
    _rank_run(tmp_path, "a")
    _rank_run(tmp_path, "b")
    _same_checkpoints(str(tmp_path / "a" / "model-3.pt"), str(tmp_path / "b" / "model-3.pt"))
