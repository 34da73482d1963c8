"""GPU: the GIF encoder (tecogan_b200/csrc/gif.cu) writes the oracle's bytes (tests/golden/gif_oracle.py) and the recorded
hashes for batches of different animations; the summary quantisation is convert_image_dtype's; buffers are reused and
bad inputs rejected; Network.image_summary encodes the training step's own tensors without touching training state; and
main.py --mode train --summary_dir writes the reference's GIF summaries to <summary_dir>/gif."""
import ctypes as C
import glob
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import gif_cases as GC
from tests.conftest import ROOT
from tests.golden import gif_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases():
    return GC.cases()


@pytest.mark.parametrize("name", list(GC.HASHES))
def test_device_bytes_equal_oracle_and_hashes(cases, name):
    from tecogan_b200.gif import encode_gif
    batch = cases[name]
    files = encode_gif(torch.from_numpy(batch).cuda())
    assert len(files) == len(batch)
    for i, (a, data) in enumerate(zip(batch, files)):
        ref, _ = O.encode(a)
        assert data == ref, (name, i, len(data), len(ref))
        assert GC.sha(data) == GC.HASHES[name][i]


def test_batch_has_no_cross_talk(cases):
    """Each animation of a batch encodes as it does alone, and in any position of the batch."""
    from tecogan_b200.gif import GifEncoder
    enc = GifEncoder()
    b = cases["lr_summary"]
    together = enc.encode(torch.from_numpy(b).cuda())
    flipped = enc.encode(torch.from_numpy(b[::-1].copy()).cuda())
    assert flipped == together[::-1]
    for i in range(len(b)):
        assert enc.encode(torch.from_numpy(b[i:i + 1]).cuda()) == [together[i]]


def test_convert_image_u8_boundaries():
    from tecogan_b200.gif import convert_image_u8
    k = np.arange(256, dtype=np.float32)
    b = (k / np.float32(255.5)).astype(np.float32)
    vals = np.concatenate([b, np.nextafter(b, np.float32(-1)), np.nextafter(b, np.float32(2)),
                           np.array([-0.1, 1.2, np.nan, -np.inf, np.inf, 0.0, -0.0, 1.0, 255.0 / 255.5, 1e30],
                                    dtype=np.float32)]).astype(np.float32)
    for dep in (False, True):
        x = vals * 2 - 1 if dep else vals
        x = x.astype(np.float32)
        got = convert_image_u8(torch.from_numpy(x).cuda(), deprocess=dep).cpu().numpy()
        np.testing.assert_array_equal(got, O.convert_image_dtype(x, deprocess=dep))
    got = convert_image_u8(torch.from_numpy(vals).cuda()).cpu().numpy()
    assert got[-8] == 0 and got[-9] == 255 and got[-10] == 0       # NaN -> 0, 1.2 -> 255, -0.1 -> 0


def test_repeated_calls_reuse_buffers(cases):
    from tecogan_b200 import gif
    x = torch.from_numpy(cases["noise"]).cuda()
    first = gif.encode_gif(x)
    ws = gif._state["ws"].data_ptr()
    assert gif.encode_gif(x) == first
    assert gif._state["ws"].data_ptr() == ws
    other = gif.encode_gif(torch.from_numpy(cases["ties"]).cuda())          # another size: new buffers, right bytes
    assert other == [O.encode(a)[0] for a in cases["ties"]]
    assert gif.encode_gif(x) == first


def test_bad_inputs_are_rejected():
    from tecogan_b200.gif import convert_image_u8, encode_gif, plan_bytes
    ok = torch.zeros((1, 2, 4, 4, 3), dtype=torch.uint8, device="cuda")
    for bad in (ok.cpu(), ok.float(), ok[..., :2].contiguous(), ok[0], ok.transpose(2, 3),
                torch.zeros((1, 0, 4, 4, 3), dtype=torch.uint8, device="cuda"),
                torch.zeros((1, 1, 4, 65536, 3), dtype=torch.uint8, device="cuda")):
        with pytest.raises(ValueError):
            encode_gif(bad)
    for dims in ((1, 0, 4, 4), (0, 1, 4, 4), (1, 1, 65536, 1), (1, 1, 0, 5), (1, 1 << 12, 1 << 9, 1 << 8)):
        with pytest.raises(ValueError):
            plan_bytes(*dims)
    assert plan_bytes(1, 1, 65535, 1)[0] > 0
    with pytest.raises(ValueError):
        convert_image_u8(torch.zeros(4, device="cuda", dtype=torch.float64))


def test_c_abi_rejects_small_or_misaligned_buffers():
    from tecogan_b200._ffi import lib
    L = lib()
    n, t, h, w = 2, 3, 9, 11
    ws, cap = C.c_int64(0), C.c_int64(0)
    assert L.teco_gif_plan_bytes(n, t, h, w, C.byref(ws), C.byref(cap)) == 0
    x = torch.zeros((n, t, h, w, 3), dtype=torch.uint8, device="cuda")
    wsb = torch.empty(ws.value + 256, dtype=torch.uint8, device="cuda")
    out = torch.empty(cap.value, dtype=torch.uint8, device="cuda")
    ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda tt, off=0: C.c_void_p(tt.data_ptr() + off)
    assert L.teco_gif_encode_rgb8(P(x), n, t, h, w, P(wsb), ws.value - 1, P(out), cap.value, P(ln), s) == -1
    assert L.teco_gif_encode_rgb8(P(x), n, t, h, w, P(wsb), ws.value, P(out), cap.value - 1, P(ln), s) == -1
    assert L.teco_gif_encode_rgb8(P(x), n, t, h, w, P(wsb, 16), ws.value, P(out), cap.value, P(ln), s) == -1
    assert L.teco_gif_encode_rgb8(None, n, t, h, w, P(wsb), ws.value, P(out), cap.value, P(ln), s) == -1
    assert L.teco_gif_encode_rgb8(P(x), n, 0, h, w, P(wsb), ws.value, P(out), cap.value, P(ln), s) == -1
    assert L.teco_convert_image_u8(P(x), P(x), 0, 0, s) == -1
    assert L.teco_convert_image_u8(P(x), P(x), 4, 2, s) == -1
    torch.cuda.synchronize()
    assert (ln == 0).all()                                 # a rejected call wrote nothing
    assert L.teco_gif_encode_rgb8(P(x), n, t, h, w, P(wsb), ws.value, P(out), cap.value, P(ln), s) == 0
    torch.cuda.synchronize()
    lens = ln.tolist()
    data = out[:sum(lens)].cpu().numpy().tobytes()
    ref = O.encode(np.zeros((t, h, w, 3), np.uint8))[0]
    assert data == ref + ref


# ------------------------------------------------------------------------------------- Network.image_summary
def _golden_net(name):
    sys.path.insert(0, os.path.dirname(__file__))
    from test_gpu_train_monitoring import _case, _net
    g, FL, P = _case(name)
    return g, FL, _net(g, FL, P)


def _state(net):
    st = net.train
    t = {"static_in": st.static_in, "static_tg": st.static_tg, "bucket": st.bucket}
    for tag, opt in (("g", st.opt_g), ("f", st.opt_f), ("d", st.opt_d)):
        if opt is not None:
            t.update({tag + "_flat": opt.flat, tag + "_m": opt.m, tag + "_v": opt.v})
    t.update({"summary/%d" % i: v for i, v in enumerate(st._summary_src[:3])})
    t.update({"warppre/%d" % i: v for i, v in enumerate(st._summary_src[3])})
    return {k: v.detach().clone() for k, v in t.items()}


@pytest.mark.parametrize("name", ["teco_pp", "frvsr"])
def test_image_summary_is_the_step_tensors_encoded_and_leaves_training_alone(name):
    g, FL, net = _golden_net(name)
    ri, rt = torch.from_numpy(g["r_inputs"]), torch.from_numpy(g["r_targets"])
    res = net.train()
    before = _state(net)
    host = (net.train.global_step, list(net.train.loss_ema), net.train.tb_ema, net.train.counter1, net.train.counter2)
    items = net.image_summary()
    after = _state(net)
    for k in before:
        assert torch.equal(before[k], after[k]), k             # bit for bit: the summary writes nothing training reads
    assert host == (net.train.global_step, list(net.train.loss_ema), net.train.tb_ema, net.train.counter1,
                    net.train.counter2)
    assert net.image_summary() == items

    B = FL.batch_size
    k = min(4, B)
    if FL.pingpang:
        ri = torch.cat((ri, torch.flip(ri[:, :-1], dims=(1,))), dim=1)
        rt = torch.cat((rt, torch.flip(rt[:, :-1], dims=(1,))), dim=1)
    T = ri.shape[1]
    gen = res["gen_outputs"].cpu().numpy()
    warp = np.stack([w.cpu().numpy() for w in net.train._summary_src[3]], 1)
    assert gen.shape[1] == T and warp.shape[1] == T - 1
    want = [("LR", O.convert_image_dtype(ri.numpy())), ("HR", O.convert_image_dtype(rt.numpy(), True)),
            ("Generated", O.convert_image_dtype(gen, True)), ("WarpPreGen", O.convert_image_dtype(warp, True))]
    exp = []
    for nm, u8 in want:
        for i in range(k):
            tag = "image_summaries/%s/gif" % nm + ("" if k == 1 else "/%d" % i)
            exp.append((tag, u8.shape[2], u8.shape[3], O.encode(u8[i])[0]))
    assert [e[:3] for e in items] == [e[:3] for e in exp]
    for got, e in zip(items, exp):
        assert got[3] == e[3], got[0]


# ------------------------------------------------------------------------------------------ main.py end to end
def _main(cwd, *args):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(ROOT, "main.py")] + list(args)
    cmd += ["--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")]
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _gif_frames(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    assert im.info.get("loop") == 0
    out = []
    for i in range(im.n_frames):
        im.seek(i)
        assert im.info.get("duration") == 330
        out.append(np.array(im.convert("RGB")))
    return np.stack(out)


@pytest.mark.parametrize("model", ["frvsr_b1", "tecogan_pp_b2"])
def test_main_train_writes_gif_summaries(tmp_path, model):
    from tensorboard.backend.event_processing import event_accumulator as ea
    args = ["--mode", "train", "--synthetic_data", "--max_iter", "4", "--summary_freq", "2", "--save_freq", "100",
            "--display_freq", "2", "--crop_size", "16", "--RNN_N", "3", "--num_resblock", "2", "--output_ext", "png",
            "--output_dir", "run", "--summary_dir", "summ"]
    args += ["--ratio", "0", "--batch_size", "1"] if model == "frvsr_b1" else ["--pingpang", "--batch_size", "2"]
    _main(str(tmp_path), *args)
    assert len(glob.glob(str(tmp_path / "summ" / "events.out.tfevents.*"))) == 1
    files = glob.glob(str(tmp_path / "summ" / "gif" / "events.out.tfevents.*"))
    assert len(files) == 1
    acc = ea.EventAccumulator(str(tmp_path / "summ" / "gif"), size_guidance={ea.IMAGES: 0})
    acc.Reload()
    k = 1 if model == "frvsr_b1" else 2
    T = 3 if model == "frvsr_b1" else 5
    names = ("LR", "HR", "Generated", "WarpPreGen")
    tags = ["image_summaries/%s/gif" % n + ("" if k == 1 else "/%d" % i) for n in names for i in range(k)]
    assert sorted(acc.Tags()["images"]) == sorted(tags)
    for tag in tags:
        evs = acc.Images(tag)
        assert [e.step for e in evs] == [2, 4]
        side = 16 if "/LR/" in tag + "/" else 64
        n_frames = T - 1 if "WarpPreGen" in tag else T
        for e in evs:
            assert (e.height, e.width) == (side, side)
            f = _gif_frames(e.encoded_image_string)
            assert f.shape == (n_frames, side, side, 3), (tag, f.shape)
