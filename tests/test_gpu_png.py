"""GPU: tecogan_b200.png.encode_png writes the bytes cv2.imencode writes, for every seeded frame of tests/png_cases.py
(sizes the engines produce, degenerate shapes, content classes, constructed streams), for a generator output, and through
save_img in main.py --mode inference and test_while_train.  CV2_SHA256 records cv2's bytes for the seeded frames, so a
frame is checked against the live cv2 and against the recorded one (tests/test_png_host.py checks the record on the
host)."""
import argparse
import glob
import hashlib
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from tests import png_cases as PC
from tests.conftest import GOLDEN, ROOT

CV2_SHA256 = {
    "smooth_32x32": "a789023b32a84d1b41b669800997f6bc049fbd8a304bb1e539357f33365847f8",
    "smooth_128x128": "0f059be3cff84b9b4927129b76510717e5ab733d7b12542966969bdc72ba439c",
    "smooth_512x512": "c5a7390edc00e9eb7717ee4b4acadb3fd271d8f45f8cbde6668e56f304f33fd6",
    "smooth_1080x1920": "8498b61d7ff12856785a43a55cc71944dadc8569d870addf5c98fb0790497b84",
    "smooth_2160x3840": "819897b6131d81f469931e7c97407f75f7cbeed2545f1d7e6c0fb99a272df739",
    "noise_1x1": "22ff0f06ff3418d7695601b989fa7bd7ab87dfc7de88d90eb146c83a36ac47f2",
    "noise_h1": "a161f7ffde751aeafb7171c078a726130aa11c3d55955de76e7bc1e9b4398929",
    "noise_w1": "8c69203193acdaf87258050cf3137bb55ce847ca9d4f3aaf5493c5e602b8b7a9",
    "low_w1": "632184d5418e98fa7b2440481d65be5dc5cb56d361b7e6c0c267a82654998e90",
    "low_odd": "79685565e80ef4c55a9762d94bc2a2161fce551192f4a787c66c8d97390883e6",
    "smooth_odd": "78926f00d88660b6a8ed470329556c3380ee8aeddf90c790a460f7b7f74436bf",
    "noise_576x720": "e2b869903a489c7cd7853397d794b52b15b2e234403e20de45bef5db1e44706e",
    "noise_then_smooth": "4356ac33750081e3f89a1d28b480988498252052c09e9984a79129b264bd0097",
    "constant": "39021fc1a8c24098c2bc1bba67f000cedbbc92f985fac0262aaf91f99baf60f4",
    "constant_1x1": "ba043dcbb5447c973c8a52a57528135016177312d263d33cd591d38f5cc8ebe8",
    "exact_blocks": "61dc1a89461e47c5076e94cecf3cb05988a7db6e4f8a31cbb21bacfa1e5ad104",
    "long_codes": "e683c796d31cc03b08c2ae228edba9a6539a93b6ca40c7e4167fae50a3b74a16",
    "one_literal": "25fab439b5d830fb95110763ef11420260e575b04f82890988759efcd1c3fca0",
    "runs_3": "00573092f713fea3b6f250bd44d925eea94dcc9e1a1897c8ebf3d18ae9c12c10",
    "runs_4": "833be5aa5d99a4590470242e234b56d20cf0b3d0a7e9e05087ea67f5d491a8b5",
    "runs_258": "e7aa85990628b835677a27f56234f5e872342dcfb5fe5cb4d75f87d152f42f6d",
    "runs_259": "b988feeae2cc26d2e450a55b32cc0247f37b0ec6cae620aaa394d13d1f1a5e03",
    "runs_260": "27f215ae7c6c003a8fe91d637c3364fb353153b54b7be1fc151d13ca69a7af68",
    "runs_261": "5929a2230918a121d0eb1c257a16568009d597afc4fe90d4ba93461326c48675",
}


def _cv2_png(rgb):
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(rgb[:, :, ::-1]))
    assert ok
    return buf.tobytes()


@pytest.fixture(scope="module")
def cases():
    return PC.cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CV2_SHA256))
def test_encode_matches_cv2(cases, name):
    from tecogan_b200.png import encode_png
    rgb = cases[name]
    got = encode_png(torch.from_numpy(rgb).cuda())
    ref = _cv2_png(rgb)
    assert hashlib.sha256(ref).hexdigest() == CV2_SHA256[name]
    assert got == ref, (name, len(got), len(ref))


@pytest.mark.gpu
def test_repeated_calls_reuse_buffers(cases):
    from tecogan_b200 import png
    a, b = cases["smooth_128x128"], cases["low_odd"]
    first = png.encode_png(torch.from_numpy(a).cuda())
    ws = png._state["ws"].data_ptr()
    for _ in range(3):
        assert png.encode_png(torch.from_numpy(a).cuda()) == first
    assert png._state["ws"].data_ptr() == ws
    assert png.encode_png(torch.from_numpy(b).cuda()) == _cv2_png(b)      # another size, then back
    assert png.encode_png(torch.from_numpy(a).cuda()) == first


@pytest.mark.gpu
def test_rejects_bad_input():
    from tecogan_b200.png import encode_png
    with pytest.raises(ValueError):
        encode_png(torch.zeros(4, 4, 3, dtype=torch.uint8))                  # CPU tensor
    with pytest.raises(ValueError):
        encode_png(torch.zeros(4, 4, 3, device="cuda"))                       # float
    with pytest.raises(ValueError):
        encode_png(torch.zeros(4, 4, 4, dtype=torch.uint8, device="cuda"))   # not RGB
    with pytest.raises(ValueError):
        encode_png(torch.zeros(4, 6, 3, dtype=torch.uint8, device="cuda")[:, ::2])
    with pytest.raises(ValueError):
        encode_png(torch.zeros(0, 4, 3, dtype=torch.uint8, device="cuda"))


@pytest.mark.gpu
def test_c_abi_rejects_small_buffers():
    import ctypes as C
    from tecogan_b200 import _ffi, png
    ws, cap = png.plan_bytes(16, 16)
    x = torch.zeros(16, 16, 3, dtype=torch.uint8, device="cuda")
    w = torch.empty(ws, dtype=torch.uint8, device="cuda")
    o = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.empty(1, dtype=torch.int64, device="cuda")
    f = _ffi.lib().teco_png_encode_rgb8
    s = _ffi.stream_ptr()
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws - 1, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap - 1, _ffi.ptr(n), s) == -1
    assert f(None, 16, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 0, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    with pytest.raises(ValueError):
        png.plan_bytes(16, 0)


@pytest.mark.gpu
def test_generator_output_576x720():
    """The calendar fixture through the generator with seeded weights: an HR frame as save_img quantises it."""
    from oracle import teco_oracle as O
    from tecogan_b200 import config, kernels as K, variables as V
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.png import encode_png
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=4)), O.init_fnet(seed=4321)
    V.set_default_store(V.VariableStore()).load({**pg, **pf})
    config.set_precision("fp32")
    fr = np.load(os.path.join(GOLDEN, "calendar_lr.npz"))["full_u8"][:3].astype(np.float32) / 255.0
    outs = InferenceEngine(144, 180, 4).run_sequence([torch.from_numpy(f).cuda() for f in fr])
    for o in outs:
        u8 = K.to_u8(o[0]).contiguous()
        assert tuple(u8.shape) == (576, 720, 3)
        assert encode_png(u8) == _cv2_png(u8.cpu().numpy())


def _write_lr(root, n=8, h=24, w=28):
    p = os.path.join(root, "LR", "calendar")
    os.makedirs(p)
    g = np.random.default_rng(3)
    base = PC.smooth(h + 8, w + 8, 21)
    for i in range(n):
        fr = np.clip(base[i % 4:i % 4 + h, i // 4:i // 4 + w].astype(np.int32) + g.integers(-3, 4, (h, w, 3)), 0, 255)
        cv2.imwrite(os.path.join(p, "%04d.png" % (i + 1)), fr.astype(np.uint8)[:, :, ::-1])
    return p


def _same_as_lossless(png_dir, bmp_dir, names):
    """Every .png equals cv2's PNG of the frame the host path wrote losslessly as .bmp."""
    assert names
    for name in names:
        rgb = cv2.imread(os.path.join(bmp_dir, name + ".bmp"), cv2.IMREAD_UNCHANGED)[:, :, ::-1]
        got = open(os.path.join(png_dir, name + ".png"), "rb").read()
        assert got == _cv2_png(rgb), name


@pytest.mark.gpu
def test_main_inference_png_end_to_end(tmp_path):
    _write_lr(str(tmp_path))
    for ext in ("png", "bmp"):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            os.path.join(ROOT, "main.py"), "--mode", "inference", "--checkpoint", "random:5", "--num_resblock", "2",
            "--input_dir_LR", "./LR/calendar/", "--output_dir", "out_" + ext, "--output_pre", "", "--output_ext", ext,
            "--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")]
        r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    names = sorted(os.path.splitext(os.path.basename(f))[0] for f in glob.glob(str(tmp_path / "out_png" / "*.png")))
    assert len(names) == 8
    _same_as_lossless(str(tmp_path / "out_png"), str(tmp_path / "out_bmp"), names)


@pytest.mark.gpu
def test_while_train_png(tmp_path, monkeypatch):
    import main as M
    from oracle import teco_oracle as O
    from tecogan_b200 import variables as V
    _write_lr(str(tmp_path), n=10)
    monkeypatch.chdir(str(tmp_path))
    pg, pf = O.damp_generator(O.init_generator(seed=7, num_resblock=2)), O.init_fnet(seed=8)
    V.set_default_store(V.VariableStore()).load({**pg, **pf})
    for ext in ("png", "bmp"):
        fl = argparse.Namespace(output_dir=str(tmp_path / ("run_" + ext)), precision="fp32", num_resblock=2,
                                output_ext=ext)
        M.test_while_train(fl, 3)
    names = ["000000003_%04d" % i for i in range(1, 11)]
    assert sorted(os.path.splitext(f)[0] for f in os.listdir(str(tmp_path / "run_png" / "train"))) == names
    _same_as_lossless(str(tmp_path / "run_png" / "train"), str(tmp_path / "run_bmp" / "train"), names)


@pytest.mark.gpu
def test_save_img_routes_and_unwritable_path(tmp_path):
    """.PNG in any case goes to the device encoder; an unwritable path is ignored as cv2.imwrite's False is."""
    from tecogan_b200.lib.ops import save_img
    img = torch.rand(20, 30, 3, device="cuda")
    save_img(str(tmp_path / "a.PNG"), img)
    save_img(str(tmp_path / "b.jpg"), img)
    save_img(str(tmp_path / "missing" / "c.png"), img)
    u8 = (img.clamp(0, 1) * 255).cpu()
    got = open(str(tmp_path / "a.PNG"), "rb").read()
    rgb = cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_UNCHANGED)[:, :, ::-1]
    assert got == _cv2_png(rgb)
    assert np.abs(rgb.astype(np.int32) - u8.numpy().astype(np.int32)).max() <= 1
    assert os.path.getsize(str(tmp_path / "b.jpg")) > 0
    assert not os.path.exists(str(tmp_path / "missing"))
