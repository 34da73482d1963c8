"""GPU: the inference input read on the device.  teco_gauss_blur_down4 equals cv2.GaussianBlur(frame, (0, 0),
sigmaX=1.5)[::4, ::4] / 255 and the numpy restatement (tests/golden/gauss_blur_oracle.py) bit for bit, on uint8 and uint16
frames batched per launch; teco_frames_to_f32 equals frame / 255; inference_data_loader gives the inputs the host formula
of the reference (lib/dataloader.py:11-50, restated here with cv2) gives, for every PNG flavour a sequence may hold; and
main.py --mode inference writes the same files from them as from host-loaded frames."""
import argparse
import os
import shutil

import cv2
import numpy as np
import pytest
import torch

from tests import png_decode_cases as PD
from tests.conftest import GOLDEN
from tests.golden import gauss_blur_oracle as G
from tests.golden import make_golden_gauss_blur as MG

LARGE = [(576, 720), (480, 720), (576, 704), (534, 1280), (1080, 1921)]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _cv2_down(frame_rgb):
    return G.reference_input(np.ascontiguousarray(frame_rgb[:, :, ::-1]), True)


def _frames(g, n, H, W, dt):
    return g.integers(0, np.iinfo(dt).max + 1, (n, H, W, 3)).astype(dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.uint8, np.uint16])
def test_blur_down4_small_sizes(dt):
    """Every width 2..40 (each class of the 3W-float row modulo 8) at every height 2..20, three frames per launch."""
    from tecogan_b200 import kernels as K
    g = np.random.default_rng(7 if dt == np.uint8 else 8)
    for W in range(2, 41):
        for H in range(2, 21):
            fr = _frames(g, 3, H, W, dt)
            got = K.gauss_blur_down4(torch.from_numpy(fr).cuda()).cpu().numpy()
            for k in range(3):
                assert _same(got[k], _cv2_down(fr[k])), (H, W, k)
            assert _same(got[0], G.down4_rgb(fr[0])), (H, W)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", LARGE)
def test_blur_down4_large_sizes(H, W):
    from tecogan_b200 import kernels as K
    g = np.random.default_rng(H + W)
    for dt, n in ((np.uint8, 3), (np.uint16, 2)):
        fr = _frames(g, n, H, W, dt)
        got = K.gauss_blur_down4(torch.from_numpy(fr).cuda()).cpu().numpy()
        assert got.shape == (n, (H + 3) // 4, (W + 3) // 4, 3)
        for k in range(n):
            assert _same(got[k], _cv2_down(fr[k])), (H, W, dt, k)
        assert _same(got[-1], G.down4_rgb(fr[-1])), (H, W, dt)


@pytest.mark.gpu
def test_blur_down4_fixture_and_frame_lists():
    """The cv2 outputs recorded in tests/golden/gauss_blur.npz; frames passed as a list of separate tensors."""
    from tecogan_b200 import kernels as K
    z = np.load(os.path.join(GOLDEN, "gauss_blur.npz"))
    for i, f in enumerate(MG.frames()):
        want = np.ascontiguousarray(z["blur%d" % i][::4, ::4]) / np.float32(255.0)
        dev = torch.from_numpy(f).cuda()
        got = K.gauss_blur_down4([dev, dev.clone()]).cpu().numpy()
        assert _same(got[0], want) and _same(got[1], want), MG.CASES[i]


@pytest.mark.gpu
def test_blur_down4_refuses_bad_frames():
    from tecogan_b200 import kernels as K
    for shape in ((1, 1, 8, 3), (1, 8, 1, 3)):
        with pytest.raises(ValueError, match="1-pixel side"):
            K.gauss_blur_down4(torch.zeros(shape, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        K.gauss_blur_down4(torch.zeros((1, 8, 8, 3), dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        K.gauss_blur_down4([torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"),
                            torch.zeros((8, 9, 3), dtype=torch.uint8, device="cuda")])


@pytest.mark.gpu
def test_frames_to_f32():
    from tecogan_b200 import kernels as K
    g = np.random.default_rng(3)
    for dt, (H, W) in ((np.uint8, (144, 180)), (np.uint16, (7, 5)), (np.uint8, (1, 1))):
        fr = _frames(g, 4, H, W, dt)
        got = K.frames_to_f32([torch.from_numpy(f).cuda() for f in fr]).cpu().numpy()
        assert _same(got, fr.astype(np.float32) / np.float32(255.0)), (dt, H, W)


# ------------------------------------------------------------------------------------------ the loader
def _write_folder(d, h, w):
    """One file of each flavour, numbered so that the reference's numeric sort differs from a plain sort, and a file
    the loader skips."""
    os.makedirs(d)
    g = np.random.default_rng(h * w)
    rgb = lambda: g.integers(0, 256, (h, w, 3)).astype(np.uint8)
    files = {
        "f_1.png": cv2.imencode(".png", rgb())[1].tobytes(),
        "f_2.png": PD.made(h, w, 3, 8, 11),                                        # palette
        "f_3.png": PD.made(h, w, 0, 8, 12),                                        # grey
        "f_4.png": PD.made(h, w, 6, 8, 13),                                        # RGBA
        "f_5.png": cv2.imencode(".png", g.integers(0, 65536, (h, w, 3)).astype(np.uint16))[1].tobytes(),
        "f_6.png": cv2.imencode(".png", g.integers(0, 65536, (h, w)).astype(np.uint16))[1].tobytes(),   # 16-bit grey
        "f_7.png": PD.png_file(h, w, 2, 8, PD.compress(PD.filter_rows(PD.pack_rows(
            PD.image(h, w, 2, 8, 14)[0], w, 2, 8), 3, (1,))), before=(PD._exif_orientation(1),)),  # eXIf, upright
        "f_8.png": PD.made(h, w, 2, 8, 15),
        "f_10.png": cv2.imencode(".png", rgb())[1].tobytes(),
        "f_9.png": PD.made(h, w, 3, 4, 16),                                        # 4-bit palette
        "f_11.png": PD.png_file(h, w, 2, 8, PD.compress(PD.filter_rows(PD.pack_rows(
            PD.image(h, w, 2, 8, 17)[0], w, 2, 8), 3, (1,))), before=(PD._exif_orientation(6),)),  # eXIf, turned
        "notes.txt": b"not a frame",
    }
    for name, data in files.items():
        with open(os.path.join(d, name), "wb") as f:
            f.write(data)
    return d


def _host_inputs(paths, down):
    """The parent's host formula: cv.imread(name, 3) -> RGB float32 [-> GaussianBlur[::4, ::4]] / 255."""
    return [G.reference_input(cv2.imread(p, 3), down) for p in paths]


def _flags(lr=None, hr=None, n=-1):
    return argparse.Namespace(input_dir_LR=lr, input_dir_HR=hr, input_dir_len=n)


def _check_loader(data, folder, names, down):
    paths = [os.path.join(folder, n) for n in names]
    assert data.paths_LR == paths[5:0:-1] + paths
    want = _host_inputs(paths, down)
    want = want[5:0:-1] + want
    assert len(data.inputs) == len(want)
    for k, (got, w) in enumerate(zip(data.inputs, want)):
        assert got.is_cuda and got.dtype == torch.float32 and got.dim() == 3
        assert _same(got.cpu().numpy(), w), (k, data.paths_LR[k])
    for k in range(min(5, len(paths) - 1)):             # the warm-up frames are the frames they repeat
        assert data.inputs[k].data_ptr() == data.inputs[10 - k].data_ptr()


@pytest.mark.gpu
@pytest.mark.parametrize("down", [False, True])
def test_loader_matches_host_formula(tmp_path, down):
    from tecogan_b200.lib.dataloader import inference_data_loader, read_inputs
    h, w = (61, 83) if down else (20, 27)
    folder = _write_folder(str(tmp_path / "seq"), h, w)
    names = ["f_%d.png" % k for k in range(1, 12)]
    flags = _flags(hr=folder) if down else _flags(lr=folder)
    _check_loader(inference_data_loader(flags), folder, names, down)
    short = inference_data_loader(argparse.Namespace(**{**vars(flags), "input_dir_len": 7}))
    _check_loader(short, folder, names[:7], down)
    # one file per window: the same frames
    paths = [os.path.join(folder, n) for n in names]
    for got, want in zip(read_inputs(paths, down, window_bytes=1), _host_inputs(paths, down)):
        assert _same(got.cpu().numpy(), want)


@pytest.mark.gpu
def test_loader_errors_and_lr_preference(tmp_path):
    from tecogan_b200.lib.dataloader import inference_data_loader
    with pytest.raises(ValueError, match="Input directory not found"):
        inference_data_loader(_flags(lr=str(tmp_path / "none"), hr=str(tmp_path / "none")))
    lr = _write_folder(str(tmp_path / "lr"), 12, 10)
    hr = _write_folder(str(tmp_path / "hr"), 48, 40)
    data = inference_data_loader(_flags(lr=lr, hr=hr, n=3))
    assert [tuple(t.shape) for t in data.inputs] == [(12, 10, 3)] * 5
    with open(os.path.join(lr, "f_0.png"), "wb") as f:
        f.write(b"\x89PNG broken")
    with pytest.raises(ValueError, match="cannot decode"):
        inference_data_loader(_flags(lr=lr))


@pytest.mark.gpu
def test_calendar_frames(tmp_path):
    from tecogan_b200.lib.dataloader import inference_data_loader
    d = tmp_path / "calendar"
    d.mkdir()
    for k in (1, 2):
        shutil.copy(os.path.join(GOLDEN, "calendar_lr_%04d.png" % k), str(d / ("%04d.png" % k)))
    data = inference_data_loader(_flags(lr=str(d)))
    full = np.load(os.path.join(GOLDEN, "calendar_lr.npz"))["full_u8"]
    assert [os.path.basename(p) for p in data.paths_LR] == ["0002.png", "0001.png", "0002.png"]
    for got, k in zip(data.inputs, (1, 0, 1)):
        assert _same(got.cpu().numpy(), full[k].astype(np.float32) / np.float32(255.0))


@pytest.mark.gpu
@pytest.mark.parametrize("down", [False, True])
def test_main_inference_matches_host_loaded_frames(tmp_path, monkeypatch, down):
    """main.py --mode inference from device-read input writes the files it writes from the parent's host-loaded
    frames (fed to the same engine as CPU tensors)."""
    import main as M
    from tecogan_b200.lib import dataloader as DL
    monkeypatch.chdir(str(tmp_path))
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    seq = tmp_path / "seq"
    seq.mkdir()
    g = np.random.default_rng(5)
    h, w = (128, 144) if down else (32, 36)
    base = cv2.resize(g.integers(0, 256, (h // 8, w // 8, 3)).astype(np.uint8), (w + 16, h + 16),
                      interpolation=cv2.INTER_CUBIC)
    for i in range(8):
        cv2.imwrite(str(seq / ("%04d.png" % (i + 1))), base[i:i + h, 2 * i:2 * i + w])
    args = ["--mode", "inference", "--checkpoint", "random:5", "--num_resblock", "2", "--output_pre", "",
            "--output_ext", "png", "--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0"),
            "--input_dir_HR" if down else "--input_dir_LR", str(seq)]
    M.main(args + ["--output_dir", "dev"])
    monkeypatch.setattr(DL, "read_inputs", lambda paths, d: [torch.from_numpy(a) for a in _host_inputs(paths, d)])
    M.main(args + ["--output_dir", "host"])
    names = sorted(os.listdir(str(tmp_path / "dev")))
    assert names == sorted(os.listdir(str(tmp_path / "host"))) and len(names) == 8
    for n in names:
        assert open(str(tmp_path / "dev" / n), "rb").read() == open(str(tmp_path / "host" / n), "rb").read(), n
