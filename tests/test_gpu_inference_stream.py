"""GPU: the streaming inference command (main.super_resolve_frames over lib/dataloader.py::stream_inputs) writes the files
of the serial loop -- inference_data_loader, then InferenceEngine.step, then save_img, frame after frame -- byte for byte:
LR and HR input, PNG / JPEG / a cv2-only extension, bf16 and fp32, the edges of the warm-up padding, sequences spanning
several decoding windows with and without --input_dir_len, and sequences holding a 16-bit PNG and a file that is not a
PNG.  Its device memory does not grow with the sequence, and an error in the reader or the writer is raised with both
threads joined.  Fixtures are generated from the seeds below."""
import argparse
import itertools
import os
import threading

import cv2
import numpy as np
import pytest
import torch

NRB = 2
LR_HW = (32, 36)


def _write_seq(d, n, hr=False, seed=0, sixteen=(), not_png=()):
    """n smooth moving frames 0001.png ..; file k in `sixteen` is a 16-bit PNG, in `not_png` a BMP named .png."""
    os.makedirs(d, exist_ok=True)
    h, w = (LR_HW[0] * 4, LR_HW[1] * 4) if hr else LR_HW
    g = np.random.default_rng(seed)
    base = cv2.resize(g.integers(0, 256, (h // 4 + 4, w // 4 + 4 + n, 3)).astype(np.uint8), None, fx=4, fy=4,
                      interpolation=cv2.INTER_CUBIC)
    for k in range(n):
        fr = np.clip(base[8:8 + h, 2 * k:2 * k + w].astype(np.int32) + g.integers(-3, 4, (h, w, 3)), 0, 255)
        p = os.path.join(d, "%04d.png" % (k + 1))
        if k in sixteen:
            cv2.imwrite(p, (fr * 256 + g.integers(0, 256, fr.shape)).astype(np.uint16))
        elif k in not_png:
            with open(p, "wb") as f:
                f.write(cv2.imencode(".bmp", fr.astype(np.uint8))[1].tobytes())
        else:
            cv2.imwrite(p, fr.astype(np.uint8))
    return d


def _flags(folder, hr=False, n=-1):
    return argparse.Namespace(input_dir_LR=None if hr else folder, input_dir_HR=folder if hr else None, input_dir_len=n)


def _weights(precision):
    import main as M
    from tecogan_b200 import config, variables as V
    config.set_precision(precision)
    M.load_checkpoint(V.set_default_store(V.VariableStore(seed=1)), "random:5", NRB)


def _serial(flags, out_dir, name, ext):
    """The serial loop of the parent, written out: every input resident, one step, save_img, the next step."""
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_data_loader
    from tecogan_b200.lib.ops import save_img
    data = inference_data_loader(flags)
    h, w = data.inputs[0].shape[:2]
    eng = InferenceEngine(h, w, NRB)
    os.makedirs(out_dir, exist_ok=True)
    n = len(data.inputs)
    for i in range(n):
        out = eng.step(data.inputs[i], next_lr=data.inputs[i + 1] if i + 1 < n else None)
        torch.cuda.synchronize()
        if i >= 5:
            stem = os.path.splitext(os.path.basename(data.paths_LR[i]))[0]
            save_img(os.path.join(out_dir, "%s_%s.%s" % (name, stem, ext)), out[0])


def _streamed(flags, out_dir, name, ext, window_bytes=None):
    import main as M
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_paths, padded, stream_inputs
    paths, down = inference_paths(flags)
    os.makedirs(out_dir, exist_ok=True)
    frames = stream_inputs(paths, down, window_bytes=window_bytes)
    try:
        first = next(frames)
        eng = InferenceEngine(first.shape[0], first.shape[1], NRB)
        M.super_resolve_frames(eng, padded(paths), itertools.chain([first], frames), out_dir, name, ext)
    finally:
        frames.close()


def _same_dirs(a, b, count):
    os.makedirs(a, exist_ok=True)
    os.makedirs(b, exist_ok=True)
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)) and len(names) == count, (names, sorted(os.listdir(b)))
    for n in names:
        with open(os.path.join(a, n), "rb") as f, open(os.path.join(b, n), "rb") as g:
            assert f.read() == g.read(), n


LR_FRAME_BYTES = LR_HW[0] * LR_HW[1] * 3          # one decoded 8-bit LR frame: the window unit of the cases below

CASES = [  # id, n, hr, ext, precision, frames per window (None: the default budget), --input_dir_len, sixteen, not_png
    ("lr_png_bf16", 8, False, "png", "bf16", None, -1, (), ()),
    ("hr_png_bf16", 8, True, "png", "bf16", None, -1, (), ()),
    ("lr_jpg_bf16", 8, False, "jpg", "bf16", None, -1, (), ()),
    ("lr_bmp_bf16", 8, False, "bmp", "bf16", None, -1, (), ()),
    ("hr_jpg_fp32", 8, True, "jpg", "fp32", None, -1, (), ()),
    ("lr_png_fp32", 8, False, "png", "fp32", None, -1, (), ()),
    ("lr_bmp_fp32", 7, False, "bmp", "fp32", 2, -1, (), ()),
    ("three_frames", 3, False, "png", "bf16", None, -1, (), ()),
    ("three_frames_windows", 3, False, "jpg", "bf16", 1, -1, (), ()),
    ("six_frames", 6, False, "png", "bf16", None, -1, (), ()),
    ("six_frames_windows", 6, True, "png", "bf16", 1, -1, (), ()),
    ("windows", 20, False, "png", "bf16", 3, -1, (), ()),
    ("windows_len", 20, False, "jpg", "bf16", 3, 13, (), ()),
    ("windows_hr_len", 20, True, "png", "bf16", 2, 9, (), ()),
    ("sixteen_and_not_png", 12, False, "png", "bf16", 3, -1, (2, 7), (4, 9)),
    ("sixteen_and_not_png_hr", 12, True, "jpg", "bf16", 2, -1, (7,), (2,)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stream_matches_serial_loop(tmp_path, case):
    name, n, hr, ext, precision, fpw, dir_len, sixteen, not_png = case
    from tecogan_b200 import config
    seq = _write_seq(str(tmp_path / "seq"), n, hr, seed=n + 31 * len(name), sixteen=sixteen, not_png=not_png)
    flags = _flags(seq, hr, dir_len)
    window = None if fpw is None else fpw * LR_FRAME_BYTES * (16 if hr else 1)
    prev = config.precision()
    try:
        _weights(precision)
        _serial(flags, str(tmp_path / "serial"), "out", ext)
        before = threading.active_count()
        _streamed(flags, str(tmp_path / "stream"), "out", ext, window)
        assert threading.active_count() == before
    finally:
        config.set_precision(prev)
    m = n if dir_len < 0 else dir_len
    # the first 5 entries of the padded sequence are not saved: a 3-frame sequence (5 entries) writes no file at all
    _same_dirs(str(tmp_path / "serial"), str(tmp_path / "stream"), m + min(5, m - 1) - 5)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_engine_u8_is_save_img_quantisation(precision):
    """out_u8, which the writer copies, is to_u8(out01), which save_img quantises."""
    from tecogan_b200 import config, kernels as K
    from tecogan_b200.engine import InferenceEngine
    prev = config.precision()
    try:
        _weights(precision)
        eng = InferenceEngine(*LR_HW, NRB)
        g = torch.Generator().manual_seed(3)
        frames = [torch.rand(*LR_HW, 3, generator=g).cuda() for _ in range(5)]
        for i, f in enumerate(frames):
            eng.step(f, next_lr=frames[i + 1] if i + 1 < len(frames) else None)
            assert torch.equal(eng.out_u8[0], K.to_u8(eng.out01[0])), i
    finally:
        config.set_precision(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("hr", [False, True], ids=["lr", "hr"])
def test_main_matches_serial_loop(tmp_path, monkeypatch, hr):
    import main as M
    from tecogan_b200 import config
    monkeypatch.chdir(str(tmp_path))
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    seq = _write_seq(str(tmp_path / "seq"), 9, hr, seed=11)
    prev = config.precision()
    try:
        before = threading.active_count()
        M.main(["--mode", "inference", "--checkpoint", "random:5", "--num_resblock", str(NRB), "--output_pre", "",
                "--output_ext", "png", "--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0"),
                "--input_dir_HR" if hr else "--input_dir_LR", seq, "--output_dir", "main"])
        assert threading.active_count() == before
        _weights("bf16")
        _serial(_flags(seq, hr), str(tmp_path / "serial"), "output", "png")
    finally:
        config.set_precision(prev)
    _same_dirs(str(tmp_path / "main"), str(tmp_path / "serial"), 9)


@pytest.mark.gpu
def test_while_train_matches_serial_loop(tmp_path, monkeypatch):
    import main as M
    from tecogan_b200 import config
    monkeypatch.chdir(str(tmp_path))
    _write_seq(str(tmp_path / "LR" / "calendar"), 12, seed=12)
    prev = config.precision()
    try:
        _weights("bf16")
        config.set_precision("fp32")                  # test_while_train restores the precision it found
        before = threading.active_count()
        fl = argparse.Namespace(output_dir=str(tmp_path / "run"), precision="bf16", num_resblock=NRB, output_ext="jpg")
        M.test_while_train(fl, 3)
        assert threading.active_count() == before
        assert config.precision() == "fp32"
        config.set_precision("bf16")
        _serial(_flags("./LR/calendar/", n=10), str(tmp_path / "serial"), "000000003", "jpg")
    finally:
        config.set_precision(prev)
    _same_dirs(str(tmp_path / "run" / "train"), str(tmp_path / "serial"), 10)


def _peak(tmp_path, n, window):
    import gc
    seq = _write_seq(str(tmp_path / ("seq%d" % n)), n, seed=5)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _streamed(_flags(seq), str(tmp_path / ("out%d" % n)), "out", "png", window)
    torch.cuda.synchronize()
    assert len(os.listdir(str(tmp_path / ("out%d" % n)))) == n
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_peak_memory_flat_in_sequence_length(tmp_path):
    from tecogan_b200 import config
    prev = config.precision()
    window = 4 * LR_FRAME_BYTES
    f32_window = 4 * LR_FRAME_BYTES * 4
    try:
        _weights("bf16")
        _peak(tmp_path, 12, window)                   # module loads, encoder and allocator warm-up
        short, long_ = _peak(tmp_path, 48, window), _peak(tmp_path, 240, window)
    finally:
        config.set_precision(prev)
    assert long_ - short < f32_window, (short, long_)


@pytest.mark.gpu
def test_undecodable_file_raises_and_joins(tmp_path):
    from tecogan_b200 import config
    seq = _write_seq(str(tmp_path / "seq"), 30, seed=6)
    with open(os.path.join(seq, "%04d.png" % 21), "wb") as f:          # frame 20 (0-based) of the sequence
        f.write(b"\x89PNG broken")
    prev = config.precision()
    try:
        _weights("bf16")
        with pytest.raises(ValueError, match="cannot decode") as serial_err:
            _serial(_flags(seq), str(tmp_path / "serial"), "out", "png")
        before = threading.active_count()
        with pytest.raises(ValueError, match="cannot decode") as stream_err:
            _streamed(_flags(seq), str(tmp_path / "stream"), "out", "png", 3 * LR_FRAME_BYTES)
        assert threading.active_count() == before
    finally:
        config.set_precision(prev)
    assert str(serial_err.value) == str(stream_err.value)
    # the documented difference: frames before the broken file may already be written
    written = sorted(os.listdir(str(tmp_path / "stream")))
    assert written == ["out_%04d.png" % k for k in range(1, len(written) + 1)] and len(written) <= 20


@pytest.mark.gpu
@pytest.mark.parametrize("ext", ["png", "bmp"])
def test_writer_exception_raises_and_joins(tmp_path, monkeypatch, ext):
    from tecogan_b200 import config
    from tecogan_b200.lib import ops
    seq = _write_seq(str(tmp_path / "seq"), 30, seed=7)
    real, calls = ops.write_image, []

    def failing(path, codec, data):
        calls.append(path)
        if len(calls) == 7:
            raise RuntimeError("disk full")
        real(path, codec, data)
    monkeypatch.setattr(ops, "write_image", failing)
    prev = config.precision()
    try:
        _weights("bf16")
        before = threading.active_count()
        with pytest.raises(RuntimeError, match="disk full"):
            _streamed(_flags(seq), str(tmp_path / "stream"), "out", ext, 3 * LR_FRAME_BYTES)
        assert threading.active_count() == before
    finally:
        config.set_precision(prev)
    assert sorted(os.listdir(str(tmp_path / "stream"))) == ["out_%04d.%s" % (k, ext) for k in range(1, 7)]
