"""CPU: the schedule of the streaming inference input (tecogan_b200.lib.dataloader.stream_inputs) -- every file decoded
once, in windows within their budget, the frames handed out in the reference's padded order with the warm-up entries
being the frames they repeat, the reader thread joined on every exit -- and the extension dispatch save_img and the
streaming writer share (lib/ops.py::image_codec, write_image)."""
import os
import threading

import cv2
import numpy as np
import pytest


def _write_seq(d, n, sizes=None, other=()):
    """n frames 0001.png .. (sizes[k] = (h, w), 8-bit unless listed as 16-bit in `other`)."""
    os.makedirs(d, exist_ok=True)
    g = np.random.default_rng(n)
    paths = []
    for k in range(n):
        h, w = sizes[k] if sizes else (6, 8)
        dt = np.uint16 if k in other else np.uint8
        p = os.path.join(d, "%04d.png" % (k + 1))
        cv2.imwrite(p, g.integers(0, np.iinfo(dt).max + 1, (h, w, 3)).astype(dt))
        paths.append(p)
    return paths


class _Recorder:
    """read_inputs(paths, down) stand-in: one marker object per file, every call recorded."""

    def __init__(self, fail_at=None):
        self.calls, self.fail_at = [], fail_at

    def __call__(self, paths, down):
        self.calls.append((list(paths), down))
        if self.fail_at is not None and self.fail_at in paths:
            raise ValueError("inference_data_loader: cannot decode " + self.fail_at)
        return [("frame", p) for p in paths]


@pytest.mark.parametrize("n", [1, 2, 3, 5, 6, 7, 20])
@pytest.mark.parametrize("frames_per_window", [1, 2, 4, 100])
def test_schedule_order_and_budget(tmp_path, monkeypatch, n, frames_per_window):
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), n)
    budget = 6 * 8 * 3 * frames_per_window
    rec = _Recorder()
    monkeypatch.setattr(DL, "read_inputs", rec)
    before = threading.active_count()
    got = list(DL.stream_inputs(paths, True, window_bytes=budget))
    assert threading.active_count() == before
    assert got == [("frame", p) for p in DL.padded(paths)]
    decoded = [p for ps, _ in rec.calls for p in ps]
    assert decoded == paths                                   # each file once, in file order
    assert all(down is True for _, down in rec.calls)
    assert all(len(ps) <= frames_per_window for ps, _ in rec.calls)
    assert [(paths.index(ps[0]), paths.index(ps[-1]) + 1) for ps, _ in rec.calls] == DL.input_windows(paths, budget)
    # the warm-up entries are the objects of frames 1..5, not copies
    k = min(5, n - 1)
    for p in range(k):
        assert got[p] is got[k + (k - p)]


def test_windows_count_16bit_and_other_files(tmp_path):
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), 4, sizes=[(6, 8), (6, 8), (4, 4), (6, 8)], other=(1,))
    other = str(tmp_path / "seq" / "0005.png")
    with open(other, "wb") as f:
        f.write(b"not a png at all, 31 bytes long")
    paths.append(other)
    cost = [144, 288, 48, 144, 31]
    assert [DL._input_cost(p) for p in paths] == cost
    for budget in (1, 144, 200, 288, 432, 10 ** 6):
        ws = DL.input_windows(paths, budget)
        assert [i for i, _ in ws] == sorted(set(i for i, _ in ws)) and ws[0][0] == 0 and ws[-1][1] == len(paths)
        assert all(b == c for (_, b), (c, _) in zip(ws, ws[1:]))
        assert all(j - i == 1 or sum(cost[i:j]) <= budget for i, j in ws)
    assert DL.input_windows(paths, 288) == [(0, 1), (1, 2), (2, 5)]


def test_windows_default_budget(tmp_path):
    from tecogan_b200 import png
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), 3)
    assert DL.input_windows(paths) == DL.input_windows(paths, png.BATCH_BYTES) == [(0, 3)]


def test_reader_runs_at_most_one_window_ahead(tmp_path, monkeypatch):
    """While the consumer holds frame k, the reader has decoded no window beyond the one after frame k's (and, during
    the warm-up, the windows up to file 5)."""
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), 16)
    rec = _Recorder()
    monkeypatch.setattr(DL, "read_inputs", rec)
    windows = DL.input_windows(paths, 6 * 8 * 3 * 2)
    window_of = {p: w for w, (i, j) in enumerate(windows) for p in paths[i:j]}
    gen = DL.stream_inputs(paths, False, window_bytes=6 * 8 * 3 * 2)
    seen = set()
    for pos, (_, p) in enumerate(gen):
        seen.add(window_of[p])
        if pos >= 10:                                         # past the warm-up and the second pass over frames 1..5
            assert len(rec.calls) <= max(seen) + 2
    assert len(rec.calls) == len(windows)


@pytest.mark.parametrize("close_at", [0, 3, 12])
def test_reader_joined_when_closed_early(tmp_path, monkeypatch, close_at):
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), 30)
    monkeypatch.setattr(DL, "read_inputs", _Recorder())
    before = threading.active_count()
    gen = DL.stream_inputs(paths, False, window_bytes=6 * 8 * 3)
    for pos, _ in enumerate(gen):
        if pos == close_at:
            break
    gen.close()
    assert threading.active_count() == before


def test_decode_error_reaches_the_consumer(tmp_path, monkeypatch):
    from tecogan_b200.lib import dataloader as DL
    paths = _write_seq(str(tmp_path / "seq"), 30)
    monkeypatch.setattr(DL, "read_inputs", _Recorder(fail_at=paths[20]))
    before = threading.active_count()
    got = []
    with pytest.raises(ValueError, match="cannot decode .*0021.png"):
        for f in DL.stream_inputs(paths, False, window_bytes=6 * 8 * 3 * 3):
            got.append(f)
    assert threading.active_count() == before
    assert got == [("frame", p) for p in DL.padded(paths)[:5 + 18]]      # frames up to the failing window


def test_inference_paths_listing_and_errors(tmp_path):
    import argparse
    from tecogan_b200.lib import dataloader as DL
    d = tmp_path / "lr"
    d.mkdir()
    for name in ("f_10.png", "f_9.png", "f_1.png", "notes.txt", "f_2.jpg"):
        (d / name).write_bytes(b"x")
    fl = lambda lr, hr, n=-1: argparse.Namespace(input_dir_LR=lr, input_dir_HR=hr, input_dir_len=n)
    paths, down = DL.inference_paths(fl(str(d), None))
    assert [os.path.basename(p) for p in paths] == ["f_1.png", "f_9.png", "f_10.png"] and down is False
    paths, down = DL.inference_paths(fl(str(tmp_path / "none"), str(d), 2))
    assert [os.path.basename(p) for p in paths] == ["f_1.png", "f_9.png"] and down is True
    with pytest.raises(ValueError, match="Input directory not found"):
        DL.inference_paths(fl(None, str(tmp_path / "none")))
    assert DL.padded(list(range(8))) == [5, 4, 3, 2, 1, 0, 1, 2, 3, 4, 5, 6, 7]
    assert DL.padded([0, 1, 2]) == [2, 1, 0, 1, 2]


# ------------------------------------------------------------------------------------------ extension dispatch
def test_image_codec_routes():
    from tecogan_b200.lib.ops import image_codec
    assert image_codec("a/b.png", 10, 10) == "png"
    assert image_codec("a/b.PNG", 70000, 10) == "png"
    for ext in ("jpg", "JPG", "jpeg", "Jpeg", "jpe"):
        assert image_codec("b." + ext, 65500, 65500) == "jpeg", ext
        assert image_codec("b." + ext, 65501, 10) == "cv2", ext
        assert image_codec("b." + ext, 10, 65501) == "cv2", ext
    for ext in ("bmp", "tif", "webp", "ppm", "png.bmp", "jpgx"):
        assert image_codec("b." + ext, 10, 10) == "cv2", ext
    assert image_codec("b.png", 10, 10, on_device=False) == "cv2"
    assert image_codec("b.jpg", 10, 10, on_device=False) == "cv2"


def test_write_image(tmp_path):
    from tecogan_b200.lib.ops import save_img, write_image
    write_image(str(tmp_path / "a.png"), "png", b"bytes")
    assert (tmp_path / "a.png").read_bytes() == b"bytes"
    write_image(str(tmp_path / "missing" / "a.png"), "png", b"bytes")        # ignored
    write_image(str(tmp_path / "missing" / "a.jpg"), "jpeg", b"bytes")
    assert not (tmp_path / "missing").exists()
    rgb = np.random.default_rng(1).integers(0, 256, (5, 7, 3)).astype(np.uint8)
    write_image(str(tmp_path / "b.bmp"), "cv2", rgb)
    assert np.array_equal(cv2.imread(str(tmp_path / "b.bmp"), cv2.IMREAD_UNCHANGED)[:, :, ::-1], rgb)
    # save_img of a host image goes through the same cv2 branch
    img = np.random.default_rng(2).random((5, 7, 3))
    save_img(str(tmp_path / "c.png"), img)
    want = np.clip(img * 255.0, 0, 255).astype(np.uint8)
    assert np.array_equal(cv2.imread(str(tmp_path / "c.png"), cv2.IMREAD_UNCHANGED)[:, :, ::-1], want)
