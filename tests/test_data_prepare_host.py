"""CPU: the training-data preparation without a device.  The numpy restatement of cv2.resize(fx=fy=0.5, INTER_AREA)
(tests/golden/area_oracle.py), which teco_area_half_u8 is held to, equals cv2 bit for bit on every size 2..40 x 2..40 and
on frame sizes of the source videos; dataPrepare.py's flags are the reference's; prepare() numbers the scenes, skips
missing, unreadable and small videos, writes nothing under --TEST and removes only the sources it processed (the device
stage replaced by a recorder); the log file is named as the reference names it."""
import datetime
import os

import cv2
import numpy as np
import pytest

import dataPrepare
from tecogan_b200 import data_prepare as D
from tests.golden import area_oracle as A

LARGE = [(721, 1281), (720, 1281), (1080, 1920), (2160, 4096), (1081, 1919)]


def _cv2(frame):
    return cv2.resize(frame, (0, 0), fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)


def _check(frame):
    want, got = _cv2(frame), A.area_half(frame)
    assert got.shape == want.shape and got.dtype == np.uint8, (frame.shape, got.shape, want.shape)
    assert np.array_equal(got, want), frame.shape


def test_out_size_rounds_half_to_even():
    assert [A.out_size(n) for n in (2, 3, 5, 7, 721, 1080, 1081, 1919)] == [1, 2, 2, 4, 360, 540, 540, 960]
    for n in range(2, 200):
        assert A.out_size(n) == _cv2(np.zeros((2, n, 3), np.uint8)).shape[1]


@pytest.mark.parametrize("H", range(2, 41))
def test_oracle_equals_cv2_small(H):
    g = np.random.default_rng(H)
    for W in range(2, 41):
        _check(g.integers(0, 256, (H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("H,W", LARGE)
def test_oracle_equals_cv2_large(H, W):
    _check(np.random.default_rng(H * W).integers(0, 256, (H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("v", [0, 1, 2, 127, 254, 255])
def test_oracle_equals_cv2_constant(v):
    for H, W in [(2, 2), (3, 3), (7, 11), (40, 39)] + LARGE:
        _check(np.full((H, W, 3), v, np.uint8))


def test_oracle_refuses_bad_frames():
    for f in (np.zeros((1, 8, 3), np.uint8), np.zeros((8, 1, 3), np.uint8), np.zeros((8, 8, 3), np.uint16),
              np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8), np.uint8)):
        with pytest.raises(ValueError):
            A.area_half(f)


def test_flags_are_the_reference_s():
    f = dataPrepare.parse_flags([])
    assert (f.start_id, f.duration, f.disk_path, f.REMOVE, f.TEST, f.threads) == (
        2000, 120, "/mnt/netdisk/data/video/", False, False, 4)
    assert f.summary_dir == os.path.join("/mnt/netdisk/data/video/", "log/")
    assert list(vars(f)) == ["start_id", "duration", "disk_path", "summary_dir", "REMOVE", "TEST", "threads"]
    f = dataPrepare.parse_flags(["--start_id", "7", "--duration", "3", "--disk_path", "/x", "--summary_dir", "/y",
                                 "--REMOVE", "--TEST", "--threads", "2"])
    assert (f.start_id, f.duration, f.disk_path, f.summary_dir, f.REMOVE, f.TEST, f.threads) == (
        7, 3, "/x", "/y", True, True, 2)


def test_table_is_the_reference_s():
    assert len(D.VIDEOS) == 28
    assert sum(len(v) for v in D.VIDEOS.values()) == 308
    assert list(D.VIDEOS)[0] == "121649159" and list(D.VIDEOS)[-1] == "89936769"


def test_log_file_name():
    t = datetime.datetime(2026, 3, 4, 5, 6)
    assert dataPrepare.log_path("/s/log/", t) == "/s/log/logfile_03040506.txt"
    assert dataPrepare.log_path("/s/log", t) == "/s/log/logfile_03040506.txt"


def _video(path, w, h, n=3):
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 25, (w, h))
    assert vw.isOpened()
    for i in range(n):
        vw.write(np.full((h, w, 3), 10 * i, np.uint8))
    vw.release()


@pytest.fixture
def disk(tmp_path):
    """Sources: 11 valid (400x400), 22 missing, 33 unreadable, 44 small (320x480), 55 valid (480x400), 66 twice."""
    d = str(tmp_path)
    _video(os.path.join(d, "11.avi"), 400, 400)
    with open(os.path.join(d, "33.mp4"), "wb") as f:
        f.write(b"not a video")
    _video(os.path.join(d, "44.avi"), 320, 480)
    _video(os.path.join(d, "55.avi"), 480, 400)
    _video(os.path.join(d, "66.avi"), 480, 400)
    _video(os.path.join(d, "66.mkv"), 480, 400)
    return d


TABLE = {"11": [0, 5], "22": [1], "33": [2, 3], "44": [4], "55": [6, 7, 8], "66": [9]}


def _tree(d):
    return sorted(os.path.relpath(os.path.join(r, n), d) for r, ds, fs in os.walk(d) for n in ds + fs)


def _recorder(monkeypatch):
    calls = []
    monkeypatch.setattr(D, "cuda_device", lambda device=None: "cuda:0")
    monkeypatch.setattr(D, "prepare_video", lambda path, scenes, duration, device, stop=None:
                        calls.append((os.path.basename(path), [(os.path.basename(os.path.dirname(t)), s)
                                                               for t, s in scenes], duration)))
    return calls


def test_scene_numbering_and_skips(disk, capsys, monkeypatch):
    calls = _recorder(monkeypatch)
    assert D.prepare(TABLE, disk, 100, 12) == 2
    out = capsys.readouterr().out.splitlines()
    assert out[0] == "Try loading 10x12."
    assert "Skipped invalid link or other error:https://vimeo.com/22" in out
    assert "Skipped invalid link or other error:https://vimeo.com/33" in out
    assert "Skipped videos of small size 320x480" in out
    assert "Skipped invalid link or other error:https://vimeo.com/66" in out
    assert out[-1] == "Done: get 5 valid folders with 12 frames from 2 videos."
    folders = [l for l in out if l.startswith("folder ")]
    assert folders[0] == "folder %s: 12x[400,400]//2 at frame 0 of %s" % (
        os.path.join(disk, "scene_0100/"), os.path.join(disk, "11.avi"))
    assert calls == [("11.avi", [("scene_0100", 0), ("scene_0101", 5)], 12),
                     ("55.avi", [("scene_0102", 6), ("scene_0103", 7), ("scene_0104", 8)], 12)]
    assert all(os.path.isdir(os.path.join(disk, "scene_%04d" % k)) for k in range(100, 105))
    assert not os.path.exists(os.path.join(disk, "scene_0105"))


def test_test_mode_writes_nothing(disk, capsys, monkeypatch):
    calls = _recorder(monkeypatch)
    before = _tree(disk)
    assert D.prepare(TABLE, disk, 100, 12, save_frames=False, remove=True) == 2
    assert _tree(disk) == before and calls == []
    out = capsys.readouterr().out.splitlines()
    assert len([l for l in out if l.startswith("folder ")]) == 5
    assert out[-1] == "Done: get 5 valid folders with 12 frames from 2 videos."


def test_remove_deletes_only_processed_sources(disk, capsys, monkeypatch):
    calls = _recorder(monkeypatch)
    D.prepare(TABLE, disk, 0, 4, remove=True)
    assert len(calls) == 2
    left = set(os.listdir(disk))
    assert {"11.avi", "55.avi"}.isdisjoint(left)
    assert {"33.mp4", "44.avi", "66.avi", "66.mkv"} <= left
    out = capsys.readouterr().out.splitlines()
    assert ["remove  " + os.path.join(disk, n) for n in ("11.avi", "55.avi")] == [l for l in out if l.startswith("remove")]


def test_worker_error_is_raised(disk, monkeypatch):
    monkeypatch.setattr(D, "cuda_device", lambda device=None: "cuda:0")

    def fail(path, scenes, duration, device, stop=None):
        raise OSError("disk full")
    monkeypatch.setattr(D, "prepare_video", fail)
    with pytest.raises(OSError, match="disk full"):
        D.prepare(TABLE, disk, 0, 4, remove=True)
    assert {"11.avi", "55.avi"} <= set(os.listdir(disk))


def test_command_test_mode_writes_only_its_log(disk, capsys):
    before = _tree(disk)
    dataPrepare.main(["--disk_path", disk, "--duration", "12", "--TEST"], videos=TABLE)
    after = _tree(disk)
    new = sorted(set(after) - set(before))
    assert len(new) == 2 and new[0] == "log" and new[1].startswith(os.path.join("log", "logfile_"))
    with open(os.path.join(disk, new[1])) as f:
        log = f.read().splitlines()
    assert log[0] == "[Configurations]:" and "\tTEST: True" in log and log[8] == "End of configuration"
    assert log[-1] == "Done: get 5 valid folders with 12 frames from 2 videos."
    assert capsys.readouterr().out.splitlines() == log
