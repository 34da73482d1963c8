"""CPU: `dataPrepare.py --scene_threshold` without a device.  The window rule over score lists; the scores from SADs; the
video listing; the flag, absent unless given and refused before anything runs when bad; the printed table; scan()'s
lines, skips and table with the device pass (scan_video) replaced by given SADs; prepare() on scanned sources, which
prints their paths and reads them in sequence; and sequential reading, which gives the frames seeking gives."""
import os

import cv2
import numpy as np
import pytest

import dataPrepare
from tecogan_b200 import data_prepare as D

T = 10.0
UNDER = float(np.nextafter(T, 0.0))


# ---- the window rule -------------------------------------------------------------------------------------------------

def _scores(n, cuts, value=50.0):
    s = [0.0] * n
    for i in cuts:
        s[i] = value
    return s


def test_no_cut():
    assert D.scene_starts(_scores(20, []), T, 6) == [0, 6, 12]
    assert D.scene_starts(_scores(18, []), T, 6) == [0, 6, 12]
    assert D.scene_starts(_scores(17, []), T, 6) == [0, 6]
    assert D.scene_starts(_scores(5, []), T, 6) == []
    assert D.scene_starts([], T, 6) == []
    assert D.scene_starts(_scores(3, []), T, 1) == [0, 1, 2]


def test_cut_at_frame_1():
    assert D.scene_starts(_scores(13, [1]), T, 6) == [1, 7]
    assert D.scene_starts(_scores(13, [1]), T, 1)[:2] == [0, 1]


def test_frame_0_is_not_read():
    assert D.scene_starts([100.0] + [0.0] * 11, T, 6) == [0, 6]


def test_threshold_is_inclusive():
    assert D.scene_starts(_scores(20, [8], T), T, 4) == [0, 4, 8, 12, 16]
    assert D.scene_starts(_scores(20, [8], UNDER), T, 4) == [0, 4, 8, 12, 16]
    assert D.scene_starts(_scores(20, [7], T), T, 4) == [0, 7, 11, 15]             # a cut: frames 4..6 dropped
    assert D.scene_starts(_scores(20, [7], UNDER), T, 4) == [0, 4, 8, 12, 16]      # not a cut


@pytest.mark.parametrize("D_", [1, 2, 5, 8])
def test_shots_of_d_minus_1_d_and_2d_plus_1(D_):
    lens = [D_ - 1, D_, 2 * D_ + 1]
    cuts = [lens[0], lens[0] + lens[1]]
    n = sum(lens)
    got = D.scene_starts(_scores(n, [c for c in cuts if c > 0]), T, D_)
    want = [cuts[0]] + [cuts[1], cuts[1] + D_]
    if D_ == 1:                                  # a shot of 0 frames: frame 0 starts the 1-frame shot
        want = [0, 1, 2, 3]
    assert got == want


def test_several_cuts():
    s = _scores(40, [3, 10, 11, 25, 39])
    # shots [0, 3) [3, 10) [10, 11) [11, 25) [25, 39) [39, 40)
    assert D.scene_starts(s, T, 4) == [3, 11, 15, 19, 25, 29, 33]


def test_duration_below_1_raises():
    with pytest.raises(ValueError):
        D.scene_starts(_scores(5, []), T, 0)


def test_scores_follow_main_s_rule():
    """values = 3: a SAD of 765 is a mafd of 100.  Frame 1 scores min(100, |100 - 0|), frame 2 min(100, 0)."""
    assert D.frame_scores([0, 765, 765, 0, 0], 3) == [0.0, 100.0, 0.0, 0.0, 0.0]
    assert D.frame_scores([0, 153, 765], 3) == [0.0, 20.0, 80.0]
    assert D.frame_scores([], 0) == []


# ---- the listing -----------------------------------------------------------------------------------------------------

def _touch(path):
    with open(path, "wb") as f:
        f.write(b"x")


def test_listing(tmp_path):
    d = str(tmp_path)
    for n in ["b.MP4", "a.avi", "A.mkv", "c.Ts", "c.webm", "d.txt", "e", "f.mpeg", "g.m4v", "h.MOV", "i.mpg", "j.ts",
              "k.tar.mkv"]:
        _touch(os.path.join(d, n))
    os.makedirs(os.path.join(d, "scene_0000"))
    os.makedirs(os.path.join(d, "log"))
    os.makedirs(os.path.join(d, "dir.mp4"))                      # a directory, whatever its name
    _touch(os.path.join(d, "scene_0000", "z.mp4"))               # not recursed into
    got = D.list_sources(d)
    j = lambda *ns: [os.path.join(d, n) for n in ns]             # noqa: E731
    assert got == [("A", j("A.mkv")), ("a", j("a.avi")), ("b", j("b.MP4")), ("c", j("c.Ts", "c.webm")),
                   ("f", j("f.mpeg")), ("g", j("g.m4v")), ("h", j("h.MOV")), ("i", j("i.mpg")), ("j", j("j.ts")),
                   ("k.tar", j("k.tar.mkv"))]


def test_listing_is_in_file_name_order(tmp_path):
    d = str(tmp_path)
    for n in ["a.mp4", "a-b.mp4", "a_c.mkv", "B.avi"]:
        _touch(os.path.join(d, n))
    assert [s for s, _ in D.list_sources(d)] == ["B", "a-b", "a", "a_c"]


# ---- the flag --------------------------------------------------------------------------------------------------------

def test_flag_absent_unless_given():
    assert not hasattr(dataPrepare.parse_flags([]), "scene_threshold")
    f = dataPrepare.parse_flags(["--scene_threshold", "12.5", "--TEST"])
    assert f.scene_threshold == "12.5"
    assert list(vars(f)) == ["start_id", "duration", "disk_path", "summary_dir", "REMOVE", "TEST", "threads",
                             "scene_threshold"]


@pytest.mark.parametrize("argv", [["--scene_threshold", v] for v in ("0", "-1", "100.01", "nan", "inf", "ten", "")]
                         + [["--scene_threshold", "10", "--duration", "0"]])
def test_bad_flag_refused_before_anything_runs(tmp_path, monkeypatch, argv):
    def fail(*a, **k):
        raise AssertionError("ran")
    for name in ("scan", "prepare", "video_size", "list_sources", "cuda_device"):
        monkeypatch.setattr(D, name, fail)
    disk = str(tmp_path / "disk")
    with pytest.raises(ValueError):
        dataPrepare.main(["--disk_path", disk] + argv)
    assert not os.path.exists(disk)


def test_table_format():
    assert D.format_table({"a": [0, 120], "b c": [7], 'q"': [1, 2, 3]}) == "\n".join([
        "video_data_dict = {", '    "a" : [0, 120],', '    "b c" : [7],', '    "q\\"" : [1, 2, 3],', "}"])
    assert D.format_table({}) == "video_data_dict = {\n}"
    table = {"x": [0, 5], "y": [9]}
    text = D.format_table(table)
    assert eval(text.split("=", 1)[1]) == table                 # noqa: S307 -- pasted back, it is the same table


# ---- scan() with given SADs ------------------------------------------------------------------------------------------

def _video(path, w, h, n=3):
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 25, (w, h))
    assert vw.isOpened()
    for i in range(n):
        vw.write(np.full((h, w, 3), 10 * i, np.uint8))
    vw.release()


VALUES = 3                                       # every fake SAD below is over 3 values: 765 is a mafd of 100


@pytest.fixture
def disk(tmp_path):
    """a: 20 frames, a cut at 7; b: 5 frames (no scene); bad.mp4 unreadable; c: 12 frames; dup twice; small 320x480."""
    d = str(tmp_path)
    _video(os.path.join(d, "a.avi"), 400, 400)
    _video(os.path.join(d, "b.avi"), 480, 400)
    with open(os.path.join(d, "bad.mp4"), "wb") as f:
        f.write(b"not a video")
    _video(os.path.join(d, "c.AVI"), 400, 416)
    _video(os.path.join(d, "dup.avi"), 400, 400)
    _video(os.path.join(d, "dup.mkv"), 400, 400)
    _video(os.path.join(d, "small.avi"), 320, 480)
    _touch(os.path.join(d, "notes.txt"))
    return d


SADS = {"a.avi": [0] * 7 + [765] + [0] * 12, "b.avi": [0] * 5, "c.AVI": [0] * 12}


def _fake_scan(monkeypatch, seen=None):
    monkeypatch.setattr(D, "cuda_device", lambda device=None: "cuda:0")

    def scan_video(path, device, stop=None):
        if seen is not None:
            seen.append(os.path.basename(path))
        return SADS[os.path.basename(path)], VALUES
    monkeypatch.setattr(D, "scan_video", scan_video)


@pytest.mark.parametrize("threads", [1, 3])
def test_scan_lines_and_table(disk, capsys, monkeypatch, threads):
    seen = []
    _fake_scan(monkeypatch, seen)
    table, sources = D.scan(disk, T, 6, threads=threads)
    assert sorted(seen) == ["a.avi", "b.avi", "c.AVI"]
    assert table == {"a": [0, 7, 13], "c": [0, 6]} and list(table) == ["a", "c"]
    assert sources == {"a": os.path.join(disk, "a.avi"), "c": os.path.join(disk, "c.AVI")}
    p = lambda n: os.path.join(disk, n)                          # noqa: E731
    assert capsys.readouterr().out.splitlines() == [
        p("a.avi") + ": 20 frames", "scene cut before frame 7, score 100.0000", "3 scenes of 6 frames",
        p("b.avi") + ": 5 frames", "0 scenes of 6 frames",
        p("bad.mp4"), "Skipped invalid link or other error:" + p("bad.mp4"),
        p("c.AVI") + ": 12 frames", "2 scenes of 6 frames",
        "Skipped %s, %s: 2 files share the name dup" % (p("dup.avi"), p("dup.mkv")),
        p("small.avi"), "Skipped videos of small size 320x480",
        "video_data_dict = {", '    "a" : [0, 7, 13],', '    "c" : [0, 6],', "}"]


def test_scan_without_videos_needs_no_device(tmp_path, capsys, monkeypatch):
    def fail(device=None):
        raise RuntimeError("no device")
    monkeypatch.setattr(D, "cuda_device", fail)
    assert D.scan(str(tmp_path), T, 6) == ({}, {})
    assert capsys.readouterr().out.splitlines() == ["video_data_dict = {", "}"]


def test_scan_worker_error_is_raised(disk, monkeypatch):
    import threading
    monkeypatch.setattr(D, "cuda_device", lambda device=None: "cuda:0")

    def scan_video(path, device, stop=None):
        if path.endswith("b.avi"):
            raise RuntimeError("decode failed")
        return SADS[os.path.basename(path)], VALUES
    monkeypatch.setattr(D, "scan_video", scan_video)
    with pytest.raises(RuntimeError, match="decode failed"):
        D.scan(disk, T, 6, threads=2)
    assert not [t.name for t in threading.enumerate() if t.name.startswith("dataPrepare")]


# ---- prepare() on scanned sources ------------------------------------------------------------------------------------

def _recorder(monkeypatch):
    calls = []
    monkeypatch.setattr(D, "cuda_device", lambda device=None: "cuda:0")
    monkeypatch.setattr(D, "prepare_video", lambda path, scenes, duration, device, stop=None, seek=True:
                        calls.append((os.path.basename(path), [(os.path.basename(os.path.dirname(t)), s)
                                                               for t, s in scenes], duration, seek)))
    return calls


def test_prepare_scanned_sources(disk, capsys, monkeypatch):
    calls = _recorder(monkeypatch)
    sources = {"a": os.path.join(disk, "a.avi"), "c": os.path.join(disk, "c.AVI")}
    assert D.prepare({"a": [0, 7, 13], "c": [0, 6]}, disk, 40, 6, remove=True, sources=sources) == 2
    assert calls == [("a.avi", [("scene_0040", 0), ("scene_0041", 7), ("scene_0042", 13)], 6, False),
                     ("c.AVI", [("scene_0043", 0), ("scene_0044", 6)], 6, False)]
    out = capsys.readouterr().out.splitlines()
    assert out[0] == "Try loading 5x6." and out[1] == sources["a"]
    assert out[2] == "folder %s: 6x[400,400]//2 at frame 0 of %s" % (os.path.join(disk, "scene_0040/"), sources["a"])
    assert sources["c"] in out and not [l for l in out if "vimeo" in l]
    assert [l for l in out if l.startswith("remove")] == ["remove  " + sources["a"], "remove  " + sources["c"]]
    assert out[-1] == "Done: get 5 valid folders with 6 frames from 2 videos."
    left = set(os.listdir(disk))
    assert {"a.avi", "c.AVI"}.isdisjoint(left) and {"b.avi", "bad.mp4", "dup.avi", "small.avi"} <= left


def test_command_test_mode_with_the_flag(disk, capsys, monkeypatch):
    _fake_scan(monkeypatch)
    calls = _recorder(monkeypatch)
    before = sorted(os.listdir(disk))
    dataPrepare.main(["--disk_path", disk, "--duration", "6", "--TEST", "--scene_threshold", "10", "--start_id", "3"])
    assert calls == []
    assert sorted(os.listdir(disk)) == sorted(before + ["log"])
    logs = os.listdir(os.path.join(disk, "log"))
    with open(os.path.join(disk, "log", logs[0])) as f:
        log = f.read().splitlines()
    assert "\tscene_threshold: 10.0" in log
    assert '    "a" : [0, 7, 13],' in log
    assert "folder %s: 6x[400,416]//2 at frame 6 of %s" % (os.path.join(disk, "scene_0007/"),
                                                           os.path.join(disk, "c.AVI")) in log
    assert log[-1] == "Done: get 5 valid folders with 6 frames from 2 videos."
    assert capsys.readouterr().out.splitlines() == log


# ---- reading in sequence ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def counting_video(tmp_path_factory):
    """30 MJPG frames, each different (every frame is a keyframe: seeking is exact)."""
    path = str(tmp_path_factory.mktemp("seq") / "v.avi")
    g = np.random.default_rng(3)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 25, (64, 48))
    for i in range(30):
        vw.write(g.integers(0, 256, (48, 64, 3)).astype(np.uint8))
    vw.release()
    return path


def test_reading_in_sequence_gives_the_seeked_frames(counting_video):
    starts = [0, 4, 11, 20]
    seq = list(D.scene_frames(counting_video, starts, 4, seek=False))
    sought = list(D.scene_frames(counting_video, starts, 4))
    assert [(k, i) for k, i, _ in seq] == [(k, i) for k in range(4) for i in range(4)]
    assert all(np.array_equal(a[2], b[2]) for a, b in zip(seq, sought)) and len(seq) == 16


def test_reading_in_sequence_refuses_overlaps_and_runs_out(counting_video):
    with pytest.raises(ValueError):
        list(D.scene_frames(counting_video, [0, 3], 4, seek=False))
    with pytest.raises(RuntimeError, match="cannot read frame 30"):
        list(D.scene_frames(counting_video, [27], 4, seek=False))
    with pytest.raises(RuntimeError, match="cannot read frame 30"):
        list(D.scene_frames(counting_video, [40], 4, seek=False))
