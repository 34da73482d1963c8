"""Host side of `main.py --scene_threshold`: the score and cut rule restated in numpy float64 and worked by hand, the
scene order (lib/dataloader.py::scene_order) against the reference's padded order on every cut set of short streams,
the step driver (scene_steps) and the y4m reader's scene stream on host frames, and the flag."""
import itertools
import os
import threading

import numpy as np
import pytest
import torch

from tecogan_b200 import y4m
from tecogan_b200.lib.dataloader import (DeviceHandoff, padded, scene_order, scene_score, scene_steps,
                                         scene_threshold)


def q8(x):
    """q(x) = clamp(rint(float32(255 x)), 0, 255), half-even."""
    return np.clip(np.rint(np.float32(255.0) * np.asarray(x, np.float32)), 0, 255).astype(np.int64)


def sad(a, b):
    return int(np.abs(q8(a) - q8(b)).sum())


def scores(frames):
    """score_i of every frame (score_0 = 0): mafd_i = 100 SAD_i / (3 h w 255), score_i = min(mafd_i, |mafd_i - mafd_{i-1}|)
    with mafd_0 = 0, in float64."""
    out, prev = [0.0], 0.0
    for a, b in zip(frames, frames[1:]):
        mafd = np.float64(100.0) * np.float64(sad(a, b)) / np.float64(b.size * 255)
        out.append(float(min(mafd, abs(mafd - prev))))
        prev = mafd
    return out


def cuts(frames, t):
    return [i for i, s in enumerate(scores(frames)) if i > 0 and s >= t]


def flat(v, hw=(4, 5)):
    """A frame whose every value is the byte v, as the readers make it (u / 255 in float32)."""
    return np.full(hw + (3,), np.float32(v) / np.float32(255.0), np.float32)


# ---- the score -------------------------------------------------------------------------------------------------------

def test_q8_recovers_every_byte_and_clamps():
    u = np.arange(256)
    assert np.array_equal(q8(u.astype(np.float32) / np.float32(255.0)), u)
    u16 = np.array([0, 127, 128, 65535], np.float32) / np.float32(255.0)      # 16-bit sources: /255, up to 257
    assert q8(u16).tolist() == [0, 127, 128, 255]
    assert q8([-0.5, -1e-9, 1.0000001, 3.0]).tolist() == [0, 0, 255, 255]
    assert q8(np.array([0.5, 1.5, 2.5], np.float32) / np.float32(255.0)).tolist() == [0, 2, 2]   # half-even


def test_identical_frames_score_zero():
    f = [flat(90)] * 5
    assert scores(f) == [0.0] * 5 and cuts(f, 1e-9) == []


def test_full_scale_flip_scores_100():
    f = [flat(0), flat(255), flat(0)]
    assert scores(f) == [0.0, 100.0, 0.0]          # frame 2: mafd 100, unchanged from frame 1, so its score is 0
    assert cuts(f, 100) == [1]                     # T equal to the score is a cut (>=)


def test_frame_one_compares_with_mafd_zero():
    f = [flat(0), flat(51)]                        # SAD = 60 * 51: mafd = 100 * 51 / 255 = 20 exactly
    assert scores(f) == [0.0, 20.0]
    assert cuts(f, 20) == [1] and cuts(f, 20.000001) == []


def test_sustained_pan_stays_below_the_diff_term():
    """Every frame differs from the last by mafd 20, above T = 10; the change of mafd is 0, so only frame 1 (compared
    with mafd_0 = 0) scores 20."""
    f = [flat(v) for v in (0, 51, 102, 153, 204, 255)]
    assert scores(f) == [0.0, 20.0, 0.0, 0.0, 0.0, 0.0]
    assert cuts(f, 10) == [1]
    g = np.random.default_rng(3)                   # a real pan: a textured frame moving one pixel a frame
    tex = g.integers(0, 256, (6, 40, 3))
    pan = [tex[:, k:k + 30].astype(np.float32) / np.float32(255.0) for k in range(8)]
    s = scores(pan)
    assert min(s[2:]) >= 0.0 and max(s[2:]) < 5.0 < s[1]


def test_cut_inside_a_pan():
    """A pan of mafd 5 (below T = 10), a jump to mafd 80 at frame 4 (score min(80, 75) = 75), then the pan again: frame
    5 scores min(5, 75) = 5, not a cut."""
    def frame(level, jump):
        x = np.zeros((1, 20, 3), np.float32)
        x[:, :5] = np.float32(level) / np.float32(255.0)       # 15 of 60 values move by 51: mafd 100 * 765 / 15300 = 5
        if jump:
            x[:, 5:] = np.float32(1.0)                         # and 45 values by 255 at the cut
        return x
    seq = [frame(0, False), frame(51, False), frame(102, False), frame(153, False), frame(204, True), frame(255, True),
           frame(204, True)]
    s = scores(seq)
    assert s[1:4] == [5.0, 0.0, 0.0]
    assert s[4] == 75.0                              # SAD 15 * 51 + 45 * 255 = 12240: mafd 80, change 75
    assert s[5] == 5.0 and s[6] == 0.0
    assert cuts(seq, 10) == [4]


def test_package_score_is_the_restatement():
    g = np.random.default_rng(8)
    prev = 0.0
    for _ in range(200):
        values = int(g.integers(1, 1 << 24)) * 3
        s = int(g.integers(0, values * 255 + 1))
        want = 100.0 * s / (values * 255)
        assert scene_score(s, values, prev) == (want, min(want, abs(want - prev)))
        prev = want


# ---- the order -------------------------------------------------------------------------------------------------------

def test_no_cut_is_the_padded_order():
    for n in range(6, 30):
        steps = list(scene_order((k, False) for k in range(n)))
        assert [k for k, _, _ in steps] == padded(list(range(n)))
        assert [w for _, w, _ in steps] == [p >= 5 for p in range(len(steps))]
        assert [r for _, _, r in steps] == [p == 0 for p in range(len(steps))]


def _want(n, cut_set):
    """Each scene as the reference runs a sequence: padded(scene), the first m entries not written, reset first."""
    starts = [0] + sorted(cut_set)
    out = []
    for a, b in zip(starts, starts[1:] + [n]):
        scene = list(range(a, b))
        m = min(5, len(scene) - 1)
        out += [(k, p >= m, p == 0) for p, k in enumerate(padded(scene))]
    return out


def test_every_cut_set_up_to_14_frames():
    for n in range(1, 15):
        for bits in range(1 << max(n - 1, 0)):
            cut_set = {k for k in range(1, n) if bits >> (k - 1) & 1}
            pulled = []

            def pairs():
                for k in range(n):
                    pulled.append(k)
                    yield k, k in cut_set or k == 0 and bool(bits & 1)      # frame 0's flag is ignored
            starts = [0] + sorted(cut_set)
            scene_of = {k: max(s for s in starts if s <= k) for k in range(n)}
            steps = []
            for k, write, reset in scene_order(pairs()):
                c = scene_of[k]
                # read lazily: six frames past the scene's first, or one past this step
                assert len(pulled) <= max(c + 6, k + 2), (n, cut_set, k, len(pulled))
                steps.append((k, write, reset))
            assert steps == _want(n, cut_set), (n, cut_set)
            assert [k for k, w, _ in steps if w] == list(range(n))                      # each frame written once, in order
            for p, (k, write, reset) in enumerate(steps):
                c = scene_of[k]
                assert reset == (p == 0 or scene_of[steps[p - 1][0]] != c)        # reset before each scene's first step
                if not write:
                    L = sum(1 for j in range(n) if scene_of[j] == c)
                    assert c < k <= c + min(5, L - 1)
                if p + 1 < len(steps) and not steps[p + 1][2]:
                    assert scene_of[steps[p + 1][0]] == c           # the look-ahead never spans a boundary
            firsts = [p for p, s in enumerate(steps) if s[2]]
            assert len(firsts) == len(starts)


def test_warm_up_order_inside_each_scene():
    steps = list(scene_order((k, k in (9, 12)) for k in range(19)))
    assert [k for k, _, _ in steps] == padded(list(range(9))) + padded([9, 10, 11]) + padded(list(range(12, 19)))
    assert [k for k, w, _ in steps if not w] == [5, 4, 3, 2, 1, 11, 10, 17, 16, 15, 14, 13]
    assert [p for p, s in enumerate(steps) if s[2]] == [0, 14, 19]


# ---- the step driver, on host frames ---------------------------------------------------------------------------------

class HostFeed:
    """DeviceHandoff's consumer interface over host frames, recording what is held."""

    def __init__(self, frames, sads):
        self.frames, self.sads = frames, sads
        self.held, self.peak, self.released = set(), 0, []

    def take(self, k):
        if k >= len(self.frames):
            return None
        self.held.add(k)
        self.peak = max(self.peak, len(self.held))
        return self.frames[k]

    def value(self, k):
        assert k in self.held
        return self.sads[k]

    def drop(self, k):
        self.held.remove(k)


def _sads(frames):
    return [0] + [sad(a, b) for a, b in zip(frames, frames[1:])]


def _scene_frames(lengths, hw=(2, 3)):
    """Scenes of flat frames: within a scene each frame moves by 1 (mafd 0.39), between scenes by 128 (mafd 50)."""
    frames, v = [], 0
    for L in lengths:
        for k in range(L):
            frames.append(torch.from_numpy(flat(v + k, hw)))
        v = (v + 128) % 200
    return frames


def test_scene_steps_find_the_cuts_and_drop_each_frame_once():
    frames = _scene_frames([9, 3, 7])
    feed = HostFeed(frames, _sads([f.numpy() for f in frames]))
    steps = list(scene_steps(feed, 10.0, feed.released.append))
    assert [(s.index, s.write, s.reset) for s in steps] == _want(19, {9, 12})
    want = scores([f.numpy() for f in frames])
    assert [(s.start, s.score) for s in steps[1:] if s.reset] == [(9, want[9]), (12, want[12])]
    assert want[9] > 10 and want[12] > 10 and max(want[1:9] + want[10:12] + want[13:]) < 1
    assert steps[0].start == 0 and steps[0].score is None
    assert all(s.frame is frames[s.index] for s in steps)
    assert feed.released == list(range(19)) and not feed.held
    assert feed.peak <= 7                          # a scene's frames c .. c+5 and the step before it at most


def test_scene_steps_hold_a_bounded_number_of_frames():
    frames = _scene_frames([4] * 40)
    feed = HostFeed(frames, _sads([f.numpy() for f in frames]))
    steps = list(scene_steps(feed, 10.0, feed.released.append))
    assert sum(s.reset for s in steps) == 40 and sum(s.write for s in steps) == 160
    assert feed.peak <= 7


@pytest.mark.parametrize("lengths", [[9, 3, 7], [1, 1, 2], [2], [6, 1, 6]])
def test_y4m_scene_stream_on_host_frames(tmp_path, lengths):
    """Y4MReader.scenes() drives the reader thread through DeviceHandoff with READ_CREDITS frames: every frame is read
    once, written once in order, and the thread is joined.  The device conversion is replaced by host frames and their
    SADs."""
    frames = _scene_frames(lengths)
    n = len(frames)
    p = str(tmp_path / "a.y4m")
    with open(p, "wb") as f:
        f.write(y4m.format_header(8, 8) + b"".join(b"FRAME\n" + bytes([k]) * 96 for k in range(n)))
    r = y4m.Y4MReader(p)
    sads = _sads([f.numpy() for f in frames])
    read = []

    def chunks(scores=False):
        assert scores
        buf = np.empty(96, np.uint8)
        for k in itertools.count():
            if not y4m.read_frame(r.f, buf, k):
                return
            read.append(k)
            yield k, [frames[int(buf[0])]], torch.tensor([sads[k]])
    r._chunks = chunks
    before = threading.active_count()
    steps = list(r.scenes(10.0))
    assert threading.active_count() == before and read == list(range(n))
    starts = list(itertools.accumulate([0] + lengths[:-1]))
    assert [(s.index, s.write, s.reset) for s in steps] == _want(n, set(starts[1:]))
    assert [r.name(s.index) for s in steps if s.write] == ["%04d" % (k + 1) for k in range(n)]


def test_handoff_values_are_per_frame():
    def chunks():
        yield 0, ["a", "b"], torch.tensor([0, 7])
        yield 2, ["c"], torch.tensor([9])
    feed = DeviceHandoff(chunks(), 4, "t")
    try:
        assert [feed.take(k) for k in range(3)] == ["a", "b", "c"] and feed.take(3) is None
        assert [feed.value(k) for k in range(3)] == [0, 7, 9]
        feed.drop(1)
        with pytest.raises(KeyError):
            feed.value(1)
    finally:
        feed.close()


# ---- the flag --------------------------------------------------------------------------------------------------------

def test_flag_is_opt_in():
    import main as M
    from tests.test_train_monitoring_host import PARENT_FLAG_DEFAULTS
    assert not hasattr(M.parse_flags([]), "scene_threshold")
    assert vars(M.parse_flags([])) == PARENT_FLAG_DEFAULTS
    assert vars(M.parse_flags(["--scene_threshold", "10"])) == dict(PARENT_FLAG_DEFAULTS, scene_threshold="10")


@pytest.mark.parametrize("argv,match", [
    (["--mode", "train", "--scene_threshold", "10"], "inference only"),
    (["--scene_threshold", "0"], r"\(0, 100\]"),
    (["--scene_threshold", "-3"], r"\(0, 100\]"),
    (["--scene_threshold", "100.5"], r"\(0, 100\]"),
    (["--scene_threshold", "nan"], r"\(0, 100\]"),
    (["--scene_threshold", "inf"], r"\(0, 100\]"),
    (["--scene_threshold", "ten"], "not a number"),
    (["--scene_threshold", ""], "not a number"),
])
def test_flag_refused_before_set_up(argv, match, tmp_path, monkeypatch):
    """Refused before anything is set up: no environment change, no output directory."""
    import main as M
    monkeypatch.delenv("CUDA_VISIBLE_DEVICES", raising=False)
    out = str(tmp_path / "out")
    with pytest.raises(ValueError, match=match):
        M.main(argv + ["--output_dir", out, "--checkpoint", "random:1", "--input_dir_LR", str(tmp_path)])
    assert not os.path.exists(out) and "CUDA_VISIBLE_DEVICES" not in os.environ


def test_threshold_values():
    assert scene_threshold("10") == 10.0 and scene_threshold("100") == 100.0 and scene_threshold("1e-3") == 1e-3
