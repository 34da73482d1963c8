"""GPU: `dataPrepare.py --scene_threshold`.  teco_frame_sads_u8 equals the numpy int64 SAD of consecutive frames on
aligned and unaligned frames, frame sizes that are not a multiple of 16 bytes, one frame with and without `prev`, frames
larger than one grid pass and more pairs than one grid row; it equals frame_sad_q8 on the same frames made float by
frames_to_f32; malformed calls raise and launch nothing.  On MJPG videos with planted cuts (every frame a keyframe, so
cv2 seeks exactly) the scan finds the planted table with the scores of the cv2-halved frames, and the command writes the
files the reference's loop writes for that table, byte for byte, with --threads 1 and 4 alike; --TEST writes only its
log, and --REMOVE deletes only the sources whose scenes were written."""
import hashlib
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

import dataPrepare
from tecogan_b200 import _ffi
from tecogan_b200 import data_prepare as D
from tecogan_b200 import kernels as K

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _np_sads(frames, prev=None):
    f = frames.reshape(len(frames), -1).astype(np.int64)
    out = np.zeros(len(f), np.int64)
    out[1:] = np.abs(f[1:] - f[:-1]).sum(1)
    if prev is not None:
        out[0] = np.abs(f[0] - prev.reshape(-1).astype(np.int64)).sum()
    return out


def _check(frames, prev=None):
    """frames: uint8 CUDA tensor [n, ...] (any offset), prev one frame or None."""
    out = torch.full((frames.shape[0],), -7, dtype=torch.int64, device="cuda")
    K.frame_sads_u8(frames, prev, out)
    want = _np_sads(frames.cpu().numpy(), None if prev is None else prev.cpu().numpy())
    assert np.array_equal(out.cpu().numpy(), want), (tuple(frames.shape), frames.data_ptr() % 16)
    return want


def _rand(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=g)


def _at(t, offset):
    """A contiguous copy of t starting `offset` bytes past a 256-byte aligned address."""
    buf = torch.zeros(t.numel() + 256 + offset, dtype=torch.uint8, device="cuda")
    start = (-buf.data_ptr()) % 256 + offset
    v = buf[start:start + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 256 == offset % 256
    return v


# ---- the kernel ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(5, 16, 16, 3), (3, 540, 960, 3), (4, 1080, 1920, 3), (2, 200, 216, 3), (6, 16)])
def test_aligned_frames(shape):
    f = _rand(shape, sum(shape))
    assert f.data_ptr() % 16 == 0 and f[0].numel() % 16 == 0
    _check(f)
    _check(f, _rand(shape[1:], 1))
    _check(f, f[-1].clone())
    same = f[:1].expand(shape).contiguous()
    assert not _check(same, f[0].clone()).any()


@pytest.mark.parametrize("shape", [(4, 7, 13, 3), (3, 201, 213, 3), (5, 1), (3, 17), (2, 541, 959, 3)])
def test_frame_bytes_not_a_multiple_of_16(shape):
    f = _rand(shape, sum(shape))
    assert f[0].numel() % 16
    _check(f)
    _check(f, _rand(shape[1:], 2))


@pytest.mark.parametrize("offset", [1, 3, 4, 8, 15])
def test_unaligned_pointers(offset):
    f = _rand((3, 64, 96, 3), offset)
    prev = _rand((64, 96, 3), offset + 1)
    _check(_at(f, offset))
    _check(_at(f, offset), prev)
    _check(f, _at(prev, offset))                 # aligned frames, unaligned prev
    _check(_at(f, offset), _at(prev, offset))


def test_one_frame():
    f = _rand((1, 33, 47, 3), 4)
    assert _check(f)[0] == 0
    _check(f, _rand((33, 47, 3), 5))
    f = _rand((1, 32, 48, 3), 6)
    assert _check(f)[0] == 0
    _check(f, _rand((32, 48, 3), 7))


@pytest.mark.parametrize("offset", [0, 5])
def test_frames_larger_than_one_grid_pass(offset):
    """16 MiB frames: one pass of the whole grid covers 4 KiB per CTA on the 16-byte path and 256 B on the byte path,
    at most a few MiB with every CTA of the device resident, so each thread strides through its frame several times."""
    side = 2048
    f = _at(_rand((2, side, side, 4), 8), offset)
    _check(f)
    _check(f[:1], _at(_rand((side, side, 4), 9), offset))


@pytest.mark.parametrize("frame_bytes", [3, 16])
def test_more_pairs_than_one_grid_row(frame_bytes):
    f = _rand((70001, frame_bytes), frame_bytes)
    _check(f)
    _check(f, _rand((frame_bytes,), 10))


def test_equals_frame_sad_q8_on_the_same_frames():
    for shape in [(4, 200, 216, 3), (3, 7, 13, 3)]:
        f = _rand(shape, 11)
        sads = K.frame_sads_u8(f).cpu().numpy()
        f32 = K.frames_to_f32(f)
        one = torch.empty(1, dtype=torch.int64, device="cuda")
        for i in range(1, shape[0]):
            K.frame_sad_q8(f32[i - 1].contiguous(), f32[i].contiguous(), one)
            assert int(one.item()) == int(sads[i]), (shape, i)


def test_malformed_calls_raise_without_a_launch():
    f = _rand((3, 8, 8, 3), 12)
    out = torch.full((3,), -7, dtype=torch.int64, device="cuda")
    bad_frames = [f.float(), f.cpu(), f[:, :, ::2], f[:0], torch.zeros((3, 0), dtype=torch.uint8, device="cuda"),
                  f.to(torch.int8), "f"]
    for x in bad_frames:
        with pytest.raises(ValueError):
            K.frame_sads_u8(x, None, out if torch.is_tensor(x) and x.shape[:1] == (3,) else None)
    for p in [f[0].float(), f[0].cpu(), f[0, :7], f[0].reshape(192), f[0][:, ::2], f[:2], "p"]:
        with pytest.raises(ValueError):
            K.frame_sads_u8(f, p, out)
    for o in [out.int(), out[:2], torch.zeros(4, dtype=torch.int64, device="cuda"), out.cpu(), out.float(),
              torch.zeros((3, 2), dtype=torch.int64, device="cuda")[:, 0], "out"]:
        with pytest.raises(ValueError):
            K.frame_sads_u8(f, None, o)
    P, N = _ffi.ptr, _ffi.ptr(None)
    for args in [(N, 192, 3, N, P(out)), (P(f), 192, 3, N, N), (P(f), 192, 0, N, P(out)), (P(f), 192, -1, N, P(out)),
                 (P(f), 0, 3, N, P(out)), (P(f), -192, 3, N, P(out)), (P(f), 1 << 62, 3, N, P(out))]:
        with pytest.raises(ValueError):
            _ffi.call("teco_frame_sads_u8", *args, _ffi.stream_ptr())
    torch.cuda.synchronize()
    assert out.tolist() == [-7, -7, -7]                          # nothing was written
    K.frame_sads_u8(f, None, out)
    assert out.tolist() == _np_sads(f.cpu().numpy()).tolist()   # later launches still work


# ---- the command -----------------------------------------------------------------------------------------------------

DURATION, THRESHOLD = 5, "10"
# name, width, height, shot lengths: a cut starts every shot after the first
FIXTURES = [("b", 416, 400, [9, 6]), ("a", 400, 432, [11, 7, 15]), ("c", 400, 400, [4]), ("small", 320, 400, [6])]
TABLE = {"a": [0, 5, 11, 18, 23, 28], "b": [0, 9]}             # "c" has no 5-frame scene; "small" is skipped
CUTS = {"a": [11, 18], "b": [9], "c": []}


def _shots(w, h, lens, seed):
    """Smooth noise drifting (1, 2) pixels a frame; shots alternate dark (0..127) and bright (128..255) textures."""
    g = np.random.default_rng(seed)
    frames = []
    for k, n in enumerate(lens):
        small = g.integers(0, 256, ((h + 64) // 16 + 1, (w + 64) // 16 + 1, 3)).astype(np.uint8)
        base = cv2.resize(small, (w + 64, h + 64), interpolation=cv2.INTER_CUBIC) // 2 + (128 if k % 2 else 0)
        frames += [base[j:j + h, 2 * j:2 * j + w].copy() for j in range(n)]
    return frames


@pytest.fixture(scope="module")
def videos(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("videos"))
    for k, (name, w, h, lens) in enumerate(FIXTURES):
        vw = cv2.VideoWriter(os.path.join(d, name + ".avi"), cv2.VideoWriter_fourcc(*"MJPG"), 25, (w, h))
        assert vw.isOpened()
        for f in _shots(w, h, lens, seed=k):
            vw.write(f)
        vw.release()
    return d


def _disk(videos, d):
    os.makedirs(d)
    for n in os.listdir(videos):
        os.symlink(os.path.join(videos, n), os.path.join(d, n))
    return d


def _half(frame):
    return cv2.resize(frame, (0, 0), fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)


def _host_sads(path):
    """Every frame decoded in order by cv2 and halved by cv2; the SADs of consecutive ones on the host -> (sads,
    values)."""
    cam = cv2.VideoCapture(path)
    frames = []
    while True:
        ok, f = cam.read()
        if not ok:
            break
        frames.append(_half(f))
    cam.release()
    return _np_sads(np.stack(frames)).tolist(), frames[0].size


def _host_scores(path):
    return D.frame_scores(*_host_sads(path))


def _reference(disk, out, table, start_id, duration):
    """The reference's loop over the table, restated: a seek before every frame, cv2.resize INTER_AREA, cv2.imwrite."""
    cur = start_id
    for stem, starts in table.items():
        for s in starts:
            d = os.path.join(out, "scene_%04d/" % cur)
            os.makedirs(d)
            cam = cv2.VideoCapture(os.path.join(disk, stem + ".avi"))
            for i in range(duration):
                cam.set(1, i + s)
                ok, f = cam.read()
                assert ok
                cv2.imwrite(d + "col_high_%04d.png" % i, _half(f))
            cam.release()
            cur += 1


def _digests(root):
    res = {}
    for r, _, fs in os.walk(root):
        for n in fs:
            if n.endswith(".png"):
                with open(os.path.join(r, n), "rb") as f:
                    res[os.path.relpath(os.path.join(r, n), root)] = hashlib.sha256(f.read()).hexdigest()
    return res


@pytest.mark.parametrize("window", [None, 1, 3, 7])
def test_scan_video_equals_the_host_sads(videos, monkeypatch, window):
    """Staging windows of the default size (a whole fixture video) and of 1, 3 and 7 frames of video "a": the windows
    are chained through prev, and their sums come back in order."""
    if window is not None:
        monkeypatch.setattr(D, "WINDOW_BYTES", window * 3 * 400 * 432)
    dev = torch.device("cuda", torch.cuda.current_device())
    for stem in ("a", "b"):
        path = os.path.join(videos, stem + ".avi")
        assert D.scan_video(path, dev) == _host_sads(path)


def test_scan_finds_the_planted_cuts(videos, capsys):
    table, sources = D.scan(videos, float(THRESHOLD), DURATION, threads=2)
    assert table == TABLE and list(table) == ["a", "b"]
    assert sources == {k: os.path.join(videos, k + ".avi") for k in TABLE}
    out = capsys.readouterr().out.splitlines()
    for stem, cuts in CUTS.items():
        scores = _host_scores(os.path.join(videos, stem + ".avi"))
        assert [i for i, s in enumerate(scores) if i > 0 and s >= float(THRESHOLD)] == cuts
        i = out.index("%s: %d frames" % (os.path.join(videos, stem + ".avi"), len(scores)))
        assert out[i + 1:i + 1 + len(cuts)] == ["scene cut before frame %d, score %.4f" % (c, scores[c]) for c in cuts]
        assert out[i + 1 + len(cuts)] == "%d scenes of %d frames" % (len(TABLE.get(stem, [])), DURATION)
    assert "Skipped videos of small size 320x400" in out
    assert out[-4:] == ["video_data_dict = {", '    "a" : [0, 5, 11, 18, 23, 28],', '    "b" : [0, 9],', "}"]


@pytest.fixture(scope="module")
def runs(videos, tmp_path_factory):
    """The command with --threads 1 and 4 -> {threads: (disk, digests, stdout lines)}."""
    import io
    from contextlib import redirect_stdout
    res = {}
    for threads in (1, 4):
        disk = _disk(videos, str(tmp_path_factory.mktemp("run") / "disk"))
        buf = io.StringIO()
        with redirect_stdout(buf):
            dataPrepare.main(["--disk_path", disk, "--duration", str(DURATION), "--start_id", "100",
                              "--scene_threshold", THRESHOLD, "--threads", str(threads)])
        res[threads] = (disk, _digests(disk), buf.getvalue().splitlines())
    return res


def test_command_writes_the_reference_s_files(videos, runs, tmp_path):
    ref = str(tmp_path / "ref")
    _reference(videos, ref, TABLE, 100, DURATION)
    want = _digests(ref)
    assert len(want) == 8 * DURATION
    disk, got, out = runs[1]
    assert got == want
    assert out[-1] == "Done: get 8 valid folders with %d frames from 2 videos." % DURATION
    assert "folder %s: %dx[400,432]//2 at frame 28 of %s" % (
        os.path.join(disk, "scene_0105/"), DURATION, os.path.join(disk, "a.avi")) in out
    assert not os.path.exists(os.path.join(disk, "scene_0108"))


def test_threads_give_identical_trees(runs):
    assert runs[1][1] == runs[4][1] and len(runs[1][1]) == 8 * DURATION
    strip = lambda lines, disk: [l.replace(disk, "<disk>") for l in lines if "threads" not in l]   # noqa: E731
    assert strip(runs[1][2], runs[1][0]) == strip(runs[4][2], runs[4][0])


def test_test_mode_writes_only_the_log(videos, tmp_path):
    disk = _disk(videos, str(tmp_path / "disk"))
    before = sorted(os.listdir(disk))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "dataPrepare.py"), "--disk_path", disk, "--duration",
                        str(DURATION), "--scene_threshold", THRESHOLD, "--TEST"], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    assert sorted(os.listdir(disk)) == sorted(before + ["log"])
    logs = os.listdir(os.path.join(disk, "log"))
    assert len(logs) == 1
    with open(os.path.join(disk, "log", logs[0])) as f:
        assert f.read().splitlines() == r.stdout.splitlines()
    out = r.stdout.splitlines()
    assert '    "a" : [0, 5, 11, 18, 23, 28],' in out
    assert out[-1] == "Done: get 8 valid folders with %d frames from 2 videos." % DURATION


def test_remove_deletes_only_processed_sources(videos, tmp_path, capsys):
    disk = _disk(videos, str(tmp_path / "disk"))
    dataPrepare.main(["--disk_path", disk, "--duration", str(DURATION), "--scene_threshold", THRESHOLD, "--REMOVE"])
    left = set(os.listdir(disk))
    assert {"a.avi", "b.avi"}.isdisjoint(left) and {"c.avi", "small.avi"} <= left
    assert len(_digests(disk)) == 8 * DURATION
    out = capsys.readouterr().out.splitlines()
    assert [l for l in out if l.startswith("remove")] == ["remove  " + os.path.join(disk, n) for n in ("a.avi", "b.avi")]
