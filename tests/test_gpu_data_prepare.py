"""GPU: the training-data preparation on the device.  teco_area_half_u8 equals cv2.resize(fx=fy=0.5, INTER_AREA) byte for
byte, with and without the channel swap, on every size 2..40 x 2..40 and on source-video sizes; one launch takes frames
from different buffers; nothing outside the output is written; bad frames raise.  prepare() on generated videos writes
the files the reference's loop writes (a seek before every frame, cv2.resize, cv2.imwrite), byte for byte, and so does
dataPrepare.py run as a command.

cv2.VideoWriter rounds frame sides down to even, so the fixture videos have even sides; their halves are odd (201, 213),
and the odd source sides are covered by the kernel cases."""
import hashlib
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from tecogan_b200 import _ffi
from tecogan_b200 import data_prepare as D
from tecogan_b200 import kernels as K

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LARGE = [(721, 1281), (720, 1281), (1080, 1920), (2160, 4096), (1081, 1919)]


def _cv2(frame):
    return cv2.resize(frame, (0, 0), fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)


def _check(frames):
    """frames: uint8 [N, H, W, 3] numpy -> kernel output, plain and swapped, equals cv2 frame by frame."""
    dev = torch.from_numpy(frames).cuda()
    plain = K.area_half(dev).cpu().numpy()
    swapped = K.area_half(dev, swap_rb=True).cpu().numpy()
    for f, p, s in zip(frames, plain, swapped):
        want = _cv2(f)
        assert p.shape == want.shape and np.array_equal(p, want), f.shape
        assert np.array_equal(s, want[:, :, ::-1]), f.shape


@pytest.mark.parametrize("H", range(2, 41))
def test_kernel_equals_cv2_small(H):
    g = np.random.default_rng(H)
    for W in range(2, 41):
        _check(g.integers(0, 256, (2, H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("H,W", LARGE)
def test_kernel_equals_cv2_large(H, W):
    _check(np.random.default_rng(H * W).integers(0, 256, (2, H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("v", [0, 1, 254, 255])
def test_kernel_equals_cv2_constant(v):
    for H, W in [(3, 3), (7, 11)] + LARGE[:2]:
        _check(np.full((1, H, W, 3), v, np.uint8))


def test_one_launch_over_frames_from_different_buffers():
    """Separate tensors, and frames at odd byte offsets inside one buffer, in one table."""
    g = np.random.default_rng(7)
    H, W = 37, 29
    a = torch.from_numpy(g.integers(0, 256, (H, W, 3)).astype(np.uint8)).cuda()
    big = torch.from_numpy(g.integers(0, 256, 5 + 2 * H * W * 3).astype(np.uint8)).cuda()
    b = big[5:5 + H * W * 3].view(H, W, 3)
    c = big[5 + H * W * 3:].view(H, W, 3)
    out = K.area_half([a, b, c, a], swap_rb=True).cpu().numpy()
    for o, f in zip(out, [a, b, c, a]):
        assert np.array_equal(o, _cv2(f.cpu().numpy())[:, :, ::-1])


def test_nothing_written_outside_the_output():
    for H, W in [(3, 3), (39, 41), (720, 1281)]:
        N, oh, ow = 3, K.area_half_size(H), K.area_half_size(W)
        frames = torch.from_numpy(np.random.default_rng(H).integers(0, 256, (N, H, W, 3)).astype(np.uint8)).cuda()
        guard = 4096
        buf = torch.full((2 * guard + N * oh * ow * 3,), 0xA5, dtype=torch.uint8, device="cuda")
        out = buf[guard:guard + N * oh * ow * 3].view(N, oh, ow, 3)
        K.area_half(frames, out=out)
        torch.cuda.synchronize()
        assert bool((buf[:guard] == 0xA5).all()) and bool((buf[guard + out.numel():] == 0xA5).all())
        want = np.stack([_cv2(f) for f in frames.cpu().numpy()])
        assert np.array_equal(out.cpu().numpy(), want)


def test_bad_frames_raise():
    for shape, dtype in [((1, 8, 3), torch.uint8), ((8, 1, 3), torch.uint8), ((8, 8, 3), torch.uint16),
                         ((8, 8, 3), torch.float32), ((8, 8, 4), torch.uint8), ((65536, 2, 3), torch.uint8),
                         ((2, 65536, 3), torch.uint8)]:
        with pytest.raises(ValueError):
            K.area_half(torch.zeros(shape, dtype=dtype, device="cuda"))
    with pytest.raises(ValueError):
        K.area_half(torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"),
                    out=torch.empty((1, 4, 5, 3), dtype=torch.uint8, device="cuda"))
    table = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty(64, dtype=torch.uint8, device="cuda")
    for N, H, W in [(0, 8, 8), (1, 1, 8), (1, 8, 65536), (65536, 8, 8)]:
        with pytest.raises(ValueError):
            _ffi.call("teco_area_half_u8", _ffi.ptr(table), N, H, W, _ffi.ptr(out), 0, _ffi.stream_ptr())
    K.area_half(torch.zeros((4, 4, 3), dtype=torch.uint8, device="cuda"))      # later launches still work
    torch.cuda.synchronize()


# ---- end to end ------------------------------------------------------------------------------------------------

FIXTURES = [("1001", "FFV1", ".mkv", 426, 402, 240), ("1002", "mp4v", ".mp4", 720, 480, 300)]
TABLE = {"1001": [0, 150], "999": [3], "1002": [7, 200, 251]}
DURATION = 16


def _write_video(path, fourcc, w, h, n, seed):
    g = np.random.default_rng(seed)
    base = g.integers(0, 256, (h + 64, w + 64, 3)).astype(np.uint8)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*fourcc), 25, (w, h))
    assert vw.isOpened(), path
    for i in range(n):
        y, x = (3 * i) % 64, (5 * i) % 64
        f = base[y:y + h, x:x + w].copy()
        f[(i * 7) % h, :, :] = 255 - f[(i * 7) % h]
        vw.write(f)
    vw.release()


@pytest.fixture(scope="module")
def sources(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("videos"))
    for k, (vid, fourcc, ext, w, h, n) in enumerate(FIXTURES):
        _write_video(os.path.join(d, vid + ext), fourcc, w, h, n, seed=k)
    return d


def _reference(disk, out, table, start_id, duration):
    """The reference's loop, restated: a seek before every frame, cv2.resize INTER_AREA, cv2.imwrite."""
    cur = start_id
    for vid, starts in table.items():
        path = D.source_file(disk, vid)
        if path is None:
            continue
        for s in starts:
            d = os.path.join(out, "scene_%04d/" % cur)
            os.makedirs(d)
            cam = cv2.VideoCapture(path)
            for i in range(duration):
                cam.set(1, i + s)
                ok, f = cam.read()
                assert ok
                cv2.imwrite(d + "col_high_%04d.png" % i, _cv2(f))
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


@pytest.fixture(scope="module")
def reference(sources, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("reference"))
    _reference(sources, out, TABLE, 2000, DURATION)
    return _digests(out)


@pytest.mark.parametrize("threads", [1, 2])
def test_prepare_equals_reference_loop(sources, reference, tmp_path, threads):
    disk = str(tmp_path)
    for n in os.listdir(sources):
        os.symlink(os.path.join(sources, n), os.path.join(disk, n))
    assert D.prepare(TABLE, disk, 2000, DURATION, threads=threads) == 2
    got = _digests(disk)
    assert len(got) == 5 * DURATION
    assert sorted(got) == sorted(reference)
    assert got == reference


def test_command_equals_reference_loop(sources, tmp_path):
    """dataPrepare.py as a command, with its own table: video 204313990 starts its one scene at frame 110."""
    disk = str(tmp_path / "disk")
    os.makedirs(disk)
    src = os.path.join(sources, "1002.mp4")
    os.symlink(src, os.path.join(disk, "204313990.mp4"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "dataPrepare.py"), "--disk_path", disk, "--duration", "12",
                        "--start_id", "5", "--threads", "2"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.splitlines()[-1] == "Done: get 1 valid folders with 12 frames from 1 videos."
    ref = str(tmp_path / "ref")
    _reference(disk, ref, {"204313990": [110]}, 5, 12)
    assert _digests(disk) == _digests(ref) and len(_digests(ref)) == 12
    logs = os.listdir(os.path.join(disk, "log"))
    assert len(logs) == 1 and logs[0].startswith("logfile_")
    with open(os.path.join(disk, "log", logs[0])) as f:
        assert f.read().splitlines() == r.stdout.splitlines()


def test_worker_error_joins_and_raises(sources, tmp_path):
    """A scene past the end of its video: the error reaches the caller, with every worker and writer thread joined."""
    import threading
    disk = str(tmp_path)
    os.symlink(os.path.join(sources, "1002.mp4"), os.path.join(disk, "1002.mp4"))
    os.symlink(os.path.join(sources, "1001.mkv"), os.path.join(disk, "1001.mkv"))
    with pytest.raises(RuntimeError, match="cannot read frame"):
        D.prepare({"1001": [0], "1002": [295]}, disk, 0, DURATION, threads=2)
    assert not [t.name for t in threading.enumerate() if t.name.startswith(("dataPrepare", "FrameWriter"))]
