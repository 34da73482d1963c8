"""CPU: the YUV4MPEG2 input and output of `main.py --input_y4m / --output_y4m` without a device.  The numpy restatement
of cv2 4.13's I420 conversions (tests/golden/yuv_oracle.py), which tecogan_b200/csrc/yuv.cu is held to, equals
cv2.cvtColor byte for byte in both directions; the header parser (tecogan_b200/y4m.py) reads what it writes and refuses
every stream the conversion does not cover; a truncated frame raises; the flags are opt-in and their conflicts are
refused before anything is set up."""
import io
import os

import cv2
import numpy as np
import pytest

from tecogan_b200 import y4m
from tests.golden import yuv_oracle as O

EVEN = range(2, 41, 2)


def check_both(rgb, i420):
    assert np.array_equal(O.rgb_to_i420(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)), rgb.shape
    assert np.array_equal(O.i420_to_rgb(i420), cv2.cvtColor(i420, cv2.COLOR_YUV2RGB_I420)), i420.shape


@pytest.mark.parametrize("h", EVEN)
def test_oracle_equals_cv2_sweep(h):
    g = np.random.default_rng(h)
    for w in EVEN:
        check_both(g.integers(0, 256, (h, w, 3)).astype(np.uint8), g.integers(0, 256, (3 * h // 2, w)).astype(np.uint8))


@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840)])
def test_oracle_equals_cv2_video_sizes(hw):
    g = np.random.default_rng(hw[0])
    h, w = hw
    check_both(g.integers(0, 256, (h, w, 3)).astype(np.uint8), g.integers(0, 256, (3 * h // 2, w)).astype(np.uint8))


@pytest.mark.parametrize("v", [0, 255])
def test_oracle_equals_cv2_constant(v):
    for h, w in [(2, 2), (8, 10), (36, 40)]:
        check_both(np.full((h, w, 3), v, np.uint8), np.full((3 * h // 2, w), v, np.uint8))


def test_chroma_is_the_top_left_pixel():
    """cv2 takes U and V from the block's top-left pixel: a red pixel at (0, 0) moves them, one at (1, 1) does not."""
    a = np.zeros((2, 2, 3), np.uint8)
    a[0, 0] = (255, 0, 0)
    b = np.zeros((2, 2, 3), np.uint8)
    b[1, 1] = (255, 0, 0)
    assert O.rgb_to_i420(a)[2:].ravel().tolist() == [90, 240]
    assert O.rgb_to_i420(b)[2:].ravel().tolist() == [128, 128]
    for x in (a, b):
        assert np.array_equal(O.rgb_to_i420(x), cv2.cvtColor(x, cv2.COLOR_RGB2YUV_I420))


# ---- the container ---------------------------------------------------------------------------------------------------

def test_header_round_trip():
    line = y4m.format_header(3840, 2160, '30000:1001', '1:1')
    assert line == b'YUV4MPEG2 W3840 H2160 F30000:1001 Ip A1:1 C420paldv XCOLORRANGE=LIMITED\n'
    assert y4m.parse_header(line[:-1]) == y4m.Header(3840, 2160, '30000:1001', '1:1')
    assert y4m.format_header(16, 8) == b'YUV4MPEG2 W16 H8 F25:1 Ip A1:1 C420paldv XCOLORRANGE=LIMITED\n'


@pytest.mark.parametrize("line,want", [
    (b'YUV4MPEG2 W960 H540', (960, 540, '25:1', '1:1')),
    (b'YUV4MPEG2 W960 H540 F24:1 Ip A0:0 C420jpeg XYSCSS=420JPEG', (960, 540, '24:1', '0:0')),
    (b'YUV4MPEG2 H540 W960 C420mpeg2 I? XCOLORRANGE=LIMITED F60:1', (960, 540, '60:1', '1:1')),
    (b'YUV4MPEG2 W8 H8 C420 A128:117', (8, 8, '25:1', '128:117')),
    (b'YUV4MPEG2 W8 H65534 C420paldv Ip', (8, 65534, '25:1', '1:1')),
])
def test_header_accepted(line, want):
    assert tuple(y4m.parse_header(line)) == want


@pytest.mark.parametrize("line,field", [
    (b'YUV4MPEG W960 H540', 'magic'),
    (b'yuv4mpeg2 W960 H540', 'magic'),
    (b'YUV4MPEG2 H540', 'W'),
    (b'YUV4MPEG2 W960', 'H'),
    (b'YUV4MPEG2 Wabc H540', 'W'),
    (b'YUV4MPEG2 W961 H540', 'W961'),
    (b'YUV4MPEG2 W960 H541', 'H541'),
    (b'YUV4MPEG2 W6 H540', 'W6'),
    (b'YUV4MPEG2 W960 H4', 'H4'),
    (b'YUV4MPEG2 W65536 H540', 'W65536'),
    (b'YUV4MPEG2 W960 H540 C444', 'C444'),
    (b'YUV4MPEG2 W960 H540 C422', 'C422'),
    (b'YUV4MPEG2 W960 H540 Cmono', 'Cmono'),
    (b'YUV4MPEG2 W960 H540 C420p10', 'C420p10'),
    (b'YUV4MPEG2 W960 H540 C420 XCOLORRANGE=FULL', 'yuv420p'),
    (b'YUV4MPEG2 W960 H540 It', 'It'),
    (b'YUV4MPEG2 W960 H540 Ib', 'Ib'),
    (b'YUV4MPEG2 W960 H540 Im', 'Im'),
    (b'YUV4MPEG2 W960 H540 F25', 'F25'),
])
def test_header_refused(line, field):
    with pytest.raises(ValueError, match=field):
        y4m.parse_header(line)


def _stream(h, w, frames, header=None, cut=0):
    data = (header if header is not None else y4m.format_header(w, h)) + b''.join(
        b'FRAME\n' + f.tobytes() for f in frames)
    return data[:len(data) - cut]


def test_frames_read_in_order_and_truncation_raises(tmp_path):
    g = np.random.default_rng(3)
    frames = [g.integers(0, 256, (12, 8)).astype(np.uint8) for _ in range(3)]
    f = io.BytesIO(_stream(8, 8, frames)[len(y4m.format_header(8, 8)):])
    buf = np.empty(y4m.frame_bytes(8, 8), np.uint8)
    for k in range(3):
        assert y4m.read_frame(f, buf, k) and np.array_equal(buf, frames[k].ravel())
    assert not y4m.read_frame(f, buf, 3)
    body = _stream(8, 8, frames)[len(y4m.format_header(8, 8)):]
    for cut, what in [(1, 'frame 3 is truncated'), (96, 'frame 3 is truncated'), (97, 'FRAME line of frame 3'),
                      (100, 'FRAME line of frame 3')]:
        f = io.BytesIO(body[:len(body) - cut])
        y4m.read_frame(f, buf, 0)
        y4m.read_frame(f, buf, 1)
        with pytest.raises(ValueError, match=what):
            y4m.read_frame(f, buf, 2)
    f = io.BytesIO(b'FRAME Ixyz\n' + bytes(96) + b'FRAMX\n' + bytes(96))
    assert y4m.read_frame(f, buf, 0)                       # parameters after FRAME are ignored
    with pytest.raises(ValueError, match='frame 2 does not start with FRAME'):
        y4m.read_frame(f, buf, 1)


def test_reader_refuses_header_on_open(tmp_path):
    p = str(tmp_path / "a.y4m")
    for data, match in [(b'', 'empty'), (b'YUV4MPEG2 W8 H8 C444\nFRAME\n', 'C444'), (b'YUV4MPEG2 W8 H8', 'truncated')]:
        with open(p, 'wb') as f:
            f.write(data)
        with pytest.raises(ValueError, match=match):
            y4m.Y4MReader(p)


def test_writer_writes_header_and_frames(tmp_path):
    p = str(tmp_path / "o.y4m")
    wr = y4m.Y4MWriter(p, 8, 4, '24000:1001', '4:3')
    frames = [np.full((6, 8), k, np.uint8) for k in range(2)]
    for f in frames:
        wr.write(f)
    with pytest.raises(ValueError, match='48 bytes'):
        wr.write(np.zeros(10, np.uint8))
    wr.close()
    assert open(p, 'rb').read() == _stream(4, 8, frames, y4m.format_header(8, 4, '24000:1001', '4:3'))
    for w, h in [(9, 4), (8, 3), (0, 4)]:
        with pytest.raises(ValueError, match='even'):
            y4m.Y4MWriter(str(tmp_path / "bad.y4m"), w, h)


def test_writer_raises_on_a_closed_pipe():
    r, w = os.pipe()
    os.close(r)
    wr = y4m.Y4MWriter.__new__(y4m.Y4MWriter)
    wr.w, wr.h, wr.f = 8, 8, os.fdopen(w, 'wb', buffering=0)
    with pytest.raises(OSError):
        wr.write(np.zeros(96, np.uint8))
    wr.f.close()


# ---- the flags -------------------------------------------------------------------------------------------------------

def test_y4m_flags_are_opt_in():
    import main as M
    from tests.test_train_monitoring_host import PARENT_FLAG_DEFAULTS
    assert vars(M.parse_flags([])) == PARENT_FLAG_DEFAULTS
    for flag in ("input_y4m", "output_y4m"):
        assert not hasattr(M.parse_flags([]), flag)
        assert vars(M.parse_flags(["--" + flag, "a.y4m"])) == dict(PARENT_FLAG_DEFAULTS, **{flag: "a.y4m"})


@pytest.mark.parametrize("argv,match", [
    (["--mode", "train", "--input_y4m", "a.y4m"], "input_y4m"),
    (["--mode", "train", "--output_y4m", "a.y4m"], "output_y4m"),
    (["--input_y4m", "a.y4m", "--input_dir_LR", "LR"], "input_y4m"),
    (["--input_y4m", "a.y4m", "--input_dir_HR", "HR"], "input_y4m"),
])
def test_y4m_conflicts_refused(argv, match, tmp_path, monkeypatch):
    """Refused before anything is set up: no environment change, no output directory."""
    import main as M
    monkeypatch.delenv("CUDA_VISIBLE_DEVICES", raising=False)
    out = str(tmp_path / "out")
    with pytest.raises(ValueError, match=match):
        M.main(argv + ["--output_dir", out, "--checkpoint", "random:1"])
    assert not os.path.exists(out) and "CUDA_VISIBLE_DEVICES" not in os.environ


def test_wrappers_refuse_cpu_tensors():
    import torch
    from tecogan_b200 import kernels as K
    with pytest.raises(ValueError):
        K.rgb_to_i420(torch.zeros((8, 8, 3), dtype=torch.uint8), torch.zeros((12, 8), dtype=torch.uint8))
    with pytest.raises(ValueError):
        K.i420_to_rgb(torch.zeros((12, 8), dtype=torch.uint8))


@pytest.mark.parametrize("n", [1, 2, 3, 5, 6, 7, 12])
@pytest.mark.parametrize("limit", [-1, 4])
def test_reader_order_names_and_thread(tmp_path, n, limit):
    """Y4MReader.frames() hands the stream out in the reference's padded order, reading it once, and names() names the
    same frames; --input_dir_len cuts the stream; the reader thread is joined at the end.  The device conversion is
    replaced by the frame's first byte."""
    import threading
    from tecogan_b200.lib.dataloader import padded
    p = str(tmp_path / "a.y4m")
    with open(p, "wb") as f:
        f.write(y4m.format_header(8, 8) + b"".join(b"FRAME\n" + bytes([k]) * 96 for k in range(n)))
    r = y4m.Y4MReader(p, limit)
    read = []

    def chunks():
        buf = np.empty(96, np.uint8)
        for k in range(limit if limit > 0 else 10 ** 6):
            if not y4m.read_frame(r.f, buf, k):
                return
            read.append(k)
            yield k, [int(buf[0])]
    r._chunks = chunks
    before = threading.active_count()
    frames = r.frames()
    got = list(zip(frames, r.names()))
    assert threading.active_count() == before
    m = min(n, limit) if limit > 0 else n
    want = padded(list(range(m)))
    assert [f for f, _ in got] == want and read == list(range(m))
    assert [name for _, name in got] == ["%04d" % (k + 1) for k in want]
