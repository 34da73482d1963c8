"""GPU: the YUV4MPEG2 input and output of `main.py --input_y4m / --output_y4m`.  teco_rgb_to_i420_u8 and
teco_i420_to_rgb_u8 equal cv2.cvtColor(COLOR_RGB2YUV_I420 / COLOR_YUV2RGB_I420) byte for byte on the host sweep
(tests/test_y4m_host.py), on video sizes up to 8K, on pitched and offset buffers and across several grid-stride
passes; malformed calls raise before a launch and write nothing.  The command reads a y4m stream as it reads the PNG
files of its frames, writes to a y4m stream the frames it would write as files, with and without --outscale, from a
FIFO as from a file, and for streams shorter than the warm-up; its device memory does not grow with the stream."""
import itertools
import os
import threading

import cv2
import numpy as np
import pytest
import torch

from tecogan_b200 import _ffi
from tecogan_b200 import kernels as K
from tecogan_b200 import y4m
from tests.test_gpu_inference_stream import LR_HW, NRB, _weights, _write_seq

pytestmark = pytest.mark.gpu

EVEN = range(2, 41, 2)


def _to_i420(rgb):
    return cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)


def _to_rgb(i420):
    return cv2.cvtColor(i420, cv2.COLOR_YUV2RGB_I420)


def _check_rgb_to_i420(rgb):
    h, w = rgb.shape[:2]
    dst = torch.full((3 * h // 2, w), 0x5A, dtype=torch.uint8, device="cuda")
    got = K.rgb_to_i420(torch.from_numpy(rgb).cuda(), dst).cpu().numpy()
    assert np.array_equal(got, _to_i420(rgb)), rgb.shape


def _check_i420_to_rgb(frames):
    got = K.i420_to_rgb(torch.from_numpy(np.ascontiguousarray(frames)).cuda()).cpu().numpy()
    for k, f in enumerate(frames if frames.ndim == 3 else frames[None]):
        assert np.array_equal(got[k], _to_rgb(f)), (frames.shape, k)


@pytest.mark.parametrize("h", EVEN)
def test_kernels_equal_cv2_sweep(h):
    g = np.random.default_rng(200 + h)
    for w in EVEN:
        _check_rgb_to_i420(g.integers(0, 256, (h, w, 3)).astype(np.uint8))
        _check_i420_to_rgb(g.integers(0, 256, (3 * h // 2, w)).astype(np.uint8))


@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840), (4320, 7680)])
def test_kernels_equal_cv2_video_sizes(hw):
    g = np.random.default_rng(hw[1])
    h, w = hw
    _check_rgb_to_i420(g.integers(0, 256, (h, w, 3)).astype(np.uint8))
    _check_i420_to_rgb(g.integers(0, 256, (3 * h // 2, w)).astype(np.uint8))


@pytest.mark.parametrize("v", [0, 255])
def test_kernels_equal_cv2_constant(v):
    for h, w in [(2, 2), (8, 10), (36, 40), (540, 960)]:
        _check_rgb_to_i420(np.full((h, w, 3), v, np.uint8))
        _check_i420_to_rgb(np.full((3 * h // 2, w), v, np.uint8))


def test_i420_to_rgb_many_frames_and_offsets():
    """16 frames of 1080p are several grid-stride passes of a full grid; the same frames at an odd byte offset take the
    byte-wise path."""
    g = np.random.default_rng(4)
    frames = g.integers(0, 256, (16, 1620, 1920)).astype(np.uint8)
    _check_i420_to_rgb(frames)
    for n, (h, w) in [(3, (540, 960)), (5, (34, 38))]:
        src = g.integers(0, 256, (n, 3 * h // 2, w)).astype(np.uint8)
        buf = torch.zeros(1 + src.size, dtype=torch.uint8, device="cuda")
        view = buf[1:].view(n, 3 * h // 2, w)
        view.copy_(torch.from_numpy(src))
        got = K.i420_to_rgb(view).cpu().numpy()
        for k in range(n):
            assert np.array_equal(got[k], _to_rgb(src[k])), (n, h, w, k)


def test_rgb_to_i420_pitched_source_with_offset():
    """The writer's slot may be a row-strided view: odd offsets and pitches (byte-wise path), and 4-byte-aligned ones
    (vector path)."""
    g = np.random.default_rng(9)
    for (h, w), extra, off in [((34, 38), 7, 1), ((128, 144), 5, 3), ((120, 160), 4, 4), ((2160, 3840), 12, 8),
                               ((540, 960), 0, 0)]:
        frame = g.integers(0, 256, (h, w, 3)).astype(np.uint8)
        pitch = 3 * w + extra
        sbuf = torch.from_numpy(g.integers(0, 256, off + h * pitch).astype(np.uint8)).cuda()
        src = sbuf[off:].as_strided((h, w, 3), (pitch, 3, 1))
        src.copy_(torch.from_numpy(frame))
        dst = torch.empty((3 * h // 2, w), dtype=torch.uint8, device="cuda")
        assert np.array_equal(K.rgb_to_i420(src, dst).cpu().numpy(), _to_i420(frame)), (h, w, extra, off)


def test_malformed_calls_raise_without_a_launch():
    g = np.random.default_rng(2)
    src = torch.from_numpy(g.integers(0, 256, (16, 20, 3)).astype(np.uint8)).cuda()
    guard = 4096
    dbuf = torch.full((2 * guard + 24 * 20,), 0xA5, dtype=torch.uint8, device="cuda")
    dst = dbuf[guard:guard + 24 * 20].view(24, 20)
    odd = torch.zeros((15, 20, 3), dtype=torch.uint8, device="cuda")
    for s, d in [(src.float(), dst), (src.cpu(), dst), (src[:, :, :2], dst), (src.permute(1, 0, 2), dst),
                 (src[:, ::2], dbuf[:24 * 10].view(24, 10)), (src, dst.float()), (src, dst.cpu()), (src, dst[:23]),
                 (src, dbuf[:24 * 40].view(24, 40)[:, ::2]), (odd, dbuf[:22 * 20].view(22, 20)),
                 (src[:, :19], dbuf[:24 * 19].view(24, 19)), (src[:0], dbuf[:0].view(0, 20)), (src, "dst")]:
        with pytest.raises(ValueError):
            K.rgb_to_i420(s, d)
    planes = torch.full((2, 24, 20), 0x5A, dtype=torch.uint8, device="cuda")
    obuf = torch.full((2 * guard + 2 * 16 * 20 * 3,), 0xA5, dtype=torch.uint8, device="cuda")
    out = obuf[guard:guard + 2 * 16 * 20 * 3].view(2, 16, 20, 3)
    for f, o in [(planes.float(), None), (planes.cpu(), None), (planes[:, :, ::2], None), (planes[:, :23], None),
                 (torch.zeros((2, 24, 19), dtype=torch.uint8, device="cuda"), None), (planes[:0], None),
                 (torch.zeros((2, 4, 20), dtype=torch.uint8, device="cuda"), None), (planes, out[:1]),
                 (planes, out.float()), (planes, out.permute(0, 2, 1, 3)), ("planes", None)]:
        with pytest.raises(ValueError):
            K.i420_to_rgb(f, o)
    sp, dp, pp, op = _ffi.ptr(src), _ffi.ptr(dst), _ffi.ptr(planes), _ffi.ptr(out)
    for args in [(_ffi.ptr(None), 60, 16, 20, dp), (sp, 60, 16, 20, _ffi.ptr(None)), (sp, 59, 16, 20, dp),
                 (sp, 60, 15, 20, dp), (sp, 60, 16, 19, dp), (sp, 60, 0, 20, dp), (sp, 60, 16, 0, dp),
                 (sp, 60 * 65536, 16, 65536, dp), (sp, 60, -2, 20, dp)]:
        with pytest.raises(ValueError):
            _ffi.call("teco_rgb_to_i420_u8", *args, _ffi.stream_ptr())
    for args in [(_ffi.ptr(None), 2, 16, 20, op), (pp, 2, 16, 20, _ffi.ptr(None)), (pp, 0, 16, 20, op),
                 (pp, -1, 16, 20, op), (pp, 2, 15, 20, op), (pp, 2, 16, 21, op), (pp, 2, 65536, 20, op)]:
        with pytest.raises(ValueError):
            _ffi.call("teco_i420_to_rgb_u8", *args, _ffi.stream_ptr())
    torch.cuda.synchronize()
    assert bool((dbuf == 0xA5).all()) and bool((obuf == 0xA5).all())
    K.rgb_to_i420(src, dst)                                   # later launches still work, and stay in their buffers
    K.i420_to_rgb(planes, out)
    torch.cuda.synchronize()
    assert np.array_equal(dst.cpu().numpy(), _to_i420(src.cpu().numpy()))
    assert np.array_equal(out[1].cpu().numpy(), _to_rgb(planes[1].cpu().numpy()))
    assert bool((dbuf[:guard] == 0xA5).all()) and bool((dbuf[guard + 24 * 20:] == 0xA5).all())
    assert bool((obuf[:guard] == 0xA5).all()) and bool((obuf[guard + 2 * 16 * 20 * 3:] == 0xA5).all())


# ---- the inference command -------------------------------------------------------------------------------------------

def _main(out, *args):
    import main as M
    from tecogan_b200 import config
    prev, cuda = config.precision(), os.environ.get("CUDA_VISIBLE_DEVICES")
    try:
        M.main(["--mode", "inference", "--checkpoint", "random:5", "--num_resblock", str(NRB), "--output_pre", "",
                "--cudaID", cuda or "0", "--output_dir", out] + list(args))
    finally:
        config.set_precision(prev)
        if cuda is None:
            os.environ.pop("CUDA_VISIBLE_DEVICES", None)
        else:
            os.environ["CUDA_VISIBLE_DEVICES"] = cuda
    return {n: open(os.path.join(out, n), "rb").read() for n in sorted(os.listdir(out))}


def _read_y4m(path):
    """(header line, [I420 frames]) of a y4m file this package wrote."""
    data = open(path, "rb").read()
    head, rest = data.split(b"\n", 1)
    hd = y4m.parse_header(head)
    size = y4m.frame_bytes(hd.w, hd.h)
    frames = []
    while rest:
        assert rest[:6] == b"FRAME\n"
        frames.append(np.frombuffer(rest[6:6 + size], np.uint8).reshape(3 * hd.h // 2, hd.w))
        assert len(frames[-1].ravel()) == size
        rest = rest[6 + size:]
    return head, frames


def _sequence(d, n, seed):
    """A y4m stream of n frames (the I420 of the seeded PNG sequence) and the PNG files of its RGB frames: the input
    the stream stands for, as cv2 decodes it."""
    seq = _write_seq(str(d / "png_src"), n, seed=seed)
    rgb = [cv2.imread(os.path.join(seq, "%04d.png" % (k + 1)))[:, :, ::-1] for k in range(n)]
    planes = [_to_i420(np.ascontiguousarray(f)) for f in rgb]
    path = str(d / "in.y4m")
    with open(path, "wb") as f:
        f.write(b"YUV4MPEG2 W%d H%d F30000:1001 Ip A1:1 C420jpeg XYSCSS=420JPEG\n" % (LR_HW[1], LR_HW[0]))
        for p in planes:
            f.write(b"FRAME\n" + p.tobytes())
    pngs = str(d / "png")
    os.makedirs(pngs)
    for k, p in enumerate(planes):
        cv2.imwrite(os.path.join(pngs, "%04d.png" % (k + 1)), _to_rgb(p)[:, :, ::-1])
    return path, pngs


@pytest.fixture(scope="module")
def seq(tmp_path_factory):
    d = tmp_path_factory.mktemp("y4m")
    return _sequence(d, 11, seed=31)


def _want_frames(files):
    """The I420 frames of a run's image files, in file order: cvtColor(RGB2YUV_I420) of each decoded file."""
    return [_to_i420(np.ascontiguousarray(cv2.imdecode(np.frombuffer(files[n], np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1]))
            for n in sorted(files)]


@pytest.mark.parametrize("ext", ["png", "jpg"])
def test_y4m_in_writes_the_files_of_its_png_frames(seq, tmp_path, ext):
    path, pngs = seq
    got = _main(str(tmp_path / "a"), "--input_y4m", path, "--output_ext", ext)
    want = _main(str(tmp_path / "b"), "--input_dir_LR", pngs, "--output_ext", ext)
    assert got == want and len(got) == 11
    assert sorted(got) == ["output_%04d.%s" % (k, ext) for k in range(1, 12)]
    cut = _main(str(tmp_path / "c"), "--input_y4m", path, "--output_ext", ext, "--input_dir_len", "8")
    assert cut == _main(str(tmp_path / "d"), "--input_dir_LR", pngs, "--output_ext", ext, "--input_dir_len", "8")
    assert len(cut) == 8


@pytest.mark.parametrize("outscale", [None, "2"])
def test_y4m_out_holds_the_frames_of_the_image_files(seq, tmp_path, outscale):
    path, pngs = seq
    extra = [] if outscale is None else ["--outscale", outscale]
    files = _main(str(tmp_path / "plain"), "--input_dir_LR", pngs, "--output_ext", "png", *extra)
    out = str(tmp_path / "o.y4m")
    assert _main(str(tmp_path / "y"), "--input_dir_LR", pngs, "--output_y4m", out, *extra) == {}   # no image file
    head, frames = _read_y4m(out)
    s = 4 if outscale is None else 2
    assert head == b"YUV4MPEG2 W%d H%d F25:1 Ip A1:1 C420paldv XCOLORRANGE=LIMITED" % (LR_HW[1] * s, LR_HW[0] * s)
    want = _want_frames(files)
    assert len(frames) == len(want) == 11
    for k, (a, b) in enumerate(zip(frames, want)):
        assert np.array_equal(a, b), k
    # y4m in, y4m out: the same frames, the input's rate and aspect
    out2 = str(tmp_path / "o2.y4m")
    _main(str(tmp_path / "y2"), "--input_y4m", path, "--output_y4m", out2, *extra)
    head2, frames2 = _read_y4m(out2)
    assert head2 == head.replace(b"F25:1", b"F30000:1001")
    assert all(np.array_equal(a, b) for a, b in zip(frames2, frames)) and len(frames2) == 11


def test_odd_output_side_refused_before_the_network(seq, tmp_path, monkeypatch):
    path, _ = seq

    def no_engine(*a, **k):
        raise AssertionError("the network was built")
    monkeypatch.setattr("tecogan_b200.engine.InferenceEngine", no_engine)
    with pytest.raises(ValueError, match="odd"):          # 32 x 36 at 1.25: 40 x 45
        _main(str(tmp_path / "a"), "--input_y4m", path, "--output_y4m", str(tmp_path / "o.y4m"), "--outscale", "1.25")
    assert not os.path.exists(str(tmp_path / "o.y4m"))


def test_fifo_input_equals_file_input(seq, tmp_path):
    path, _ = seq
    want = str(tmp_path / "file.y4m")
    _main(str(tmp_path / "a"), "--input_y4m", path, "--output_y4m", want)
    fifo = str(tmp_path / "in.fifo")
    os.mkfifo(fifo)
    data = open(path, "rb").read()

    def feed():
        with open(fifo, "wb") as f:
            for a in range(0, len(data), 1000):              # in pieces that cut frames and FRAME lines
                f.write(data[a:a + 1000])
    t = threading.Thread(target=feed)
    t.start()
    try:
        got = str(tmp_path / "fifo.y4m")
        _main(str(tmp_path / "b"), "--input_y4m", fifo, "--output_y4m", got)
    finally:
        t.join()
    assert open(got, "rb").read() == open(want, "rb").read()


@pytest.mark.parametrize("n", [3, 5])
def test_short_streams_give_the_image_path_s_frames(tmp_path, n):
    path, pngs = _sequence(tmp_path, n, seed=40 + n)
    files = _main(str(tmp_path / "plain"), "--input_dir_LR", pngs, "--output_ext", "png")
    assert len(files) == {3: 0, 5: 4}[n]                     # the reference's warm-up rule
    assert _main(str(tmp_path / "a"), "--input_y4m", path, "--output_ext", "png") == files
    out = str(tmp_path / "o.y4m")
    _main(str(tmp_path / "b"), "--input_y4m", path, "--output_y4m", out)
    _, frames = _read_y4m(out)
    want = _want_frames(files)
    assert len(frames) == len(want) and all(np.array_equal(a, b) for a, b in zip(frames, want))


def test_truncated_stream_raises_at_that_frame(seq, tmp_path):
    path, _ = seq
    cut = str(tmp_path / "cut.y4m")
    data = open(path, "rb").read()
    with open(cut, "wb") as f:
        f.write(data[:-100])
    with pytest.raises(ValueError, match="frame 11 is truncated"):
        _main(str(tmp_path / "a"), "--input_y4m", cut, "--output_ext", "png")
    empty = str(tmp_path / "empty.y4m")
    with open(empty, "wb") as f:
        f.write(data.split(b"\n", 1)[0] + b"\n")
    with pytest.raises(IndexError):
        _main(str(tmp_path / "b"), "--input_y4m", empty, "--output_ext", "png")


def _peak(tmp_path, n):
    import gc
    import main as M
    from tecogan_b200.engine import InferenceEngine
    path, _ = _sequence(tmp_path / ("s%d" % n), n, seed=5)
    out = str(tmp_path / ("o%d.y4m" % n))
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    reader = y4m.Y4MReader(path)
    frames = reader.frames()
    sink = None
    try:
        first = next(frames)
        eng = InferenceEngine(first.shape[0], first.shape[1], NRB)
        sink = y4m.Y4MWriter(out, 4 * LR_HW[1], 4 * LR_HW[0])
        M.super_resolve_frames(eng, reader.names(), itertools.chain([first], frames), str(tmp_path), "out", "png",
                               None, sink)
    finally:
        frames.close()
        if sink is not None:
            sink.close()
    torch.cuda.synchronize()
    assert len(_read_y4m(out)[1]) == n
    return torch.cuda.max_memory_allocated() - base


def test_peak_memory_flat_in_sequence_length(tmp_path):
    from tecogan_b200 import config
    prev = config.precision()
    try:
        _weights("bf16")
        _peak(tmp_path, 12)                        # module loads, encoder and allocator warm-up
        short, long_ = _peak(tmp_path, 48), _peak(tmp_path, 240)
    finally:
        config.set_precision(prev)
    assert long_ - short < 4 * LR_HW[0] * LR_HW[1] * 3 * 4, (short, long_)
