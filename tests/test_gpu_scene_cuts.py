"""GPU: `main.py --scene_threshold`.  teco_frame_sad_q8 equals the integer numpy SAD of the 8-bit quantised frames bit
for bit (vector and scalar paths, rounding boundaries, values outside [0, 1], u8 and u16 sources); malformed calls raise
before a launch.  The command finds the cuts of a stream of three synthetic scenes from PNG files and from a y4m
stream, at both precisions, and writes each scene as a run on that scene alone writes it; a stream without a cut gives
the bytes of a run without the flag; device memory does not grow with the stream or its number of cuts; a reader error
is raised at the frame that needs it."""
import gc
import itertools
import os
import re

import cv2
import numpy as np
import pytest
import torch

from tecogan_b200 import _ffi
from tecogan_b200 import kernels as K
from tecogan_b200 import y4m
from tests.test_gpu_inference_stream import LR_HW, NRB, _weights
from tests.test_gpu_y4m import _main, _read_y4m

pytestmark = pytest.mark.gpu

T = "10"


def _q8(x):
    return np.clip(np.rint(np.float32(255.0) * np.asarray(x, np.float32)), 0, 255).astype(np.int64)


def _np_sad(a, b):
    return int(np.abs(_q8(a) - _q8(b)).sum())


def _dev_sad(a, b):
    out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    K.frame_sad_q8(a, b, out)
    return int(out.item())


def _check(a, b):
    assert _dev_sad(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) == _np_sad(a, b), a.shape


# ---- the kernel ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hw", [(8, 8), (7, 13), (1, 1), (3, 5), (144, 180), (540, 960), (1080, 1920)])
def test_sad_equals_numpy_on_seeded_frames(hw):
    g = np.random.default_rng(hw[0] * 7 + hw[1])
    a = (g.random(hw + (3,)) * 1.4 - 0.2).astype(np.float32)      # below 0 and above 1 included
    b = (g.random(hw + (3,)) * 1.4 - 0.2).astype(np.float32)
    _check(a, b)
    _check(a, a)
    c = a.copy()                                                   # a few values changed: the sum is small and exact
    c.flat[g.integers(0, c.size, 5)] += np.float32(0.5)
    _check(a, c)


def test_sad_of_offset_views_takes_the_scalar_path():
    g = np.random.default_rng(5)
    for h, w in [(8, 8), (144, 180), (33, 47)]:
        n = h * w * 3
        a = (g.random(n) * 1.2 - 0.1).astype(np.float32)
        b = (g.random(n) * 1.2 - 0.1).astype(np.float32)
        want = _np_sad(a, b)
        for oa, ob in [(1, 1), (0, 1), (1, 0), (2, 3), (3, 2), (0, 0)]:
            ba = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
            bb = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
            va, vb = ba[oa:oa + n].view(h, w, 3), bb[ob:ob + n].view(h, w, 3)
            va.copy_(torch.from_numpy(a).view(h, w, 3))
            vb.copy_(torch.from_numpy(b).view(h, w, 3))
            assert va.is_contiguous() and vb.is_contiguous()
            assert _dev_sad(va, vb) == want, (h, w, oa, ob)


def test_sad_at_the_rounding_boundaries():
    """255 x at k + 0.5 (half-even), and the floats on either side of each."""
    half = (np.arange(256, dtype=np.float32) + np.float32(0.5)) / np.float32(255.0)
    vals = np.concatenate([half, np.nextafter(half, np.float32(-1)), np.nextafter(half, np.float32(2)),
                           np.arange(256, dtype=np.float32) / np.float32(255.0)]).astype(np.float32)
    g = np.random.default_rng(1)
    for _ in range(4):
        a = g.permutation(vals).astype(np.float32)
        b = g.permutation(vals).astype(np.float32)
        _check(a, b)
    assert _dev_sad(torch.from_numpy(half).cuda(), torch.zeros_like(torch.from_numpy(half)).cuda()) == int(
        _q8(half).sum())


@pytest.mark.parametrize("bits", [8, 16])
def test_sad_of_frames_from_integer_sources(bits):
    g = np.random.default_rng(bits)
    top = 256 if bits == 8 else 65536
    for hw in [(32, 36), (540, 960)]:
        u, v = g.integers(0, top, hw + (3,)), g.integers(0, top, hw + (3,))
        a = u.astype(np.float32) / np.float32(255.0)               # the readers' frames: u / 255 in float32
        b = v.astype(np.float32) / np.float32(255.0)
        _check(a, b)
        if bits == 8:                                              # the bytes come back exactly
            assert _np_sad(a, b) == int(np.abs(u - v).sum())
        else:
            assert _np_sad(a, b) == int(np.abs(np.minimum(u, 255) - np.minimum(v, 255)).sum())


def test_malformed_calls_raise_without_a_launch():
    a = torch.rand(8, 8, 3, device="cuda")
    b = torch.rand(8, 8, 3, device="cuda")
    out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    for x, y, o in [(a.double(), b, out), (a, b.cpu(), out), (a.cpu(), b.cpu(), out), (a[:, ::2], b[:, ::2], out),
                    (a, b[:7], out), (a, b.view(8, 24), out), (a.half(), b.half(), out), ("a", b, out)]:
        with pytest.raises(ValueError):
            K.frame_sad_q8(x, y, o)
    for o in [out.int(), torch.zeros(2, dtype=torch.int64, device="cuda"), out.cpu(), out.float(), "out"]:
        with pytest.raises(ValueError):
            K.frame_sad_q8(a, b, o)
    for args in [(_ffi.ptr(None), _ffi.ptr(b), 192, _ffi.ptr(out)), (_ffi.ptr(a), _ffi.ptr(None), 192, _ffi.ptr(out)),
                 (_ffi.ptr(a), _ffi.ptr(b), 192, _ffi.ptr(None)), (_ffi.ptr(a), _ffi.ptr(b), -1, _ffi.ptr(out))]:
        with pytest.raises(ValueError):
            _ffi.call("teco_frame_sad_q8", *args, _ffi.stream_ptr())
    torch.cuda.synchronize()
    assert int(out.item()) == -7                                   # nothing was written
    _ffi.call("teco_frame_sad_q8", _ffi.ptr(a), _ffi.ptr(b), 0, _ffi.ptr(out), _ffi.stream_ptr())
    assert int(out.item()) == 0                                    # n = 0: zeroed, nothing summed
    assert _dev_sad(a, b) == _np_sad(a.cpu().numpy(), b.cpu().numpy())


# ---- the command -----------------------------------------------------------------------------------------------------

LENGTHS, SEEDS = (9, 3, 7), (11, 12, 13)
STARTS = (0, 9, 12)


def _scene_rgb(lengths, seeds):
    """Seeded scenes of smooth noise (8x cubic up-sampling) drifting by one pixel a frame, uint8 RGB LR frames."""
    h, w = LR_HW
    out = []
    for L, seed in zip(lengths, seeds):
        g = np.random.default_rng(seed)
        base = cv2.resize(g.integers(0, 256, (h // 8 + 4, w // 8 + 4 + L, 3)).astype(np.uint8), None, fx=8, fy=8,
                          interpolation=cv2.INTER_CUBIC)
        out += [np.ascontiguousarray(base[8:8 + h, 8 + k:8 + k + w]) for k in range(L)]
    return out


def _write_input(d, frames, kind, first=1):
    """PNG files <first>.png .. (RGB frames as cv2 writes them), or a y4m stream of their I420 planes; returns the
    flags that read it and the RGB frames the engine receives (/ 255 of these)."""
    os.makedirs(d, exist_ok=True)
    if kind == "png":
        for k, f in enumerate(frames):
            cv2.imwrite(os.path.join(d, "%04d.png" % (first + k)), np.ascontiguousarray(f[:, :, ::-1]))
        return ["--input_dir_LR", d], frames
    planes = [cv2.cvtColor(f, cv2.COLOR_RGB2YUV_I420) for f in frames]
    path = os.path.join(d, "in.y4m")
    with open(path, "wb") as f:
        f.write(y4m.format_header(LR_HW[1], LR_HW[0]))
        for p in planes:
            f.write(b"FRAME\n" + p.tobytes())
    return ["--input_y4m", path], [cv2.cvtColor(p, cv2.COLOR_YUV2RGB_I420) for p in planes]


def _scores(rgb):
    from tests.test_scene_cuts_host import scores
    return scores([f.astype(np.float32) / np.float32(255.0) for f in rgb])


def _run(out, capsys, *args):
    capsys.readouterr()
    files = _main(out, *args)
    return files, capsys.readouterr().out


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["png", "y4m"])
def test_scenes_are_super_resolved_as_sequences_of_their_own(tmp_path, capsys, kind, precision):
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    rgb = _scene_rgb(LENGTHS, SEEDS)
    flags, got_rgb = _write_input(str(tmp_path / "all"), rgb, kind)
    s = _scores(got_rgb)
    assert [i for i in range(1, 19) if s[i] >= float(T)] == [9, 12]            # what the rule finds here
    common = ["--precision", precision, "--output_ext", "png"]
    files, log = _run(str(tmp_path / "cut"), capsys, *flags, *common, "--scene_threshold", T)
    assert [int(i) for i in re.findall(r"^scene cut before frame (\d+), score ", log, re.M)] == [9, 12]
    assert "frame number 31" in log                                           # 14 + 5 + 12 steps, warm-ups included
    assert len(files) == 19 and sorted(files) == ["output_%04d.png" % (k + 1) for k in range(19)]

    def alone(scene):
        a, L = STARTS[scene], LENGTHS[scene]
        f, _ = _write_input(str(tmp_path / ("scene%d" % scene)), rgb[a:a + L], kind, first=a + 1)
        got, _ = _run(str(tmp_path / ("alone%d" % scene)), capsys, *f, *common)
        # y4m input names its frames from 0001; PNG input keeps the files' names
        return {("output_%04d.png" % (a + int(n[7:11]))) if kind == "y4m" else n: v for n, v in got.items()}
    for scene in (0, 2):
        want = alone(scene)
        assert len(want) == LENGTHS[scene]
        for n, v in want.items():
            assert files[n] == v, (scene, n)
    # scene 2 (3 frames): the engine on f2, f1, f0, f1, f2, the first two outputs dropped
    prev = config.precision()
    try:
        _weights(precision)
        lr = [torch.from_numpy(f.astype(np.float32) / np.float32(255.0)).cuda() for f in got_rgb[9:12]]
        outs = InferenceEngine(*LR_HW, NRB).run_sequence([lr[2], lr[1], lr[0], lr[1], lr[2]], out="u8")
        for k, o in enumerate(outs[2:]):
            dec = cv2.imdecode(np.frombuffer(files["output_%04d.png" % (10 + k)], np.uint8), cv2.IMREAD_COLOR)
            assert np.array_equal(dec[:, :, ::-1], o[0].cpu().numpy()), k
    finally:
        config.set_precision(prev)
    # without the flag the second and third scenes start from the previous scene's detail
    plain, log = _run(str(tmp_path / "plain"), capsys, *flags, *common)
    assert "scene cut" not in log and len(plain) == 19
    assert all(plain[n] == files[n] for n in ("output_%04d.png" % (k + 1) for k in range(9)))
    third = alone(2)
    assert any(plain[n] != v for n, v in third.items())


@pytest.mark.parametrize("kind,extra", [("png", []), ("png", ["--outscale", "2", "--output_y4m"]),
                                        ("y4m", ["--output_y4m"])], ids=["png_jpg", "png_outscale_y4m", "y4m_y4m"])
def test_single_scene_writes_the_bytes_of_a_run_without_the_flag(tmp_path, capsys, kind, extra):
    rgb = _scene_rgb((8,), (31,))
    flags, got_rgb = _write_input(str(tmp_path / "in"), rgb, kind)
    assert max(_scores(got_rgb)[2:]) < float(T) and _scores(got_rgb)[1] < float(T)
    res = []
    for name, more in (("flag", ["--scene_threshold", T]), ("plain", [])):
        args = list(extra)
        if "--output_y4m" in args:
            args.insert(args.index("--output_y4m") + 1, str(tmp_path / (name + ".y4m")))
        files, log = _run(str(tmp_path / name), capsys, *flags, *args, *more)
        res.append((files, open(str(tmp_path / (name + ".y4m")), "rb").read() if "--output_y4m" in args else None))
        assert "scene cut" not in log
    assert res[0] == res[1]
    assert len(res[0][0]) == 8 or len(_read_y4m(str(tmp_path / "flag.y4m"))[1]) == 8


def _peak(tmp_path, n, kind, capsys):
    import main as M
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import stream_scenes
    d = tmp_path / ("%s%d" % (kind, n))
    rgb = _scene_rgb((4,) * (n // 4), range(100, 100 + n // 4))
    flags, _ = _write_input(str(d), rgb, kind)
    out = str(d / "o.y4m")
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    if kind == "y4m":
        reader = y4m.Y4MReader(flags[1])
        steps, name_of = reader.scenes(10.0), reader.name
    else:
        paths = [os.path.join(flags[1], "%04d.png" % (k + 1)) for k in range(n)]
        steps = stream_scenes(paths, False, 10.0, window_bytes=3 * LR_HW[0] * LR_HW[1] * 3)
        name_of = paths.__getitem__
    sink = None
    capsys.readouterr()
    try:
        first = next(steps)
        eng = InferenceEngine(first.frame.shape[0], first.frame.shape[1], NRB)
        sink = y4m.Y4MWriter(out, 4 * LR_HW[1], 4 * LR_HW[0])
        M.super_resolve_scenes(eng, name_of, itertools.chain([first], steps), str(d), "out", "png", None, sink)
    finally:
        steps.close()
        if sink is not None:
            sink.close()
    torch.cuda.synchronize()
    log = capsys.readouterr().out
    assert len(re.findall(r"^scene cut before frame", log, re.M)) == n // 4 - 1
    assert len(_read_y4m(out)[1]) == n
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("kind", ["y4m", "png"])
def test_peak_memory_flat_with_a_cut_every_4_frames(tmp_path, capsys, kind):
    from tecogan_b200 import config
    prev = config.precision()
    try:
        _weights("bf16")
        _peak(tmp_path, 12, kind, capsys)              # module loads, encoder and allocator warm-up
        short, long_ = _peak(tmp_path, 48, kind, capsys), _peak(tmp_path, 240, kind, capsys)
    finally:
        config.set_precision(prev)
    assert long_ - short < 4 * LR_HW[0] * LR_HW[1] * 3 * 4, (short, long_)


def test_reader_errors_are_raised_at_the_frame_that_needs_them(tmp_path, capsys):
    rgb = _scene_rgb((6, 5), (3, 4))
    flags, _ = _write_input(str(tmp_path / "y"), rgb, "y4m")
    data = open(flags[1], "rb").read()
    cut = str(tmp_path / "cut.y4m")
    with open(cut, "wb") as f:
        f.write(data[:-100])
    with pytest.raises(ValueError, match="frame 11 is truncated"):
        _run(str(tmp_path / "a"), capsys, "--input_y4m", cut, "--output_ext", "png", "--scene_threshold", T)
    pflags, _ = _write_input(str(tmp_path / "p"), rgb, "png")
    with open(os.path.join(pflags[1], "0011.png"), "wb") as f:
        f.write(b"not an image")
    with pytest.raises(ValueError, match="cannot decode"):
        _run(str(tmp_path / "b"), capsys, *pflags, "--output_ext", "png", "--scene_threshold", T)
