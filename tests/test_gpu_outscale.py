"""GPU: the output resize of `main.py --outscale`.  teco_resize_lanczos4_u8 equals cv2.resize(INTER_LANCZOS4) byte for
byte on the host sweep (tests/test_resize_host.py), on the edges of its tiles and of its grid-stride loop, on frames
with row pitches and offsets, and on 8K -> 4K; malformed calls raise before a launch and write nothing.  The inference
command with --outscale writes cv2.imwrite(cv2.resize(the frame of the run without the flag, INTER_LANCZOS4)) byte for
byte, as PNG and as JPEG; --outscale 4 writes the files of the run without the flag; its device memory does not grow
with the sequence."""
import itertools
import os

import cv2
import numpy as np
import pytest
import torch

from tecogan_b200 import _ffi
from tecogan_b200 import kernels as K
from tecogan_b200 import resize as RZ
from tests.test_gpu_inference_stream import LR_FRAME_BYTES, LR_HW, NRB, _flags, _weights, _write_seq
from tests.test_resize_host import sweep_sizes

pytestmark = pytest.mark.gpu


def _cv2(frame, h, w):
    return cv2.resize(frame, (w, h), interpolation=cv2.INTER_LANCZOS4)


def _kernel(frame, h, w):
    out = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
    return K.resize_lanczos4(torch.from_numpy(frame).cuda(), out).cpu().numpy()


def _check(frame, h, w):
    got = _kernel(frame, h, w)
    assert np.array_equal(got, _cv2(frame, h, w)), (frame.shape, h, w)


@pytest.mark.parametrize("n", range(1, 41))
def test_kernel_equals_cv2_sweep(n):
    g = np.random.default_rng(100 + n)
    for H, W, h, w in sweep_sizes(n):
        _check(g.integers(0, 256, (H, W, 3)).astype(np.uint8), h, w)
        _check(g.integers(0, 256, (W, H, 3)).astype(np.uint8), w, h)


# Tiles are 64 output columns by tile_rows(H_in, H_out) output rows: 12 at a 4x down-scale, 24 at 2x, 64 from 0.72x up.
EDGES = [((4 * h, 4 * w), (h, w)) for h, w in [(11, 63), (12, 64), (13, 65), (24, 127), (25, 129)]] + \
        [((2 * h, 2 * w), (h, w)) for h, w in [(23, 63), (24, 64), (25, 65), (47, 128), (49, 193)]] + \
        [((h // 2 + 1, w // 2 + 1), (h, w)) for h, w in [(63, 63), (64, 64), (65, 65), (128, 191), (129, 192)]]


@pytest.mark.parametrize("src,dst", EDGES)
def test_kernel_equals_cv2_tile_edges(src, dst):
    _check(np.random.default_rng(src[0] * dst[1]).integers(0, 256, src + (3,)).astype(np.uint8), *dst)


@pytest.mark.parametrize("src,dst", [((4320, 7680), (2160, 3840)), ((2160, 3840), (1620, 2880)),
                                     ((1080, 1920), (2160, 3840)), ((2160, 3840), (540, 960)),
                                     ((540, 960), (8640, 15360))])
def test_kernel_equals_cv2_grid_stride(src, dst):
    """Thousands of tiles: each CTA of the persistent grid takes many."""
    _check(np.random.default_rng(src[1] + dst[0]).integers(0, 256, src + (3,)).astype(np.uint8), *dst)


@pytest.mark.parametrize("v", [0, 255])
def test_kernel_equals_cv2_constant(v):
    for (H, W), (h, w) in [((7, 9), (14, 18)), ((40, 40), (10, 10)), ((256, 320), (384, 480))]:
        _check(np.full((H, W, 3), v, np.uint8), h, w)


def test_pitch_offset_and_nothing_written_outside():
    """src and dst as row-strided views at odd byte offsets inside larger buffers; the bytes around dst stay put."""
    g = np.random.default_rng(9)
    for (H, W), (h, w) in [((37, 53), (74, 106)), ((128, 144), (96, 108)), ((120, 160), (90, 120))]:
        frame = g.integers(0, 256, (H, W, 3)).astype(np.uint8)
        sp, dp = 3 * W + 7, 3 * w + 5
        sbuf = torch.from_numpy(g.integers(0, 256, 1 + H * sp).astype(np.uint8)).cuda()
        src = sbuf[1:].as_strided((H, W, 3), (sp, 3, 1))
        src.copy_(torch.from_numpy(frame))
        guard = 4096
        dbuf = torch.full((2 * guard + h * dp,), 0xA5, dtype=torch.uint8, device="cuda")
        dst = dbuf[guard + 3:].as_strided((h, w, 3), (dp, 3, 1))
        K.resize_lanczos4(src, dst)
        torch.cuda.synchronize()
        assert np.array_equal(dst.cpu().numpy(), _cv2(frame, h, w))
        mask = torch.ones_like(dbuf, dtype=torch.bool)
        rows = (guard + 3 + torch.arange(h, device="cuda")[:, None] * dp + torch.arange(3 * w, device="cuda")[None, :])
        mask[rows.flatten()] = False
        assert bool((dbuf[mask] == 0xA5).all())


def test_malformed_calls_raise_without_a_launch():
    src = torch.from_numpy(np.random.default_rng(2).integers(0, 256, (16, 20, 3)).astype(np.uint8)).cuda()
    dst = torch.full((24, 30, 3), 0x5A, dtype=torch.uint8, device="cuda")
    tabs = RZ.tables(16, 20, 24, 30, src.device)
    bad = [
        (src.float(), dst, None), (src, dst.float(), None), (src.cpu(), dst, None), (src, dst.cpu(), None),
        (src[:, :, :2], dst, None), (src, torch.zeros((24, 30, 4), dtype=torch.uint8, device="cuda"), None),
        (src[0], dst, None), (src.permute(1, 0, 2), dst, None), (src[:, ::2], dst, None),
        (torch.zeros((16, 20, 3), dtype=torch.uint8, device="cuda"), dst[:, :, :], (tabs[1], tabs[0])),
        (src, dst, (tabs[0][:-1], tabs[1])), (src, dst, (tabs[0].long(), tabs[1])), (src, dst, (tabs[0].cpu(), tabs[1])),
        (torch.zeros((97, 20, 3), dtype=torch.uint8, device="cuda"), dst, None),          # 97 > 4 * 24 rows
        (torch.zeros((24, 121, 3), dtype=torch.uint8, device="cuda"), dst, None),         # 121 > 4 * 30 columns
        (torch.zeros((0, 20, 3), dtype=torch.uint8, device="cuda"), dst, None),
        (src, "frame", None),
    ]
    for s, d, t in bad:
        with pytest.raises(ValueError):
            K.resize_lanczos4(s, d, t)
    xt, yt = _ffi.ptr(tabs[0]), _ffi.ptr(tabs[1])
    sptr, dptr = _ffi.ptr(src), _ffi.ptr(dst)
    for args in [(sptr, 60, 16, 20, dptr, 90, 24, 30, xt, _ffi.ptr(None)), (sptr, 59, 16, 20, dptr, 90, 24, 30, xt, yt),
                 (sptr, 60, 16, 20, dptr, 89, 24, 30, xt, yt), (sptr, 60, 0, 20, dptr, 90, 24, 30, xt, yt),
                 (sptr, 60, 16, 20, dptr, 90, 24, 65536, xt, yt), (sptr, 60, 16, 20, dptr, 90, 3, 30, xt, yt)]:
        with pytest.raises(ValueError):
            _ffi.call("teco_resize_lanczos4_u8", *args, _ffi.stream_ptr())
    torch.cuda.synchronize()
    assert bool((dst == 0x5A).all())
    K.resize_lanczos4(src, dst, tabs)                       # later launches still work
    assert np.array_equal(dst.cpu().numpy(), _cv2(src.cpu().numpy(), 24, 30))


# ---- the inference command -----------------------------------------------------------------------------------------

def _main(seq, out, ext, *extra):
    import main as M
    from tecogan_b200 import config
    prev, cuda = config.precision(), os.environ.get("CUDA_VISIBLE_DEVICES")
    try:
        M.main(["--mode", "inference", "--checkpoint", "random:5", "--num_resblock", str(NRB), "--output_pre", "",
                "--output_ext", ext, "--cudaID", cuda or "0", "--input_dir_LR", seq, "--output_dir", out] + list(extra))
    finally:
        config.set_precision(prev)
        if cuda is None:
            os.environ.pop("CUDA_VISIBLE_DEVICES", None)
        else:
            os.environ["CUDA_VISIBLE_DEVICES"] = cuda
    return {n: open(os.path.join(out, n), "rb").read() for n in sorted(os.listdir(out))}


@pytest.fixture(scope="module")
def plain(tmp_path_factory):
    """The sequence and the files of the run without the flag, as PNG and as JPEG."""
    d = tmp_path_factory.mktemp("outscale")
    seq = _write_seq(str(d / "seq"), 9, seed=21)
    return seq, {ext: _main(seq, str(d / ("plain_" + ext)), ext) for ext in ("png", "jpg")}


@pytest.mark.parametrize("s,ext", list(itertools.product([1.5, 2.0, 2.5, 8.0], ["png", "jpg"])))
def test_main_outscale_equals_cv2_resize_of_the_plain_run(plain, tmp_path, s, ext):
    seq, files = plain
    got = _main(seq, str(tmp_path / "out"), ext, "--outscale", str(s))
    h, w = int(LR_HW[0] * s), int(LR_HW[1] * s)
    assert sorted(got) == [n[:-3] + ext for n in sorted(files["png"])] and len(got) == 9
    for name, data in got.items():
        bgr = cv2.imdecode(np.frombuffer(files["png"][name[:-3] + "png"], np.uint8), cv2.IMREAD_UNCHANGED)
        want = str(tmp_path / ("want." + ext))
        assert cv2.imwrite(want, _cv2(bgr, h, w))
        with open(want, "rb") as f:
            assert data == f.read(), (s, ext, name)


@pytest.mark.parametrize("ext", ["png", "jpg"])
def test_main_outscale_4_writes_the_plain_files(plain, tmp_path, ext):
    seq, files = plain
    assert _main(seq, str(tmp_path / "out"), ext, "--outscale", "4") == files[ext]


def _peak(tmp_path, n, window, out_hw):
    import gc
    import main as M
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_paths, padded, stream_inputs
    seq = _write_seq(str(tmp_path / ("seq%d" % n)), n, seed=5)
    out = str(tmp_path / ("out%d" % n))
    os.makedirs(out)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    paths, down = inference_paths(_flags(seq))
    frames = stream_inputs(paths, down, window_bytes=window)
    try:
        first = next(frames)
        eng = InferenceEngine(first.shape[0], first.shape[1], NRB)
        M.super_resolve_frames(eng, padded(paths), itertools.chain([first], frames), out, "out", "jpg", out_hw)
    finally:
        frames.close()
    torch.cuda.synchronize()
    assert len(os.listdir(out)) == n
    return torch.cuda.max_memory_allocated() - base


def test_peak_memory_flat_in_sequence_length(tmp_path):
    from tecogan_b200 import config
    prev = config.precision()
    window = 4 * LR_FRAME_BYTES
    out_hw = RZ.out_size(LR_HW[0], LR_HW[1], 2.5)
    try:
        _weights("bf16")
        _peak(tmp_path, 12, window, out_hw)           # module loads, tables, encoder and allocator warm-up
        short, long_ = _peak(tmp_path, 48, window, out_hw), _peak(tmp_path, 240, window, out_hw)
    finally:
        config.set_precision(prev)
    assert long_ - short < 4 * LR_FRAME_BYTES * 4, (short, long_)
