"""CPU: the output resize of `main.py --outscale` without a device.  The numpy restatement of cv2 4.13's fixed-point
INTER_LANCZOS4 (tests/golden/resize_oracle.py), which teco_resize_lanczos4_u8 is held to, equals cv2.resize byte for
byte on every side 1..40 at the ratios the flag produces, on exact-position (fx = 0) and 1-pixel cases and on video
sizes; the package's coefficient tables (tecogan_b200/resize.py) equal the oracle's and keep every tile's source rows
inside the kernel's shared memory; --outscale is an opt-in flag with Real-ESRGAN's size rule, refused out of range and
for training."""
import math

import cv2
import numpy as np
import pytest

from tecogan_b200 import resize as RZ
from tests.golden import resize_oracle as R

RATIOS = [1 / 4, 3 / 8, 1 / 2, 5 / 8, 3 / 4, 7 / 8, 1, 9 / 8, 3 / 2, 2, 4]
IRRATIONAL = [1 / math.sqrt(2), 2 / math.e, math.pi / 2, math.sqrt(7)]     # sizes no simple ratio gives
LARGE = [((1080, 1920), (540, 960)), ((4320, 7680), (2160, 3840)), ((270, 480), (1080, 1920))]


def _cv2(frame, h, w):
    return cv2.resize(frame, (w, h), interpolation=cv2.INTER_LANCZOS4)


def _check(frame, h, w):
    want, got = _cv2(frame, h, w), R.resize(frame, h, w)
    assert got.shape == want.shape == (h, w, 3) and got.dtype == np.uint8
    assert np.array_equal(got, want), (frame.shape, h, w)


def sweep_sizes(n):
    """(H, W, h, w) cases of input side n: n x (41 - n) at every ratio (each side rounded up, so no axis is
    down-scaled more than 4x) and at ratios no fraction of small integers gives."""
    m = 41 - n
    return [(n, m, max(1, math.ceil(n * r)), max(1, math.ceil(m * r))) for r in RATIOS + IRRATIONAL]


@pytest.mark.parametrize("n", range(1, 41))
def test_oracle_equals_cv2_sweep(n):
    g = np.random.default_rng(n)
    for H, W, h, w in sweep_sizes(n):
        _check(g.integers(0, 256, (H, W, 3)).astype(np.uint8), h, w)
        _check(g.integers(0, 256, (W, H, 3)).astype(np.uint8), w, h)


def test_exact_positions_take_the_1e30_branch():
    """fx = 0 at every output of an odd integer down-scale and of an unchanged side: tap 3 alone, weight 2048."""
    for n_in, n_out in [(21, 7), (30, 10), (17, 17), (1, 1)]:
        base, coef = R.axis_table(n_in, n_out)[0::2]
        assert (coef[:, 3] == 2048).all() and (np.delete(coef, 3, axis=1) == 0).all(), (n_in, n_out)
    g = np.random.default_rng(5)
    for (H, W), (h, w) in [((21, 30), (7, 10)), ((17, 30), (17, 10)), ((21, 17), (7, 17)), ((9, 12), (9, 12))]:
        f = g.integers(0, 256, (H, W, 3)).astype(np.uint8)
        _check(f, h, w)
    f = g.integers(0, 256, (13, 19, 3)).astype(np.uint8)
    assert np.array_equal(R.resize(f, 13, 19), f)          # the identity coefficients copy the frame


def test_one_pixel_sides():
    g = np.random.default_rng(1)
    for (H, W), (h, w) in [((1, 1), (1, 1)), ((1, 1), (4, 4)), ((1, 1), (3, 16)), ((1, 9), (2, 18)), ((9, 1), (5, 1)),
                           ((1, 40), (1, 10)), ((40, 1), (60, 4)), ((4, 4), (1, 1)), ((2, 7), (1, 2))]:
        _check(g.integers(0, 256, (H, W, 3)).astype(np.uint8), h, w)


@pytest.mark.parametrize("src,dst", LARGE)
def test_oracle_equals_cv2_video_sizes(src, dst):
    f = np.random.default_rng(src[0]).integers(0, 256, src + (3,)).astype(np.uint8)
    _check(f, *dst)


@pytest.mark.parametrize("v", [0, 255])
def test_oracle_equals_cv2_constant(v):
    """Saturated frames: the negative lobes round through the clamp at both ends."""
    for (H, W), (h, w) in [((7, 9), (14, 18)), ((40, 40), (10, 10)), ((33, 47), (50, 70))]:
        _check(np.full((H, W, 3), v, np.uint8), h, w)


PAIRS = [(n_in, n_out) for n_in in (1, 2, 7, 40, 480, 1920, 7680) for n_out in
         sorted({max(1, math.ceil(n_in / 4)), max(1, n_in // 2), n_in, n_in * 3 // 2 + 1, 2 * n_in, 4 * n_in})]


@pytest.mark.parametrize("n_in,n_out", PAIRS + [(3840, 2880), (1920, 3840), (7680, 3840), (960, 2563)])
def test_package_tables_equal_the_oracle_s(n_in, n_out):
    base, coef = RZ.axis_table(n_in, n_out)
    want_base, _, want_coef = R.axis_table(n_in, n_out)
    assert base.dtype == np.int32 and coef.dtype == np.int16
    assert np.array_equal(base, want_base) and np.array_equal(coef, want_coef)


# teco_resize_lanczos4_u8's tile height (tecogan_b200/csrc/resize.cu::tile_rows), restated: its shared memory holds the
# horizontal results of kMaxRows = 56 source rows per tile.
def _tile_rows(H_in, H_out):
    return min(64, int((56 - 10) / (H_in / H_out)) + 1)


@pytest.mark.parametrize("H_in", [4, 37, 540, 1080, 2160, 4320, 8640, 65532])
def test_tile_source_rows_fit_shared_memory(H_in):
    """Over the accepted range (H_in <= 4 H_out) no tile needs more than 56 source rows."""
    outs = {max(1, math.ceil(H_in / 4)), H_in // 4 + 1, H_in // 3, H_in // 2 + 1, H_in, 2 * H_in + 1, 4 * H_in}
    for H_out in sorted(o for o in outs if 1 <= o <= 65535 and H_in <= 4 * o):
        base, _ = RZ.axis_table(H_in, H_out)
        th = _tile_rows(H_in, H_out)
        for y0 in range(0, H_out, th):
            y1 = min(y0 + th, H_out) - 1
            lo, hi = max(base[y0] - 3, 0), min(base[y1] + 4, H_in - 1)
            assert hi - lo + 1 <= 56, (H_in, H_out, y0)


def test_outscale_flag_is_opt_in():
    import main as M
    from tests.test_train_monitoring_host import PARENT_FLAG_DEFAULTS
    assert vars(M.parse_flags([])) == PARENT_FLAG_DEFAULTS
    assert not hasattr(M.parse_flags([]), "outscale")
    assert M.parse_flags(["--outscale", "2.5"]).outscale == 2.5
    assert vars(M.parse_flags(["--outscale=1.5"])) == dict(PARENT_FLAG_DEFAULTS, outscale=1.5)


def test_output_size_rule():
    import argparse
    import main as M
    assert RZ.out_size(540, 960, 2.67) == (int(540 * 2.67), int(960 * 2.67)) == (1441, 2563)
    assert RZ.out_size(720, 1280, 1.5) == (1080, 1920)
    assert RZ.out_size(1080, 1920, 2) == (2160, 3840)
    assert RZ.out_size(7, 9, 1.1) == (7, 9)                 # int() truncates
    assert M.outscale_size(argparse.Namespace(), 540, 960) == (2160, 3840)
    assert M.outscale_size(argparse.Namespace(outscale=4.0), 540, 960) == (2160, 3840)
    assert M.outscale_size(argparse.Namespace(outscale=16.0), 33, 47) == (528, 752)
    assert M.outscale_size(argparse.Namespace(outscale=1.0), 33, 47) == (33, 47)


@pytest.mark.parametrize("argv", [["--outscale", "0.5"], ["--outscale", "0.999"], ["--outscale", "16.01"],
                                  ["--outscale", "nan"], ["--outscale", "inf"], ["--outscale", "-2"],
                                  ["--mode", "train", "--outscale", "2"], ["--mode", "train", "--outscale", "4"]])
def test_outscale_refused(argv, tmp_path, monkeypatch):
    """Refused before anything is set up: no environment change, no output directory."""
    import argparse
    import os
    import main as M
    monkeypatch.delenv("CUDA_VISIBLE_DEVICES", raising=False)
    out = str(tmp_path / "out")
    with pytest.raises(ValueError, match="outscale"):
        M.main(argv + ["--output_dir", out, "--checkpoint", "random:1"])
    assert not os.path.exists(out) and "CUDA_VISIBLE_DEVICES" not in os.environ
    if "train" not in argv:
        with pytest.raises(ValueError, match="outscale"):
            M.outscale_size(argparse.Namespace(outscale=float(argv[1])), 8, 8)


def test_wrapper_refuses_cpu_tensors():
    import torch
    from tecogan_b200 import kernels as K
    with pytest.raises(ValueError):
        K.resize_lanczos4(torch.zeros((8, 8, 3), dtype=torch.uint8), torch.zeros((16, 16, 3), dtype=torch.uint8))
