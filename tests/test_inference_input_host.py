"""CPU: the numpy restatement of cv2.GaussianBlur(frame, (0, 0), sigmaX=1.5) (tests/golden/gauss_blur_oracle.py), which
the device kernel of the inference input (tecogan_b200/csrc/gauss_blur.cu) is held to, equals cv2 bit for bit here: on
every width 2..40 (each class of the 3W-float row modulo 8) and height 2..20, on frame sizes the inference reads, on
uint16 frames, and on the recorded fixture (tests/golden/gauss_blur.npz)."""
import os

import cv2
import numpy as np
import pytest

from tests.conftest import GOLDEN
from tests.golden import gauss_blur_oracle as G
from tests.golden import make_golden_gauss_blur as MG

LARGE = [(576, 720), (480, 720), (576, 704), (534, 1280), (1080, 1921)]


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _check(frame):
    """Oracle vs cv2 on an RGB uint8/uint16 frame: the full blur, and the reference's input blur[::4, ::4] / 255."""
    rgb32 = frame.astype(np.float32)
    want = cv2.GaussianBlur(rgb32[:, :, ::-1], (0, 0), sigmaX=1.5)            # the reference's call, on BGR memory
    got = G.blur_bgr(np.ascontiguousarray(rgb32[:, :, ::-1]))
    assert _same(got, want), frame.shape
    ref = G.reference_input(np.ascontiguousarray(frame[:, :, ::-1]), True)
    assert _same(G.down4_rgb(frame), ref), frame.shape


def test_taps_are_cv2s():
    assert _same(G.TAPS, cv2.getGaussianKernel(13, 1.5, cv2.CV_32F).ravel())


def test_border101_is_cv2s():
    for n in range(2, 9):
        p = np.arange(-30, 30 + n)
        assert G.border101(p, n).tolist() == [cv2.borderInterpolate(int(q), n, cv2.BORDER_REFLECT_101) for q in p]


def test_fmaf_rounds_once():
    """a*b + c = 2^30 + 2^7 + 2^6 - 2^-34: just below a float32 midpoint, which the float64 sum rounds onto."""
    a, b = np.float32(8 * (1 + 2.0 ** -20)), np.float32(8 * (1 - 2.0 ** -20))
    c = np.float32(2.0 ** 30 + 2.0 ** 7)
    assert np.float32(float(a) * float(b) + float(c)) == np.float32(2.0 ** 30 + 2.0 ** 8)     # twice rounded
    assert G.fmaf(a, b, c) == c
    assert G.fmaf(a, b, -c) == -c
    assert G.fmaf(np.float32(3), np.float32(0.1), np.float32(0.2)) == np.float32(3 * float(np.float32(0.1)) + float(np.float32(0.2)))


@pytest.mark.parametrize("W", range(2, 41))
def test_oracle_equals_cv2_small(W):
    g = np.random.default_rng(W)
    for H in range(2, 21):
        _check(g.integers(0, 256, (H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("H,W", LARGE)
def test_oracle_equals_cv2_large(H, W):
    _check(np.random.default_rng(H * W).integers(0, 256, (H, W, 3)).astype(np.uint8))


@pytest.mark.parametrize("H,W", [(7, 9), (20, 33), (97, 180), (576, 720)])
def test_oracle_equals_cv2_uint16(H, W):
    _check(np.random.default_rng(H + W).integers(0, 65536, (H, W, 3)).astype(np.uint16))


def test_oracle_equals_fixture():
    z = np.load(os.path.join(GOLDEN, "gauss_blur.npz"))
    frames = MG.frames()
    assert len(z.files) == 2 * len(frames)
    for i, f in enumerate(frames):
        assert np.array_equal(z["frame%d" % i], f)
        got = G.blur_bgr(np.ascontiguousarray(f[:, :, ::-1]).astype(np.float32))[:, :, ::-1]
        assert _same(np.ascontiguousarray(got), z["blur%d" % i]), MG.CASES[i]


def test_one_pixel_side_is_refused():
    with pytest.raises(ValueError):
        G.blur_bgr(np.zeros((1, 8, 3), np.float32))
