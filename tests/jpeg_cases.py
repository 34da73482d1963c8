"""Seeded RGB uint8 frames for the JPEG encoder tests (tests/test_jpeg_host.py, tests/test_gpu_jpeg.py): HR sizes,
degenerate shapes, every residue of H and W modulo 16 that changes the block layout, constant frames, and frames built
from chosen quantised coefficients (ZRL runs, blocks ending on position 63, the largest size categories).  numpy only."""
import numpy as np

from tests.golden import jpeg_oracle as J
from tests.png_cases import noise, smooth

SIDES = (1, 7, 8, 9, 15, 16, 17, 24, 33)


def _idct_basis():
    k = np.arange(8)
    c = np.where(k == 0, np.sqrt(1 / 8), np.sqrt(2 / 8))[:, None] * np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16)
    return c                                            # c[u, x]: orthonormal DCT-II basis


def grey_block(zz_values, seed):
    """An 8x8 grey block (Y = the pixel value exactly, Cb = Cr = 128) whose quantised luma coefficients are zz_values
    (zigzag position -> value, every other position 0): the inverse DCT of the target, rounded with a seeded dither
    until the forward transform gives the target back."""
    target = np.zeros(64, np.int64)
    for pos, v in zz_values.items():
        target[pos] = v
    nat = np.zeros(64)
    nat[J.ZIGZAG] = target * J.quant_table(J.LUMA_BASE)[J.ZIGZAG]
    c = _idct_basis()
    f = c.T @ nat.reshape(8, 8) @ c + 128
    g = np.random.default_rng(seed)
    for _ in range(2000):
        b = np.clip(np.floor(f + g.random((8, 8))), 0, 255).astype(np.int64)
        q = J.quantise(J.fdct(b - 128), J.quant_table(J.LUMA_BASE)).reshape(64)[J.ZIGZAG]
        if np.array_equal(q, target):
            return b.astype(np.uint8)
    raise AssertionError("no block found for %s" % zz_values)


def _grey(y):
    return np.repeat(y[:, :, None], 3, 2)


def runs():
    """One MCU: runs of 16 and 32 zeros before a nonzero AC (one and two ZRLs), a run of 47 (two ZRLs + run 15),
    blocks whose last coefficient (position 63) is nonzero, so no EOB follows."""
    a = grey_block({0: 3, 1: 2, 18: -2, 51: 1, 63: 1}, 1)
    b = grey_block({0: -2, 48: 1, 63: -1}, 2)
    c = grey_block({0: 1, 63: 2}, 3)
    d = grey_block({0: -1, 1: 1, 33: -1}, 4)
    return _grey(np.block([[a, b], [c, d]]))


def extremes():
    """Black and white blocks next to each other (DC differences of 1 020, size category 10, the largest: a DC is
    -512 .. 508 at Q = 2) and half-black half-white blocks (AC category 10, the largest in baseline JPEG)."""
    k, w = np.zeros((8, 8), np.uint8), np.full((8, 8), 255, np.uint8)
    lr, tb = np.concatenate([k[:, :4], w[:, 4:]], 1), np.concatenate([w[:4], k[4:]], 0)
    return _grey(np.block([[k, w, lr, w], [w, k, tb, k]]))


def cases():
    """name -> frame, every frame the GPU test compares with cv2."""
    c = {
        "smooth_32x32": smooth(32, 32, 1), "smooth_128x128": smooth(128, 128, 2), "smooth_576x720": smooth(576, 720, 3),
        "smooth_1080x1920": smooth(1080, 1920, 4), "smooth_2160x3840": smooth(2160, 3840, 5),
        "noise_1x1": noise(1, 1, 6), "noise_1x257": noise(1, 257, 7), "noise_300x1": noise(300, 1, 8),
        "noise_576x720": noise(576, 720, 9), "smooth_99x201": smooth(99, 201, 10),
        "constant": np.full((64, 300, 3), 7, np.uint8), "constant_1x1": np.zeros((1, 1, 3), np.uint8),
        "constant_37x45": np.tile(np.array([200, 30, 90], np.uint8), (37, 45, 1)),
        "runs": runs(), "extremes": extremes(),
    }
    for i, h in enumerate(SIDES):
        for j, w in enumerate(SIDES):
            c["grid_%dx%d" % (h, w)] = (noise if (i + j) % 2 else smooth)(h, w, 100 + 10 * i + j)
    return c


# frames small enough for the host oracle (numpy and a Python entropy coder) in tests/test_jpeg_host.py
BIG = ("smooth_1080x1920", "smooth_2160x3840")
