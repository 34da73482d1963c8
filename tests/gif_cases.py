"""Seeded GIF encoder cases: each a batch [N, T, H, W, 3] uint8 of different animations (one call of the device encoder),
and the SHA-256 of every oracle file, which pins tests/golden/gif_oracle.py.  tests/test_gif_host.py checks the oracle
against cv2 and PIL and that the cases reach every rule; tests/test_gpu_gif.py holds the device to the same bytes."""
import hashlib

import numpy as np


def _smooth(rng, t, h, w, noise=6):
    """Clips that look like video: a moving colour gradient plus noise (many more than 256 colours)."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = []
    ph = rng.uniform(0, 6.28, 3)
    for k in range(t):
        f = np.stack([127 + 120 * np.sin(x / max(w, 1) * 3 + ph[c] + 0.3 * k + y / max(h, 1) * (c + 1)) for c in range(3)], -1)
        f += rng.normal(0, noise, f.shape)
        out.append(np.clip(np.rint(f), 0, 255))
    return np.stack(out).astype(np.uint8)


def _few_colours(rng, t, h, w, n):
    pal = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    return pal[rng.integers(0, n, (t, h, w))]


def _ties(t=2, h=6, w=8):
    """Median-cut ties: four colours of equal count, R and B ranges equal (an axis tie), then two splittable boxes of
    one count (a box tie)."""
    a = np.zeros((t, h, w, 3), dtype=np.uint8)
    cols = np.array([[0, 0, 0], [40, 0, 0], [0, 0, 40], [40, 0, 40]], dtype=np.uint8)
    a[:, : h // 2, : w // 2] = cols[0]
    a[:, : h // 2, w // 2:] = cols[1]
    a[:, h // 2:, : w // 2] = cols[2]
    a[:, h // 2:, w // 2:] = cols[3]
    return a


def _skewed():
    """One R range of 0..9: 13 pixels at 0, 19 at 9, so no v in [0, 8] has 2 count(R <= v) >= 32."""
    a = np.zeros((1, 4, 8, 3), dtype=np.uint8)
    a.reshape(-1, 3)[13:, 0] = 9
    return a


def cases():
    """{name: uint8 [N, T, H, W, 3]}"""
    rng = np.random.default_rng(2024)
    c = {}
    c["one_colour"] = np.stack([np.full((2, 5, 7, 3), v, dtype=np.uint8) for v in ((12, 200, 7), (255, 255, 255))])
    c["one_pixel"] = rng.integers(0, 256, (3, 1, 1, 1, 3), dtype=np.uint8)
    c["odd_lossless"] = np.stack([_few_colours(rng, 3, 17, 23, n) for n in (2, 50, 256)])
    c["ties"] = np.stack([_ties(), _ties()[:, ::-1].copy()])
    c["skewed"] = np.stack([_skewed(), _skewed()[:, ::-1].copy()])
    c["noise"] = rng.integers(0, 256, (2, 2, 70, 70, 3), dtype=np.uint8)
    c["lr_summary"] = np.stack([_smooth(rng, 10, 32, 32) for _ in range(4)])
    c["pingpong_lr"] = np.stack([_smooth(rng, 19, 32, 32) for _ in range(2)])
    c["pingpong_warp"] = np.stack([_smooth(rng, 18, 24, 40) for _ in range(2)])
    c["hr_frames"] = np.stack([_smooth(rng, 2, 128, 128, noise=3) for _ in range(2)])
    c["big"] = np.stack([_smooth(rng, 1, 256, 256, noise=2)])
    return c


def sha(data):
    return hashlib.sha256(data).hexdigest()[:16]


# SHA-256 (first 16 hex digits) of the oracle's file for every animation of every case
HASHES = {
    'one_colour': ['a1663e10b9979ab6', '6e732c300cfa2725'],
    'one_pixel': ['c311f56c92b36f5c', '91b3ba422e9ddef8', '5a8aa574632f17bc'],
    'odd_lossless': ['b3b8cd39444db786', 'b3d9ef6b96f0d15c', 'fcd5f53379b99189'],
    'ties': ['f701804006e44d69', '9c01f69c2c59479f'],
    'skewed': ['35bf9a79a2abebf7', '2a9da98f3260ce1f'],
    'noise': ['114b045b253d253f', '0c7fe8e8e0015d78'],
    'lr_summary': ['c85239997e6d61d1', 'afb42167c9d412cd', 'fa246741fb2a78b5', '6dfb5ef23c15c508'],
    'pingpong_lr': ['799b5253a46b40cd', '2388817d238a9501'],
    'pingpong_warp': ['6aad9624c4c197b9', 'b0334566e983fb4e'],
    'hr_frames': ['a4506645a48f552e', 'c239b24ddc334c08'],
    'big': ['577fa531a5cd6631'],
}
