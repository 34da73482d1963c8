"""Generate tests/golden/metrics.npz by executing the REFERENCE's own metric functions.

The reference's metrics.py cannot be imported (module-level cv2 / skimage / LPIPS imports and a flag-driven main loop), so
its pure-numpy functions `_rgb2ycbcr`, `to_uint8`, `psnr` and `crop_8x8` (metrics.py:37-70, 77-92) are taken out of the
file's syntax tree and executed unmodified with numpy (read from the checkout named by $TECOGAN_REFERENCE, never copied into the repo).
`ssim` (metrics.py:72-75) calls skimage.measure.compare_ssim, which is not installed: it is pinned in
tests/test_oracle_golden.py by a second derivation (direct window sums) instead.
Run once:  TECOGAN_REFERENCE=/path/to/TecoGAN python tests/golden/make_golden_metrics.py
"""
import ast
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.environ.get("TECOGAN_REFERENCE", "TecoGAN"), "metrics.py")
WANT = ("_rgb2ycbcr", "to_uint8", "psnr", "crop_8x8")


def reference_functions():
    tree = ast.parse(open(SRC).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in WANT]
    assert sorted(n.name for n in body) == sorted(WANT)
    ns = {"np": np}
    exec(compile(ast.Module(body=body, type_ignores=[]), SRC, "exec"), ns)
    return ns


def frames(seed, h, w, noise):
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([127 + 100 * np.sin(xx / 9.0 + c) * np.cos(yy / 7.0 - c) for c in range(3)], -1)
    tgt = np.clip(np.round(base + r.randn(h, w, 3) * 6), 0, 255).astype(np.uint8)
    out = np.clip(np.round(tgt.astype(np.float64) + r.randn(h, w, 3) * noise), 0, 255).astype(np.uint8)
    return tgt, out


def main():
    ref = reference_functions()
    kw = {}
    cases = [(0, 96, 128, 4.0), (1, 144, 180, 9.0), (2, 75, 101, 1.5), (3, 64, 64, 25.0)]
    kw["n_cases"] = np.int64(len(cases))
    for i, (seed, h, w, noise) in enumerate(cases):
        tgt, out = frames(seed, h, w, noise)
        ct, y, x = ref["crop_8x8"](tgt)
        co, _, _ = ref["crop_8x8"](out)
        kw["tgt%d" % i], kw["out%d" % i] = tgt, out
        kw["crop%d" % i] = np.array([y, x, ct.shape[0], ct.shape[1]], dtype=np.int64)
        kw["psnr_full%d" % i] = np.float64(ref["psnr"](tgt, out))
        kw["psnr_crop%d" % i] = np.float64(ref["psnr"](ct, co))
        if h * w <= 4096:      # the Y plane itself (float64) for one small case
            kw["y_full%d" % i] = ref["_rgb2ycbcr"](ref["to_uint8"](out, 0, 255), 255)[:, :, 0]
    path = os.path.join(HERE, "metrics.npz")
    np.savez_compressed(path, **kw)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
