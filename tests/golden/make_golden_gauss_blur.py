"""tests/golden/gauss_blur.npz: seeded RGB frames and cv2.GaussianBlur(frame, (0, 0), sigmaX=1.5) of each, computed as the
reference computes it (float32 copy of the frame, channel-reversed view; lib/dataloader.py:38-41).  A host's cv2 picks
its filter code by CPU at run time, so the tests compare the restatement (gauss_blur_oracle.py) and the device kernel
with these recorded outputs as well as with the cv2 they run beside.

Generate (needs cv2 4.13; the tests do not):  python tests/golden/make_golden_gauss_blur.py
Each case i stores `frame<i>` (uint8 or uint16 [H, W, 3] RGB) and `blur<i>` (float32 [H, W, 3], RGB).  Before anything
is written, the restatement is checked against every recorded blur.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "gauss_blur.npz")
# (H, W, dtype): every W mod 8 class (n = 3W floats per row), frames under 7 pixels, and a few wider rows
CASES = [(h, w, np.uint8 if (h + w) % 2 else np.uint16) for w in range(2, 18) for h in (2, 3, 5, 7, 11)] + [
    (37, 45, np.uint8), (59, 39, np.uint16), (29, 181, np.uint16), (33, 240, np.uint8)]
SEED = 20261017


def frames():
    g = np.random.default_rng(SEED)
    return [g.integers(0, np.iinfo(dt).max + 1, (h, w, 3)).astype(dt) for h, w, dt in CASES]


def main():
    import cv2
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from tests.golden import gauss_blur_oracle as G
    out = {}
    for i, f in enumerate(frames()):
        blur = cv2.GaussianBlur(f.astype(np.float32)[:, :, ::-1], (0, 0), sigmaX=1.5)[:, :, ::-1]
        mine = G.blur_bgr(np.ascontiguousarray(f[:, :, ::-1]).astype(np.float32))[:, :, ::-1]
        assert np.array_equal(mine.view(np.uint32), blur.view(np.uint32)), CASES[i]
        out["frame%d" % i], out["blur%d" % i] = f, np.ascontiguousarray(blur)
    np.savez_compressed(OUT, **out)
    print("wrote %s: %d cases, %d bytes" % (OUT, len(CASES), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
