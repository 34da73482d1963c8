"""tests/golden/tof.npz: cv2's Farneback flows and the reference loop's tOF values, and `load()`, which rebuilds the
fixture's inputs and expected flows for the tests.

Generate (needs cv2; the tests do not):  python tests/golden/make_golden_tof.py
Inputs are not stored: `inputs()` and `sequence()` derive them from calendar_lr.npz (7 real 144x180 frames) with integer
numpy arithmetic only.  Expected values are cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0)
and the loop of metrics.py:135-169 (with cv2's cvtColor).

A full float32 flow barely compresses (its pixel-to-pixel noise is about 1e-3 px), so each case stores cv2's flow in two
parts:
  - `dflow<i>`: cv2's flow minus the host restatement's (tests/golden/farneback_oracle.py), in units of QUANT = 2^-24 px,
    int16.  `load()` adds it back to the restatement's flow; the rebuilt flow is cv2's to within 3e-8 px.
  - `sample<i>`: cv2's exact float32 flow at every SAMPLE-th row and column.  It anchors the restatement independently of
    `dflow` (tests/test_tof_host.py) and checks the rebuilt flow (to 1e-7 px).
`ill<i>` (bit-packed) marks the pixels whose final 2x2 system is near-singular: smallest eigenvalue of the box-mean
matrix below ILL_EIG, from the restatement.  There a 1e-7 change of an input moves cv2's own flow by up to ~1e-3 px
between its SIMD and scalar builds.

Checked here, before anything is written:
  - COLOR_RGB2GRAY == (9798 R + 19235 G + 3735 B + 16384) >> 15 over all 2^24 colours;
  - the restatement against cv2's flow of every case: |d| <= 1e-3 px outside the near-singular pixels, <= 2e-2 px on
    them, mean |d| <= 1e-5 px;
  - the rebuilt flow against cv2's.
"""
import functools
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden import farneback_oracle as F          # noqa: E402

ILL_EIG = 0.05
PARAMS = (None, 0.5, 3, 15, 3, 5, 1.2, 0)
CUTFR = 2
QUANT = 2.0 ** -24
SAMPLE = 7


def up2(a):
    """x2 in both directions: pixel repeat, then a [1 2 1]/4 smoothing in each direction (integer arithmetic)."""
    a = np.repeat(np.repeat(a.astype(np.int64), 2, 0), 2, 1)
    for ax in (0, 1):
        a = np.roll(a, 1, ax) + 2 * a + np.roll(a, -1, ax)
    return ((a + 8) // 16).astype(np.uint8)


def calendar():
    return np.load(os.path.join(HERE, "calendar_lr.npz"))["full_u8"]


def inputs(full):
    """[(name, prev [P,H,W] uint8 grey, next [P,H,W])] of the cases, from the calendar frames."""
    g = [F.grey(f) for f in full]
    big, nxt = up2(g[3]), up2(g[4])
    flat0, flat1 = g[1].copy(), g[2].copy()
    flat0[40:110, 50:150] = 118                                # a textureless block, the same in both frames
    flat1[40:110, 50:150] = 118
    cases = [
        ("calendar 144x180", [(g[0], g[1]), (g[2], g[3])]),
        ("x2 288x360", [(up2(g[2]), up2(g[3]))]),
        ("metric config 128x128", [(g[0][8:136, 26:154], g[1][8:136, 26:154])]),
        ("ragged 97x131", [(g[4][20:117, 30:161], g[5][20:117, 30:161])]),
        ("32x32", [(g[5][40:72, 60:92], g[6][40:72, 60:92])]),
        ("large motion (10, 12) px", [(big[40:232, 40:296], nxt[30:222, 28:284])]),
        ("flat block", [(flat0, flat1)]),
    ]
    return [(name, np.stack([np.ascontiguousarray(a) for a, _ in pairs]), np.stack([np.ascontiguousarray(b) for _, b in pairs]))
            for name, pairs in cases]


def sequence(full):
    """7-frame target / result sequence: the result is the target blurred horizontally ([1 2 1]/4), moved one pixel to
    the right on odd frames (temporal jitter, which tOF is there to see), plus a hashed noise pattern in -8..8 that
    changes from frame to frame (integer arithmetic, no random generator)."""
    t = full.astype(np.int64)
    soft = (np.roll(t, 1, 2) + 2 * t + np.roll(t, -1, 2) + 2) // 4
    soft = np.stack([np.roll(f, k % 2, 1) for k, f in enumerate(soft)])
    n, y, x, c = np.meshgrid(*(np.arange(s) for s in t.shape), indexing="ij")
    pattern = (((x * 7919 + y * 104729 + n * 1299709 + c * 15485863) * 2654435761) >> 13) % 17 - 8
    return full.copy(), np.clip(soft + pattern, 0, 255).astype(np.uint8)


@functools.lru_cache(maxsize=1)
def load():
    """Everything the tests need, as a dict: prev<i> / next<i> (grey [P,H,W]), flow<i> (cv2's flow, rebuilt),
    sample<i>, ill<i> (bool [P,H,W]), names, n_cases, seq_tgt / seq_out (RGB [7,H,W,3]), seq_tof, cutfr."""
    g = np.load(os.path.join(HERE, "tof.npz"), allow_pickle=False)
    full = calendar()
    out = {"names": g["names"], "n_cases": int(g["n_cases"]), "seq_tof": g["seq_tof"], "cutfr": int(g["cutfr"])}
    for i, (name, prev, nxt) in enumerate(inputs(full)):
        assert str(g["names"][i]) == name, (i, name)
        base = np.stack([F.farneback(a, b) for a, b in zip(prev, nxt)])
        flow = (base.astype(np.float64) + g["dflow%d" % i].astype(np.float64) * QUANT).astype(np.float32)
        ill = np.unpackbits(g["ill%d" % i], count=prev.size).reshape(prev.shape).astype(bool)
        out.update({"prev%d" % i: prev, "next%d" % i: nxt, "flow%d" % i: flow, "sample%d" % i: g["sample%d" % i],
                    "ill%d" % i: ill})
    out["seq_tgt"], out["seq_out"] = sequence(full)
    return out


def reference_tof(tgt, out):
    """metrics.py:135-169 with cv2: per-frame tOF list of a target / result sequence."""
    import cv2
    tofs, pre_t, pre_o = [], None, None
    for i in range(CUTFR, len(tgt) - CUTFR):
        o, t = out[i], tgt[i]
        if t.shape[0] < o.shape[0] or t.shape[1] < o.shape[1]:
            o = o[:t.shape[0], :t.shape[1]]
        og, tg = cv2.cvtColor(np.ascontiguousarray(o), cv2.COLOR_RGB2GRAY), cv2.cvtColor(np.ascontiguousarray(t), cv2.COLOR_RGB2GRAY)
        if i > CUTFR:
            t_of = cv2.calcOpticalFlowFarneback(pre_t, tg, *PARAMS)
            o_of = cv2.calcOpticalFlowFarneback(pre_o, og, *PARAMS)
            y, x, h, w = F.crop_window(*t_of.shape[:2])
            d = np.absolute(t_of[y:y + h, x:x + w] - o_of[y:y + h, x:x + w])
            tofs.append(np.sqrt(np.sum(d * d, axis=-1)).mean())
        pre_t, pre_o = tg, og
    return np.array(tofs, np.float64)


def main():
    import cv2
    c = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY), F.grey(rgb)), "RGB2GRAY formula"
    full = calendar()
    out, names, refs = {}, [], []
    for i, (name, prev, nxt) in enumerate(inputs(full)):
        ref = np.stack([cv2.calcOpticalFlowFarneback(a, b, *PARAMS) for a, b in zip(prev, nxt)])
        ill, base = [], []
        for p in range(prev.shape[0]):
            mine, lmin = F.farneback(prev[p], nxt[p], conditioning=True)
            bad = lmin < ILL_EIG
            d = np.abs(mine - ref[p]).max(-1)
            print("%-26s pair %d %dx%d levels %d: max |d| %.2e (%.2e on %d near-singular px), mean %.2e"
                  % (name, p, prev.shape[1], prev.shape[2], F.num_levels(*prev.shape[1:]), d[~bad].max(),
                     d[bad].max() if bad.any() else 0.0, bad.sum(), d.mean()))
            assert d[~bad].max() <= 1e-3 and d.mean() <= 1e-5, name
            assert not bad.any() or d[bad].max() <= 2e-2, name
            ill.append(bad)
            base.append(mine)
        dq = np.rint((ref.astype(np.float64) - np.stack(base).astype(np.float64)) / QUANT)
        assert np.abs(dq).max() < 2 ** 15, name
        out.update({"dflow%d" % i: dq.astype(np.int16), "sample%d" % i: ref[:, ::SAMPLE, ::SAMPLE],
                    "ill%d" % i: np.packbits(np.stack(ill))})
        names.append(name)
        refs.append(ref)
    out["n_cases"] = np.int32(len(names))
    out["names"] = np.array(names)
    tgt, res = sequence(full)
    out.update({"seq_tof": reference_tof(tgt, res), "cutfr": np.int32(CUTFR)})
    print("sequence tOF", out["seq_tof"])
    path = os.path.join(HERE, "tof.npz")
    np.savez_compressed(path, **out)
    load.cache_clear()
    g = load()
    for i, ref in enumerate(refs):
        assert np.abs(g["flow%d" % i] - ref).max() <= 1e-7, names[i]
    print("wrote %s (%.0f KB)" % (path, os.path.getsize(path) / 1e3))


if __name__ == "__main__":
    main()
