"""Seeded RGB uint8 frames for the PNG encoder tests (tests/test_png_host.py, tests/test_gpu_png.py): content classes,
degenerate shapes, and frames built by choosing the filtered stream S and inverting the Sub filter.  numpy only."""
import heapq

import numpy as np

from tests.golden import png_oracle as P


def smooth(h, w, seed):
    """Smooth noise: a coarse random grid, linearly interpolated."""
    g = np.random.default_rng(seed)
    gh, gw = h // 16 + 2, w // 16 + 2
    coarse = g.random((gh, gw, 3))
    ys, xs = np.linspace(0, gh - 1, h), np.linspace(0, gw - 1, w)
    rows = np.stack([np.stack([np.interp(xs, np.arange(gw), coarse[i, :, c]) for c in range(3)], -1) for i in range(gh)])
    out = np.stack([np.stack([np.interp(ys, np.arange(gh), rows[:, j, c]) for c in range(3)], -1) for j in range(w)], 1)
    return (out * 255).round().astype(np.uint8)


def noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def low_entropy(h, w, seed):
    return (np.random.default_rng(seed).integers(0, 3, (h, w, 3)) * 40).astype(np.uint8)


def _from_rows(body, w):
    """Rows of 3w filtered bytes -> the frame whose S is filter byte 1 + each row."""
    body = np.asarray(body, np.uint8).reshape(-1, 3 * w)
    s = np.concatenate([np.ones((len(body), 1), np.uint8), body], 1).reshape(-1)
    return P.unfilter_sub(s, len(body), w)


def _no_repeats(counts, seed):
    """A sequence holding symbol k counts[k] times with no two neighbours equal (most frequent first, greedy)."""
    g = np.random.default_rng(seed)
    heap = [(-c, int(g.integers(1 << 30)), s) for s, c in counts.items() if c]
    heapq.heapify(heap)
    out, held = [], None
    while heap:
        c, t, s = heapq.heappop(heap)
        out.append(s)
        if held:
            heapq.heappush(heap, held)
        held = (c + 1, t, s) if c + 1 < 0 else None
    assert held is None
    return out


def exact_blocks():
    """S of 2 x 16 383 literals, no two neighbours equal: two full blocks and an empty final one."""
    h, w = 258, 42                                  # 258 * (3 * 42 + 1) = 2 * 16 383
    g = np.random.default_rng(5)
    body = np.empty(h * 3 * w, np.int64)
    prev = -1
    for i in range(len(body)):
        v = int(g.integers(2, 10))
        while v == prev:
            v = int(g.integers(2, 10))
        body[i] = prev = v
        if (i + 1) % (3 * w) == 0:
            prev = -1                               # the filter byte 1 separates rows
    return _from_rows(body, w)


def long_codes():
    """One row whose filtered bytes have the Fibonacci counts 2, 3, 5, .., 987 and 1 598 (one more than 1 597, to fill
    whole pixels); with the filter byte and the end-of-block code (one each) the Huffman code is a 16-level chain, over
    the 15-bit limit."""
    fib = [1, 2]
    while fib[-1] < 1597:
        fib.append(fib[-1] + fib[-2])
    counts = {2 + k: f for k, f in enumerate(fib[1:])}
    counts[max(counts)] += 1
    w = sum(counts.values()) // 3                   # 4 179 bytes = 1 393 pixels
    return _from_rows(_no_repeats(counts, 7), w)


def one_literal():
    """S all ones (filter byte 1, every Sub difference 1): one literal value, then matches."""
    return _from_rows(np.ones(40 * 3 * 30, np.uint8), 30)


def runs_at_ends(n):
    """Runs of n bytes ending a row, runs of 1s that continue into the next row's filter byte, and a run ending S."""
    w = 100
    g = np.random.default_rng(n)
    rows = []
    for k, v in enumerate((7, 1, 1, 9)):
        head = 3 * w - (n if v != 1 else n - 1)
        r = np.empty(3 * w, np.int64)
        prev = -1
        for i in range(head):
            x = int(g.integers(2, 250))
            while x == prev or x == v:
                x = int(g.integers(2, 250))
            r[i] = prev = x
        r[head:] = v
        rows.append(r)
    return _from_rows(np.concatenate(rows), w)


def noise_then_smooth():
    """Uniform noise (stored blocks) above smooth content (dynamic blocks)."""
    return np.concatenate([noise(96, 256, 11), smooth(160, 256, 12)], 0)


def cases():
    """name -> frame, every frame the GPU test compares with cv2."""
    c = {
        "smooth_32x32": smooth(32, 32, 1), "smooth_128x128": smooth(128, 128, 2), "smooth_512x512": smooth(512, 512, 3),
        "smooth_1080x1920": smooth(1080, 1920, 4), "smooth_2160x3840": smooth(2160, 3840, 5),
        "noise_1x1": noise(1, 1, 6), "noise_h1": noise(1, 257, 7), "noise_w1": noise(300, 1, 8),
        "low_w1": low_entropy(77, 1, 9), "low_odd": low_entropy(61, 333, 10), "smooth_odd": smooth(99, 201, 13),
        "noise_576x720": noise(576, 720, 14), "noise_then_smooth": noise_then_smooth(),
        "constant": np.full((64, 300, 3), 7, np.uint8), "constant_1x1": np.zeros((1, 1, 3), np.uint8),
        "exact_blocks": exact_blocks(), "long_codes": long_codes(), "one_literal": one_literal(),
    }
    for n in (3, 4, 258, 259, 260, 261):
        c["runs_%d" % n] = runs_at_ends(n)
    return c


# frames small enough for the host oracle (pure Python) in tests/test_png_host.py
ORACLE_CASES = ("smooth_32x32", "smooth_128x128", "noise_1x1", "noise_h1", "noise_w1", "low_w1", "low_odd", "smooth_odd",
                "noise_then_smooth", "constant", "constant_1x1", "exact_blocks", "long_codes", "one_literal", "runs_3",
                "runs_4", "runs_258", "runs_259", "runs_260", "runs_261")
