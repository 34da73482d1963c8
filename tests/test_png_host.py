"""CPU: the PNG oracle (tests/golden/png_oracle.py) writes cv2.imencode's bytes, and its deflate body is zlib's Z_RLE
output.  A change in cv2's PNG settings or in zlib's run-length coding fails here before any GPU comparison."""
import hashlib
import zlib

import cv2
import numpy as np
import pytest

from tests import png_cases as PC
from tests.golden import png_oracle as P
from tests.test_gpu_png import CV2_SHA256

_CASES = PC.cases()


def _cv2_png(rgb):
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(rgb[:, :, ::-1]))
    assert ok
    return buf.tobytes()


def _zlib_rle(s):
    c = zlib.compressobj(1, zlib.DEFLATED, -15, 8, zlib.Z_RLE)
    return c.compress(s.tobytes()) + c.flush()


@pytest.mark.parametrize("name", PC.ORACLE_CASES)
def test_oracle_matches_cv2_and_zlib(name):
    rgb = _CASES[name]
    assert P.png_file(rgb) == _cv2_png(rgb), name
    s = P.filter_stream(rgb)
    assert P.deflate_rle(s) == _zlib_rle(s), name


@pytest.mark.parametrize("name", sorted(CV2_SHA256))
def test_recorded_cv2_bytes(name):
    """The GPU test's inputs and cv2's bytes for them are the recorded ones."""
    assert hashlib.sha256(_cv2_png(_CASES[name])).hexdigest() == CV2_SHA256[name], name


def test_window_bits_rule():
    """The zlib header's window: the smallest of 2^8 .. 2^15 bytes holding S, on sizes around every power of two."""
    g = np.random.default_rng(0)
    seen = set()
    for h, w in [(1, 1), (1, 2), (2, 13), (2, 42), (2, 43), (3, 28), (4, 21), (5, 34), (6, 56), (7, 48), (8, 42),
                 (8, 43), (16, 42), (16, 43), (11, 124), (32, 42), (32, 43), (64, 42), (64, 43), (128, 42), (128, 43), (300, 401)]:
        rgb = g.integers(0, 4, (h, w, 3), dtype=np.uint8)
        n = h * (3 * w + 1)
        head = _cv2_png(rgb)[41:43]             # first IDAT's first two data bytes
        assert head == P.zlib_header(n), (h, w, n, head.hex())
        seen.add(P.window_bits(n))
    assert seen == set(range(8, 16))


def test_constructed_streams():
    """The constructed frames reach what they are named for."""
    s = P.filter_stream(_CASES["exact_blocks"])
    assert len(P.tokenize(s)) == 2 * P.BLOCK_SYMBOLS and len(P.split_blocks(P.tokenize(s))[-1]) == 0
    toks = P.tokenize(P.filter_stream(_CASES["long_codes"]))
    freq = [0] * P.L_CODES
    freq[P.END_BLOCK] = 1
    for _, v in toks:
        freq[v] += 1
    assert max(P.build_tree(list(freq), 64)[0]) > 15 and max(P.build_tree(list(freq), 15)[0]) == 15
    toks = P.tokenize(P.filter_stream(_CASES["one_literal"]))
    assert {v for k, v in toks if k == 0} == {1}
    kinds = [P.block_plan(b)["kind"] for b in P.split_blocks(P.tokenize(P.filter_stream(_CASES["noise_then_smooth"])))]
    assert "stored" in kinds and kinds.index("dynamic") > kinds.index("stored")
    for n in (3, 4, 258, 259, 260, 261):
        s = P.filter_stream(_CASES["runs_%d" % n])
        row = len(s) // 4
        assert (s[row - n:row] == 7).all() and s[row - n - 1] != 7
        assert (s[2 * row - n + 1:2 * row + 1] == 1).all() and s[2 * row - n] != 1     # run crosses the row end
        assert (s[-n:] == 9).all() and s[-n - 1] != 9
