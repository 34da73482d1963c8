"""CPU: the JPEG oracle (tests/golden/jpeg_oracle.py) writes cv2.imencode('.jpg')'s bytes, the recorded hashes are cv2's
bytes for the seeded frames, and the frames reach every code path the format has.  A change in cv2's JPEG defaults or
in its libjpeg-turbo fails here before any GPU comparison."""
import hashlib

import cv2
import numpy as np
import pytest

from tests import jpeg_cases as JC
from tests.golden import jpeg_oracle as J
from tests.test_gpu_jpeg import CV2_SHA256

_CASES = JC.cases()
_SMALL = sorted(n for n in _CASES if n not in JC.BIG)


def _cv2_jpg(rgb):
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(rgb[:, :, ::-1]))
    assert ok
    return buf.tobytes()


def test_case_set():
    assert sorted(_CASES) == sorted(CV2_SHA256)
    assert {(h, w) for h in JC.SIDES for w in JC.SIDES} <= {f.shape[:2] for f in _CASES.values()}


@pytest.mark.parametrize("name", _SMALL)
def test_oracle_matches_cv2(name):
    assert J.encode(_CASES[name]) == _cv2_jpg(_CASES[name]), name


@pytest.mark.parametrize("name", sorted(CV2_SHA256))
def test_recorded_cv2_bytes(name):
    """The GPU test's inputs and cv2's bytes for them are the recorded ones."""
    assert hashlib.sha256(_cv2_jpg(_CASES[name])).hexdigest() == CV2_SHA256[name], name


def test_format_facts():
    """The header: marker order, JFIF 1.01, quality-95 tables in zigzag order, 4:2:0 SOF0, Annex K tables, SOS; the
    only bytes that change with the frame size are H and W."""
    a, b = _cv2_jpg(_CASES["grid_7x9"]), _cv2_jpg(_CASES["grid_33x17"])
    hdr = J.header(7, 9)
    assert a[:len(hdr)] == hdr and b[:len(hdr)] == J.header(33, 17) and a[-2:] == b"\xff\xd9"
    markers, i = [], 2
    while a[i:i + 2] != b"\xff\xda":
        markers.append(a[i + 1])
        i += 2 + int.from_bytes(a[i + 2:i + 4], "big")
    assert markers == [0xE0, 0xDB, 0xDB, 0xC0, 0xC4, 0xC4, 0xC4, 0xC4]
    assert a[2:20] == b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    sof = 2 + 18 + 2 * 69                                                   # SOF0: FF C0, length, precision, H, W
    assert a[sof:sof + 2] == b"\xff\xc0" and a[sof + 5:sof + 9] == bytes([0, 7, 0, 9])
    assert {i for i in range(len(hdr)) if a[i] != b[i]} <= set(range(sof + 5, sof + 9))
    assert J.quant_table([16, 11, 99, 1, 255]).tolist() == [2, 1, 10, 1, 26]
    assert b"\xff\xfe" not in a[:len(hdr)] and b"\xff\xdd" not in a[:len(hdr)]   # no comment, no restart interval


def test_bottom_rule_is_not_row_padding():
    """At even H not a multiple of 16, the last downsampled chroma row is repeated; repeating image rows before
    downsampling would give other bytes."""
    rgb = _CASES["grid_24x17"]
    st = {}
    assert J.encode(rgb, st) == _cv2_jpg(rgb) and st["bottom_rule"] == 1


def test_coverage():
    """The seeded frames reach: right and bottom dummy blocks; the bottom-row rule; odd W and odd H; both chroma biases;
    ZRL; a block with no EOB; DC-only blocks; 0xFF stuffing; every padding length 0-7; the largest size categories
    quality 95 can produce (10 for DC differences: a quantised DC is -512 .. 508; 10 for AC, baseline's largest)."""
    st = {}
    for name in _SMALL:
        J.encode(_CASES[name], st)
    assert st["dummy_right"] > 0 and st["dummy_bottom"] > 0 and st["bottom_rule"] > 0
    assert st["odd"] == {"W", "H"} and st["biases"] == {1, 2}
    assert st["zrl"] > 0 and st["no_eob"] > 0 and st["dc_only"] > 0 and st["ff"] > 0
    assert st["pad"] == set(range(8))
    assert st["max_dc_cat"] == 10 and st["max_ac_cat"] == 10
    runs = {}
    J.encode(_CASES["runs"], runs)
    assert runs["zrl"] == 9 and runs["no_eob"] == 3          # runs of 16, 32, 47, 62 and 31 zeros; three blocks end on 63
