"""CPU: the restatement of the device PNG decoder (tests/golden/inflate_oracle.py: inflate, unfilter, expand) equals
zlib and cv2 on every case of tests/png_decode_cases.py; the cases reach every feature of the deflate format and every
filter at every pixel width; the host router (tecogan_b200.png.parse_png) sends each fallback case to cv2 and every
other case to the device."""
import zlib

import cv2
import numpy as np
import pytest

from tests import png_decode_cases as D
from tests.golden import inflate_oracle as O

ORACLE_MAX_PIXELS = 100000           # the pure-Python oracle is slow; the 576 x 720 case is left to the GPU test


@pytest.fixture(scope="module")
def decoded():
    from tecogan_b200 import png as P
    out = {}
    for name, data in D.device_cases().items():
        s = P.parse_png(data)
        assert s is not None, name
        if s.h * s.w <= ORACLE_MAX_PIXELS:
            out[name] = (data, s) + O.decode(s)
    return out


def test_oracle_inflate_equals_zlib(decoded):
    for name, (_, s, _, _, _) in decoded.items():
        assert O.inflate(s.idat)[0] == zlib.decompress(s.idat), name


def test_oracle_pixels_equal_cv2(decoded):
    for name, (data, _, im, _, _) in decoded.items():
        ref = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        assert np.array_equal(im, ref[:, :, ::-1]), name


def test_cases_reach_every_feature(decoded):
    st = {}
    for _, (_, s, _, stats, _) in decoded.items():
        for k, c in stats.items():
            st.setdefault(k, set()).update(c)
    assert {0, 1, 2} <= st["block"]
    assert 65535 in st["stored_len"] and 0 in st["stored_len"]
    assert {3, 257, 258} <= st["length"] and {284, 285} <= st["len_code"]
    assert set(range(30)) <= st["dist_code"] and 33 in st["distance"]
    assert 1 in st["distance"] and 1 in st["overlap"]
    assert 15 in st["max_code_len"]
    assert {16, 17, 18} <= st["cl_symbol"]
    assert 1 in st["dist_codes_in_block"]
    assert {2 ** w for w in range(9, 16)} <= st["window"]
    seen = set()
    for _, (_, s, _, _, filters) in decoded.items():
        bpp = max(1, D.CHANNELS[s.colour] * s.depth // 8)
        seen.update((f, bpp) for f in filters)
    assert {(f, b) for f in range(5) for b in (1, 2, 3, 4)} <= seen


def test_distance_32768_is_reached():
    from tecogan_b200 import png as P
    s = P.parse_png(D.crafted_fixed())
    raw, _ = O.inflate(s.idat)
    assert raw == zlib.decompress(s.idat)
    # the last token is a 10-byte match 32 768 back
    assert raw[-10:] == raw[-10 - 32768:-32768]


def test_router_sends_fallbacks_to_cv2():
    from tecogan_b200 import png as P
    for name, (data, status) in D.fallback_cases().items():
        s = P.parse_png(data)
        if status is None:
            assert s is None, name
            continue
        assert s is not None, name
        with pytest.raises(O.InflateError):
            O.decode(s)


def test_router_keeps_frames_cv2_refuses_on_the_host():
    """cv2.imread raises above 2^30 pixels; such files stay with cv2 (so with its error), 2^30 itself goes to the device."""
    from tecogan_b200 import png as P
    z = zlib.compress(b"\x00")
    assert P.parse_png(D.png_file(33000, 33000, 0, 1, z)) is None
    assert P.parse_png(D.png_file(32768, 32768, 0, 1, z)) is not None
    assert P.parse_png(D.png_file(1, 65501, 0, 1, z)) is None


def test_device_pays_on_the_measured_workloads():
    """The per-window choice between the device and cv2 threads on the workloads of DESIGN.md section 7: the device
    keeps many-file windows and small files, cv2 takes few large frames."""
    from tecogan_b200 import png as P

    def frames(h, w, n):
        return [(h, w)] * n
    assert P.device_pays(frames(576, 720, 205), 6)           # frame store, 256 MiB windows of 576x720
    assert P.device_pays(frames(576, 720, 82), 1)            # metrics.py, a 41-frame folder pair
    assert not P.device_pays(frames(1080, 1920, 43), 6)      # frame store of 1080p frames
    assert not P.device_pays(frames(2160, 3840, 16), 1)      # metrics.py, a short 4K folder
    assert not P.device_pays(frames(2160, 3840, 82), 1)      # 256 MiB batches hold ten 4K frames: 9 x 5 s against 24 s
    assert P.device_pays(frames(40, 52, 6), 3)               # small frames: either way within the slack
    assert not P.device_pays([], 1)
