"""CPU: the GIF oracle (tests/golden/gif_oracle.py) writes files that two independent decoders, cv2 and PIL, read back as
the oracle's dithered frames with the right frame count, size, delay and looping; animations of at most 256 colours come
back exactly; the seeded cases (tests/gif_cases.py) reach every rule of the encoding and their bytes are the recorded
hashes; the summary quantisation is tf.image.convert_image_dtype's; and EventWriter.add_images events read back through
TensorBoard."""
import io

import numpy as np
import pytest

from tests import gif_cases as GC
from tests.golden import gif_oracle as O


@pytest.fixture(scope="module")
def encoded():
    out = {}
    for name, batch in GC.cases().items():
        out[name] = [(a,) + O.encode(a) for a in batch]
    return out


def _cv2_frames(data):
    import cv2
    ok, anim = cv2.imdecodeanimation(np.frombuffer(data, np.uint8))
    assert ok
    return np.stack([f[:, :, 2::-1] for f in anim.frames]), list(anim.durations), anim.loop_count


def _pil_frames(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    frames, durations = [], []
    for i in range(im.n_frames):
        im.seek(i)
        frames.append(np.array(im.convert("RGB")))
        durations.append(im.info.get("duration"))
    return np.stack(frames), durations, im.info.get("loop")


def test_hashes_pin_the_oracle(encoded):
    assert set(encoded) == set(GC.HASHES)
    for name, items in encoded.items():
        assert [GC.sha(data) for _, data, _ in items] == GC.HASHES[name], name


@pytest.mark.parametrize("decoder", ["cv2", "pil"])
def test_two_decoders_read_the_oracle_frames(encoded, decoder):
    read = _cv2_frames if decoder == "cv2" else _pil_frames
    for name, items in encoded.items():
        for a, data, info in items:
            frames, durations, loop = read(data)
            assert frames.shape == a.shape, (name, frames.shape)
            assert np.array_equal(frames, O.decoded_frames(info)), name
            assert list(durations) == [10 * O.DELAY_CS] * len(a), (name, durations)
            assert loop == 0, name


def test_at_most_256_colours_is_lossless(encoded):
    n = 0
    for name, items in encoded.items():
        for a, _, info in items:
            if len(np.unique(a.reshape(-1, 3), axis=0)) <= 256:
                assert np.array_equal(O.decoded_frames(info), a), name
                n += 1
    assert n >= 8


def test_cases_reach_every_rule(encoded):
    infos = [(name, a, info) for name, items in encoded.items() for a, _, info in items]
    assert any(info["boxes"] == 1 for _, _, info in infos)                       # one box: a single colour
    assert any(info["split_ties"]["box"] for _, _, info in infos)               # tie in the box choice
    assert any(info["split_ties"]["axis"] for _, _, info in infos)              # tie in the axis choice
    assert any(info["split_ties"]["no_v"] for _, _, info in infos)              # no v passes: v = max - 1
    assert any(info["nearest_ties"] for _, _, info in infos)                    # tie in the nearest colour
    assert any(info["boxes"] == 256 for _, _, info in infos)                    # palette full
    widths = set().union(*(info["widths"] for _, _, info in infos))
    assert widths == {9, 10, 11, 12}                                            # every code width
    assert any(info["clears"] for _, _, info in infos)                          # mid-stream Clear (noise)
    assert any(max(info["sub_blocks"]) > 1 for _, _, info in infos)             # more than one sub-block
    assert any(max(info["sub_blocks"]) == 1 for _, _, info in infos)
    shapes = {a.shape[1:3] for _, a, _ in infos}
    assert (1, 1) in shapes and (17, 23) in shapes and (256, 256) in shapes
    frames = {a.shape[0] for _, a, _ in infos}
    assert {1, 10, 19, 18} <= frames                                            # ping-pong: 2 RNN_N - 1 and one less


def test_file_layout(encoded):
    a, data, info = encoded["odd_lossless"][1]
    t, h, w, _ = a.shape
    assert data[:6] == b"GIF89a"
    assert data[6:13] == bytes([w & 255, w >> 8, h & 255, h >> 8, 0xF7, 0, 0])
    pal = np.frombuffer(data[13:13 + 768], np.uint8).reshape(256, 3)
    n = len(info["palette"])
    assert np.array_equal(pal[:n], info["palette"]) and not pal[n:].any()
    assert data[781:800] == b"\x21\xFF\x0BNETSCAPE2.0\x03\x01\x00\x00\x00"
    assert data[800:808] == b"\x21\xF9\x04\x00\x21\x00\x00\x00"
    assert data[808] == 0x2C and data[817] == 0 and data[818] == 8
    assert data.count(b"\x21\xF9\x04\x00\x21\x00\x00\x00\x2C") == t
    assert data[-1:] == b"\x3B"


def test_lzw_width_steps_match_decoders():
    """Index streams that end right at each width step (2^k - 258 codes after the Clear) and at the table's reset
    decode exactly: the pending code and EOI are written at the width the decoders expect."""
    rng = np.random.default_rng(7)
    for n in (253, 254, 255, 256, 767, 768, 1791, 1792, 3838, 3839, 3840, 3841, 7700):
        a = rng.integers(0, 256, n, dtype=np.uint8)
        a[: min(n, 256)] = np.arange(min(n, 256))                     # every index, so the palette has 256 entries
        frame = np.stack([a, a, a], -1).reshape(1, 1, n, 3)           # grey levels: 256 colours, stored exactly
        data, info = O.encode(frame)
        for read in (_cv2_frames, _pil_frames):
            got = read(data)[0]
            assert np.array_equal(got, frame), n


def test_convert_image_dtype_matches_tensorflow_rule():
    k = np.arange(256, dtype=np.float32)
    b = (k / np.float32(255.5)).astype(np.float32)
    x = np.concatenate([b, np.nextafter(b, np.float32(-1)), [-0.1, 1.2, np.nan, -np.inf, np.inf]]).astype(np.float32)
    got = O.convert_image_dtype(x)
    ref = [int(min(max(float(np.float32(v) * np.float32(255.5)), 0.0), 255.0)) if v == v else 0 for v in x]
    assert got.tolist() == ref
    assert got[-5:].tolist() == [0, 255, 0, 0, 255]
    d = O.convert_image_dtype(x * 2 - 1, deprocess=True)
    assert d[-5:].tolist() == [0, 255, 0, 0, 255]


def test_add_images_reads_back_through_tensorboard(tmp_path):
    ea = pytest.importorskip("tensorboard.backend.event_processing.event_accumulator")
    from tecogan_b200.summary import EventWriter
    a, b = GC.cases()["odd_lossless"][:2]
    da, db = O.encode(a)[0], O.encode(b)[0]
    w = EventWriter(str(tmp_path))
    w.add_images(2, [("image_summaries/LR/gif/0", 17, 23, da), ("image_summaries/LR/gif/1", 17, 23, db)])
    w.add_images(4, [("image_summaries/LR/gif", 17, 23, db)])
    w.close()
    acc = ea.EventAccumulator(str(tmp_path), size_guidance={ea.IMAGES: 0})
    acc.Reload()
    assert sorted(acc.Tags()["images"]) == ["image_summaries/LR/gif", "image_summaries/LR/gif/0",
                                            "image_summaries/LR/gif/1"]
    for tag, step, data in (("image_summaries/LR/gif/0", 2, da), ("image_summaries/LR/gif/1", 2, db),
                            ("image_summaries/LR/gif", 4, db)):
        (ev,) = acc.Images(tag)
        assert (ev.step, ev.height, ev.width, ev.encoded_image_string) == (step, 17, 23, data)
