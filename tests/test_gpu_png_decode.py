"""GPU: tecogan_b200.png.decode_png / decode_png_into give the pixels cv2.imread gives, byte for byte -- every file of
tests/png_decode_cases.py one per call and all in one mixed batch, the fallback classes with their device status,
frames up to 2160 x 3840 -- never write outside their destinations, and the two callers (FrameStore, metrics.py) are
unchanged by them.  Every test that goes through those calls also asserts which files came from the device and which
from cv2, so a device refusal cannot hide behind the cv2 fallback."""
import hashlib
import os

import cv2
import numpy as np
import pytest
import torch

from tests import png_cases as PC
from tests import png_decode_cases as D

pytestmark = pytest.mark.gpu


def _write(root, cases):
    paths = {}
    for name, data in cases.items():
        p = os.path.join(root, name + ".png")
        with open(p, "wb") as f:
            f.write(data)
        paths[name] = p
    return paths


def _cv2(path):
    im = cv2.imread(path, cv2.IMREAD_COLOR)
    return None if im is None else np.ascontiguousarray(im[:, :, ::-1])


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("png_decode"))
    dev = _write(root, D.device_cases())
    fb = D.fallback_cases()
    return dev, _write(root, {k: v[0] for k, v in fb.items()}), {k: v[1] for k, v in fb.items()}


def test_every_device_case_alone_equals_cv2(files):
    from tecogan_b200 import png as P
    dev, _, _ = files
    for name, path in dev.items():
        assert P.load_png(path) is not None, name
        s = P.load_png(path)
        buf = torch.empty(s.h * s.w * 3, dtype=torch.uint8, device="cuda")
        status = P.decode_streams([(s, 0)], buf)
        assert status.tolist() == [0], (name, P.STATUS[int(status[0])])
        assert np.array_equal(buf.view(s.h, s.w, 3).cpu().numpy(), _cv2(path)), name
        (got,) = P.decode_png([path])
        assert got.is_cuda and got.dtype == torch.uint8 and np.array_equal(got.cpu().numpy(), _cv2(path)), name


def _recording(seen):
    """imread_rgb that records the paths it decodes: the files that did not come from the device."""
    from tecogan_b200 import png as P

    def host(path):
        seen.append(path)
        return P.imread_rgb(path)
    return host


def test_one_launch_over_every_case_at_offsets(files):
    """Every device case and every stream-level fallback in one launch, streams, workspaces and destinations at
    non-zero offsets with gaps: each file gets its own status, the decoded ones equal cv2, the gaps keep the sentinel."""
    from tecogan_b200 import png as P
    dev, fb, want = files
    names = [n for n in sorted(dev)] + [n for n in sorted(fb) if want[n] is not None]
    streams = [P.load_png(dev.get(n) or fb[n]) for n in names]
    offsets, at = [], 7
    for s in streams:
        offsets.append(at)
        at += s.h * s.w * 3 + 13
    buf = torch.full((at,), 0x5A, dtype=torch.uint8, device="cuda")
    status = P.decode_streams(list(zip(streams, offsets)), buf)
    assert status.tolist() == [0 if n in dev else want[n] for n in names]
    host = buf.cpu().numpy()
    mask = np.ones(host.size, bool)
    for n, s, o in zip(names, streams, offsets):
        mask[o:o + s.h * s.w * 3] = False
        if n in dev:
            assert np.array_equal(host[o:o + s.h * s.w * 3].reshape(s.h, s.w, 3), _cv2(dev[n])), n
    assert (host[mask] == 0x5A).all()


def test_mixed_batch_with_fallbacks_equals_cv2(files):
    from tecogan_b200 import png as P
    dev, fb, _ = files
    names = sorted(dev) + sorted(fb)
    paths = [dev.get(n) or fb[n] for n in names]
    # small files only: one 576x720 frame among them would make one window cheaper on cv2 threads (device_pays)
    decodable = [(n, p) for n, p in zip(names, paths) if _cv2(p) is not None and _cv2(p).size <= 300000]
    fallback = {p for n, p in decodable if n in fb}
    for kw in (dict(threads=4), dict(batch_bytes=4096)):                   # one window; many windows and batches
        seen = []
        got = P.decode_png([p for _, p in decodable], host_decode=_recording(seen), **kw)
        for (n, p), g in zip(decodable, got):
            assert np.array_equal(g.cpu().numpy(), _cv2(p)), n
        sizes = [P.png_size(p) for _, p in decodable]
        on_host = set(fallback)                          # plus whole windows where cv2 threads are expected to win
        disk = [os.path.getsize(p) for _, p in decodable]
        for i, j in P._windows(disk, kw.get("batch_bytes", P.BATCH_BYTES)):
            if not P.device_pays([x for x in sizes[i:j] if x], kw.get("threads", 1), kw.get("batch_bytes", P.BATCH_BYTES)):
                on_host.update(p for _, p in decodable[i:j])
        assert sorted(seen) == sorted(on_host), kw
        if "threads" in kw:
            assert on_host == fallback                   # one window of many files: all on the device
    for n, p in zip(names, paths):
        if _cv2(p) is None:
            with pytest.raises(ValueError, match="cannot decode"):
                P.decode_png([p])


def test_fallback_classes_get_their_device_status(files):
    from tecogan_b200 import png as P
    _, fb, want = files
    for name, path in fb.items():
        s = P.load_png(path)
        if want[name] is None:
            assert s is None, name
            continue
        assert s is not None, name
        buf = torch.zeros(s.h * s.w * 3, dtype=torch.uint8, device="cuda")
        assert P.decode_streams([(s, 0)], buf).tolist() == [want[name]], name


def test_decode_into_leaves_every_other_byte_alone(files):
    from tecogan_b200 import png as P
    dev, fb, _ = files
    names = sorted(dev)[::3] + ["palette_index", "trailing", "exif6", "depth16"]
    paths = [dev.get(n) or fb[n] for n in names]
    ims = [_cv2(p) for p in paths]
    sizes = np.array([im.shape[:2] for im in ims], np.int64)
    gaps = np.random.default_rng(1).integers(1, 40, len(ims))
    offsets, at = [], 5
    for im, g in zip(ims, gaps):
        offsets.append(at)
        at += im.size + int(g)
    buf = torch.full((at + 17,), 0xA5, dtype=torch.uint8, device="cuda")
    seen = []
    P.decode_png_into(paths, buf, offsets, sizes, threads=3, batch_bytes=50000, host_decode=_recording(seen))
    on_host = {fb[n] for n in names[-4:]}
    for i, j in P._windows((sizes[:, 0] * sizes[:, 1] * 3).tolist(), 50000):
        if not P.device_pays(sizes[i:j], 3, 50000):
            on_host.update(paths[i:j])
    assert sorted(seen) == sorted(on_host)                                 # every other file came from the device
    assert len(on_host) < len(paths) // 2
    host = buf.cpu().numpy()
    mask = np.ones(host.size, bool)
    for im, o in zip(ims, offsets):
        assert np.array_equal(host[o:o + im.size], im.reshape(-1))
        mask[o:o + im.size] = False
    assert (host[mask] == 0xA5).all()
    with pytest.raises(ValueError, match="slot holds"):
        P.decode_png_into(paths[:1], buf, [0], [(sizes[0, 0] + 1, sizes[0, 1])])


@pytest.mark.parametrize("h,w", [(576, 720), (1080, 1920), (2160, 3840)])
def test_large_frames(tmp_path, h, w):
    from tecogan_b200 import png as P
    paths = []
    for k, frame in enumerate((PC.smooth(h, w, 7), PC.noise(h, w, 8))):
        p = str(tmp_path / ("f%d.png" % k))
        cv2.imwrite(p, np.ascontiguousarray(frame[:, :, ::-1]))
        paths.append(p)
    streams = [P.load_png(p) for p in paths]
    buf = torch.empty(2 * h * w * 3 + 5, dtype=torch.uint8, device="cuda")
    assert P.decode_streams([(streams[0], 5), (streams[1], h * w * 3 + 5)], buf).tolist() == [0, 0]
    for k, p in enumerate(paths):
        o = 5 + k * h * w * 3
        assert np.array_equal(buf[o:o + h * w * 3].view(h, w, 3).cpu().numpy(), _cv2(p)), (p, h, w)
    for threads in (1, 6):
        seen = []
        for p, g in zip(paths, P.decode_png(paths, threads=threads, host_decode=_recording(seen))):
            assert np.array_equal(g.cpu().numpy(), _cv2(p)), (p, h, w)
        assert seen == ([] if P.device_pays([(h, w)] * 2, threads) else paths), threads


def test_frame_store_matches_the_host_decoder(tmp_path):
    from tests.test_dataloader_host import Flags
    from tests.test_frame_store_host import _scenes
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader
    root = str(tmp_path / "frames")
    _scenes(root, [(40, 52), (36, 36), (47, 61)], frames=6, seed=11)
    deep = os.path.join(root, "scene_2003")                                  # one scene of 16-bit frames: host path
    os.makedirs(deep)
    g = np.random.default_rng(12)
    for f in range(6):
        cv2.imwrite(os.path.join(deep, "col_high_%04d.png" % f), g.integers(0, 65536, (38, 44, 3)).astype(np.uint16))
    F = Flags(input_video_dir=root, str_dir=2000, end_dir=2003, max_frm=5, RNN_N=3, batch_size=2, crop_size=4)
    L = HRClipLoader(F)
    seen = []
    L.decode = lambda path: (seen.append(path), HRClipLoader.decode(path))[1]
    store = FrameStore([L], "cuda", chunk_bytes=30000)
    assert sorted(seen) == sorted(p for p in store.paths if p.startswith(deep))   # only the 16-bit scene on the host
    ref = b"".join(np.ascontiguousarray(HRClipLoader.decode(p)).tobytes() for p in store.paths)
    assert store.checksum() == hashlib.sha256(ref).hexdigest()


def _folders(tmp_path, n=9):
    res, tar = tmp_path / "res", tmp_path / "tar"
    res.mkdir()
    tar.mkdir()
    for k in range(n):
        t = PC.smooth(72, 88, 100 + k)
        o = np.clip(t.astype(np.int64) + np.random.default_rng(k).integers(-9, 10, t.shape), 0, 255).astype(np.uint8)
        cv2.imwrite(str(tar / ("%04d.png" % k)), t[:, :, ::-1])
        cv2.imwrite(str(res / ("output_%04d.png" % k)), o[:, :, ::-1])
    return str(res), str(tar)


@pytest.mark.parametrize("tof", [False, True])
def test_metrics_command_writes_what_the_host_decoder_gives(tmp_path, monkeypatch, tof):
    import metrics as CLI
    res, tar = _folders(tmp_path)
    args = ["--results", res, "--targets", tar] + (["--tof"] if tof else [])
    read_rgb, seen = CLI.read_rgb, []
    monkeypatch.setattr(CLI, "read_rgb", lambda p: (seen.append(p), read_rgb(p))[1])
    CLI.main(["--output", str(tmp_path / "dev")] + args)
    assert seen == []                                                      # every frame came from the device
    monkeypatch.setattr(CLI, "read_folder", lambda paths: [torch.from_numpy(read_rgb(p)).cuda() for p in paths])
    CLI.main(["--output", str(tmp_path / "host")] + args)
    for f in ("metricsfile.txt", "metrics.csv"):
        assert open(tmp_path / "dev" / f).read() == open(tmp_path / "host" / f).read(), f
