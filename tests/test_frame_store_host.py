"""CPU: the draw / assemble split of HRClipLoader.sample() (tecogan_b200/lib/dataloader.py) leaves every sample as the
single-pass loader cut it, the frame store's sizing and rank shares, and main.frame_store_fits, the rule that picks the
device frame store or the host loader for main.py --mode train --input_video_dir."""
import os

import numpy as np
import pytest

from tests.test_dataloader_host import Flags


def _scenes(root, sizes, frames=12, seed=0):
    """Scenes 2000, 2001, ... of seeded random uint8 frames; scene i has size sizes[i] = (h, w)."""
    import cv2
    rng = np.random.default_rng(seed)
    for i, (h, w) in enumerate(sizes):
        p = os.path.join(root, "scene_%04d" % (2000 + i))
        os.makedirs(p)
        for f in range(frames):
            cv2.imwrite(os.path.join(p, "col_high_%04d.png" % f), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))


def _single_pass_sample(L, index, epoch=0):
    """HRClipLoader.sample() as one pass, the way it was written before draw() and assemble() split it: whole frames
    decoded and converted to float32 / 255, then the windows cut."""
    import cv2 as cv
    F, T, tar = L.F, L.F.RNN_N, L.tar_size

    def read(path):
        return np.ascontiguousarray(cv.imread(path, cv.IMREAD_COLOR)[:, :, ::-1]).astype(np.float32) / 255.0
    clip, start = L.clips[index // L.windows], index % L.windows
    rng = np.random.default_rng([int(F.rand_seed) & 0x7FFFFFFF, int(epoch), int(index)] + L.salt)
    moving = False
    if F.movingFirstFrame:
        step = np.floor(rng.uniform(-3.5, 4.5, size=(T, 2))).astype(np.int64)
        pos = np.cumsum(step, axis=0) - step
        span = pos.max(axis=0) - pos.min(axis=0)
        lefttop = pos - pos.min(axis=0)
        moving = not (rng.uniform() < 0.7)
    if moving:
        first = read(os.path.join(clip, 'col_high_%04d.png' % start))
        h, w = first.shape[0] - int(span[1]), first.shape[1] - int(span[0])
        frames = [first[int(lefttop[t][1]):int(lefttop[t][1]) + h, int(lefttop[t][0]):int(lefttop[t][0]) + w] for t in range(T)]
    else:
        frames = [read(os.path.join(clip, 'col_high_%04d.png' % (start + t))) for t in range(T)]
    h, w = frames[0].shape[:2]
    off_w = int(np.floor(rng.uniform(0, float(w) - tar)))
    off_h = int(np.floor(rng.uniform(0, float(h) - tar)))
    out = np.stack([f[off_h:off_h + tar, off_w:off_w + tar] for f in frames])
    if getattr(F, 'flip', True) and rng.uniform() < 0.5:
        out = out[:, :, ::-1]
    return np.ascontiguousarray(out, dtype=np.float32)


@pytest.mark.parametrize("moving,flip,salt", [(True, True, 0), (False, True, 0), (True, False, 0), (True, True, 0x7A1D)])
def test_split_sample_equals_the_single_pass_loader(tmp_path, moving, flip, salt):
    from tecogan_b200.lib.dataloader import HRClipLoader
    root = str(tmp_path / "data")
    _scenes(root, [(40, 52), (36, 36), (47, 61)])      # 36 x 36: the 24-pixel crop after the largest 12-pixel shrink
    L = HRClipLoader(Flags(input_video_dir=root, str_dir=2000, end_dir=2002, movingFirstFrame=moving, flip=flip), salt=salt)
    seen_moving = seen_flip = 0
    for epoch in range(3):
        for idx in range(len(L)):
            d = L.draw(idx, epoch)
            s = L.sample(idx, epoch)
            assert s.dtype == np.float32 and s.flags.c_contiguous
            assert np.array_equal(s.view(np.uint32), _single_pass_sample(L, idx, epoch).view(np.uint32)), (epoch, idx)
            seen_moving += len(set(d.frames)) == 1
            seen_flip += d.flip
            assert d.origin.shape == (4, 2) and d.origin.dtype == np.int64 and (d.origin >= 0).all()
    n = 3 * len(L)
    assert (0 < seen_moving < n) == moving and (0 < seen_flip < n) == flip


def test_frame_sizes_come_from_the_png_header(tmp_path):
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader
    root = str(tmp_path / "data")
    _scenes(root, [(40, 52), (36, 36)], frames=12)
    L = HRClipLoader(Flags(input_video_dir=root, str_dir=2000, end_dir=2001))
    assert L.frame_size(L.frame_path(0, 3)) == (40, 52) and L.frame_size(L.frame_path(1, 0)) == (36, 36)
    assert FrameStore.estimate_bytes([L]) == 12 * 3 * (40 * 52 + 36 * 36)      # frames 0..max_frm = 11 of each scene
    assert FrameStore.estimate_bytes([L, L]) == FrameStore.estimate_bytes([L])  # a scene is stored once


@pytest.mark.parametrize("n,world", [(0, 1), (5, 1), (7, 2), (8, 3), (2, 4)])
def test_frame_shares_cover_every_frame_once(n, world):
    from tecogan_b200.lib.dataloader import frame_shares
    shares = frame_shares(n, world)
    assert len(shares) == world and shares[0][0] == 0 and shares[-1][1] == n
    assert all(a <= b and (r == 0 or a == shares[r - 1][1]) for r, (a, b) in enumerate(shares))
    sizes = [b - a for a, b in shares]
    assert max(sizes) - min(sizes) <= 1


def test_selection_picks_the_store_when_it_fits():
    import main as M
    G = 1 << 30
    total = 80 * G                                   # margin max(1 GiB, 5 %) = 4 GiB
    fits, msg = M.frame_store_fits(10 * G, free_bytes=60 * G, reserved_bytes=8 * G, peak_bytes=6 * G, total_bytes=total)
    assert fits and "fits in" in msg                # 60 + 8 - 6 - 4 = 58 GiB of room
    fits, msg = M.frame_store_fits(59 * G, free_bytes=60 * G, reserved_bytes=8 * G, peak_bytes=6 * G, total_bytes=total)
    assert not fits and "does not fit" in msg
    assert M.frame_store_fits(58 * G, 60 * G, 8 * G, 6 * G, total)[0]                  # exactly the room
    assert not M.frame_store_fits(58 * G + 1, 60 * G, 8 * G, 6 * G, total)[0]
    # a small device: the margin is 1 GiB
    assert M.frame_store_fits(2 * G, 4 * G, 0, 1 * G, 8 * G)[0] and not M.frame_store_fits(2 * G + 1, 4 * G, 0, 1 * G, 8 * G)[0]
