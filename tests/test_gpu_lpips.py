"""GPU: LPIPS-AlexNet v0.1 and tLP100 (tecogan_b200/lpips.py -> teco_lpips_input_u8, teco_conv2d_f32, teco_maxpool3s2_f32,
teco_lpips_head_f32) against the reference's own outputs (tests/golden/lpips.npz) and the float64 oracle.

Tolerances: the network input is bit-exact; features agree with the oracle to 1e-5 x the layer's max |value| (fp32
accumulation over at most 11*11*3, 5*5*64 or 3*3*384 = 3456 products); LPIPS to 1e-6 |ref| + 1e-9 and tLP100 to
1e-4 |ref| + 1e-7, as the reference's fp32 run agrees with float64."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu


def _g():
    return np.load(os.path.join(GOLDEN, "lpips.npz"), allow_pickle=False)


def _lin(g):
    return {"lin%d.model.1.weight" % l: torch.from_numpy(g["lin%d" % l]).reshape(1, -1, 1, 1) for l in range(5)}


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _crop(img, win):
    y, x, h, w = (int(v) for v in win)
    return np.ascontiguousarray(img[y:y + h, x:x + w])


def _model(g):
    from tests.golden import lpips_oracle as LO
    from tecogan_b200.lpips import LPIPS
    return LPIPS(LO.lpips_test_weights(int(g["alex_seed"])), _lin(g))


def _close(a, r, rel=1e-6, ab=1e-9):
    return abs(a - r) <= rel * abs(r) + ab


def test_input_scaling_is_bit_exact():
    from tests.golden import lpips_oracle as LO
    from tecogan_b200._ffi import call, ptr, stream_ptr
    imgs = np.random.default_rng(5).integers(0, 256, (2, 41, 53, 3), dtype=np.uint8)
    imgs[0, 3, 4:10] = [[0, 127, 255], [128, 1, 254], [64, 191, 2], [255, 255, 255], [0, 0, 0], [126, 129, 127]]
    y0, x0, h, w = 3, 4, 35, 44
    x = torch.empty((2, h, w, 3), device="cuda", dtype=torch.float32)
    call("teco_lpips_input_u8", ptr(_cu(imgs)), 2, 41, 53, y0, x0, h, w, ptr(x), stream_ptr())
    got = x.cpu().numpy()
    for n in range(2):
        crop = imgs[n, y0:y0 + h, x0:x0 + w]
        want = (np.float32(crop / 127.5 - 1.0) - LO.LPIPS_SHIFT) / LO.LPIPS_SCALE          # numpy: float64 then fp32
        assert want.dtype == np.float32
        assert np.array_equal(got[n].view(np.uint32), want.view(np.uint32)), n


def test_features_match_oracle_at_every_golden_size_and_in_a_batch():
    from tests.golden import lpips_oracle as LO
    g = _g()
    model, alex = _model(g), LO.lpips_test_weights(int(g["alex_seed"]))

    def check(feats, frames):
        for n, img in enumerate(frames):
            for l, ref in enumerate(LO.alexnet_features(img, alex)):
                got = feats[l][n].cpu().double().numpy()
                assert got.shape == ref.shape[1:], (l, got.shape, ref.shape)
                assert np.abs(got - ref[0]).max() <= 1e-5 * np.abs(ref).max(), (n, l)
    for i in range(int(g["n_cases"])):
        win = g["crop%d" % i]
        frames = [_crop(g["tgt%d" % i], win), _crop(g["out%d" % i], win)]
        check(model.features([_cu(g["tgt%d" % i]), _cu(g["out%d" % i])], tuple(int(v) for v in win)), frames)
    T = g["seq_tgt"][:5]                                                       # N = 5 frames in one pass
    win = (3, 5, 48, 64)
    check(model.features(_cu(T), win), [_crop(t, win) for t in T])


def test_lpips_matches_reference_and_oracle():
    from tests.golden import lpips_oracle as LO
    g = _g()
    model, alex, lin = _model(g), LO.lpips_test_weights(int(g["alex_seed"])), _lin(g)
    for i in range(int(g["n_cases"])):
        win = g["crop%d" % i]
        t, o = _crop(g["tgt%d" % i], win), _crop(g["out%d" % i], win)
        got = model(_cu(t), _cu(o))
        assert _close(got, float(g["lpips%d" % i])), (i, got, float(g["lpips%d" % i]))
        want, want_l = LO.lpips(t, o, alex, lin)
        assert _close(got, want), (i, got, want)
        f = model.features([_cu(t), _cu(o)])
        total, layers = model.distances(f, f, [(0, 1)], per_layer=True)
        assert abs(total[0] - got) <= 1e-13 * got
        for l in range(5):
            assert _close(layers[0][l], want_l[l], 1e-5), (i, l, layers[0][l], want_l[l])


def test_identical_frames_batched_pairs_and_result_cut():
    g = _g()
    model = _model(g)
    t = _cu(_crop(g["tgt1"], g["crop1"]))
    o = _cu(_crop(g["out1"], g["crop1"]))
    assert model(t, t) == 0.0
    assert model(o, o.clone()) == 0.0
    # batched pairs (both orders, repeats, self pairs) against one pair per call
    frames = [t, o, _cu(_crop(g["tgt1"], (16, 20, 128, 160)))]
    f = model.features(frames)
    pairs = [(0, 1), (1, 0), (2, 0), (1, 2), (0, 1), (2, 2)]
    d = model.distances(f, f, pairs)
    for (i, j), v in zip(pairs, d):                  # equal up to the order of the float64 pixel sum (grid depends on P)
        one = model(frames[i], frames[j])
        assert abs(v - one) <= 1e-13 * abs(one), (i, j, v, one)
    assert d[5] == 0.0 and abs(d[0] - d[1]) <= 1e-13 * d[0]
    # a result larger than the target is cut to the target's size, as frame_metrics / metrics.py:134-135 do
    big = _cu(g["out1"])                                                      # 144 x 180
    small = _cu(np.ascontiguousarray(g["tgt1"][:130, :170]))
    cut = model(small, _cu(np.ascontiguousarray(g["out1"][:130, :170])))
    assert abs(model(small, big) - cut) <= 1e-13 * cut


def test_sequence_matches_reference_loop():
    from tecogan_b200 import metrics as M
    g = _g()
    model = _model(g)
    T, R, cut = _cu(g["seq_tgt"]), _cu(g["seq_out"]), int(g["cutfr"])       # results are 2 rows taller than targets
    r = M.evaluate_sequence(T, R, cutfr=cut, lpips=model)
    assert len(r["LPIPS"]) == 3 and len(r["tLP100"]) == 2
    for a, ref in zip(r["LPIPS"], g["seq_lpips"]):
        assert _close(a, ref), (a, ref)
    for a, ref in zip(r["tLP100"], g["seq_tlp100"]):
        assert _close(a, ref, 1e-4, 1e-7), (a, ref)
    assert _close(r["FolderAvg_LPIPS"], float(np.mean(g["seq_lpips"])))
    assert _close(r["FolderAvg_tLP100"], float(np.mean(g["seq_tlp100"])), 1e-4, 1e-7)
    plain = M.evaluate_sequence(T, R, cutfr=cut)
    assert set(plain) == {"PSNR", "SSIM", "FolderAvg_PSNR", "FolderAvg_SSIM"}
    assert plain["PSNR"] == r["PSNR"] and plain["SSIM"] == r["SSIM"]
    # frames split over passes: the first frame of each pass takes its tLP from the previous pass's features
    win = M.crop_window(T.shape[1], T.shape[2])
    lp1, tlp1 = model.sequence(T[:6].contiguous(), R[:6, :T.shape[1]].contiguous(), win, chunk=8)
    lp2, tlp2 = model.sequence(T[:6].contiguous(), R[:6, :T.shape[1]].contiguous(), win, chunk=2)
    assert len(tlp2) == 5
    np.testing.assert_allclose(lp2, lp1, rtol=1e-12)
    np.testing.assert_allclose(tlp2, tlp1, rtol=1e-9, atol=1e-12)


def test_misuse_raises_value_error():
    g = _g()
    model = _model(g)
    a = _cu(_crop(g["tgt0"], g["crop0"]))
    with pytest.raises(ValueError):
        model(a[:30], a[:30])                                                  # below the 31-pixel minimum
    with pytest.raises(ValueError):
        model(a[:, :30].contiguous(), a[:, :30].contiguous())
    with pytest.raises(ValueError):
        model(a.cpu(), a.cpu())                                                # no CPU path
    with pytest.raises(ValueError):
        model(a.float(), a.float())
    with pytest.raises(ValueError):
        model.features(a, (0, 0, 64, 97))                                      # window outside the frame
    f = model.features([a, a])
    with pytest.raises(ValueError):
        model.distances(f, f, [(0, 2)])
    with pytest.raises(ValueError):
        model.distances(f, f, [(-1, 0)])
    g2 = model.features(_cu(_crop(g["tgt1"], g["crop1"])))
    with pytest.raises(ValueError):
        model.distances(f, g2, [(0, 0)])                                       # different crop sizes
    from tecogan_b200._ffi import call, ptr, stream_ptr
    import ctypes as C
    out = torch.zeros(1, device="cuda", dtype=torch.float64)
    ia, ib = (C.c_int32 * 1)(0), (C.c_int32 * 1)(2)
    with pytest.raises(ValueError):                                            # the C entry point checks the indices too
        call("teco_lpips_head_f32", ptr(f[0]), 2, ptr(f[0]), 2, C.cast(ia, C.c_void_p), C.cast(ib, C.c_void_p), 1,
             f[0].shape[1], f[0].shape[2], 64, ptr(model.lin[0]), ptr(out), stream_ptr())
    with pytest.raises(ValueError):
        call("teco_maxpool3s2_f32", ptr(f[0]), ptr(f[0]), 1, 2, 5, 64, stream_ptr())


def test_metrics_command_line_with_lpips_on_png_folders(tmp_path):
    """Root metrics.py with both LPIPS flags: LPIPS / tLPx100 in the per-frame lines, LPIPS_00 / tLP100_00 columns in
    metrics.csv, averages equal to the oracle's."""
    from PIL import Image
    from oracle import teco_oracle as O
    from tests.golden import lpips_oracle as LO
    import metrics as CLI
    g = _g()
    alex = LO.lpips_test_weights(int(g["alex_seed"]))
    torch.save({**alex, "classifier.6.bias": torch.zeros(1000)}, tmp_path / "alexnet-owt-test.pth")
    torch.save(_lin(g), tmp_path / "alex.pth")
    res, tar = tmp_path / "results" / "scene", tmp_path / "HR" / "scene"
    res.mkdir(parents=True)
    tar.mkdir(parents=True)
    T = [np.roll(g["tgt0"], 3 * k, axis=0) for k in range(6)]
    R = [np.roll(g["out0"], 3 * k, axis=0) for k in range(6)]
    for k in range(6):
        Image.fromarray(T[k]).save(tar / ("%04d.png" % k))
        Image.fromarray(R[k]).save(res / ("output_%04d.png" % k))
    log = tmp_path / "log"
    r = CLI.main(["--output", str(log), "--results", str(res), "--targets", str(tar),
                  "--lpips_alexnet", str(tmp_path / "alexnet-owt-test.pth"), "--lpips_lin", str(tmp_path / "alex.pth")])
    lin = _lin(g)
    crop = lambda a: np.ascontiguousarray(O.crop_8x8(a))                      # noqa: E731
    want_lp = np.float32([LO.lpips(crop(T[k]), crop(R[k]), alex, lin)[0] for k in (2, 3)])
    want_tlp = np.float32([LO.tlp100(crop(T[2]), crop(T[3]), crop(R[2]), crop(R[3]), alex, lin)])
    assert set(r) == {"PSNR", "SSIM", "LPIPS", "tLP100"}
    assert _close(r["LPIPS"], float(want_lp.mean()), 1e-6, 1e-9)
    assert _close(r["tLP100"], float(want_tlp.mean()), 1e-4, 1e-7)
    txt = open(log / "metrics.csv").read()
    for key in ("LPIPS_00", "tLP100_00", "FolderAvg_LPIPS", "FolderAvg_tLP100", "Avg_tLP100", "FrameAvg_LPIPS"):
        assert key in txt, key
    lines = open(log / "metricsfile.txt").read().splitlines()
    frames = [l for l in lines if l.startswith("frame ")]
    assert len(frames) == 2
    assert ", lpips " in frames[0] and "tLPx100" not in frames[0]
    assert ", lpips " in frames[1] and ", tLPx100 " in frames[1] and frames[1].index("tLPx100") < frames[1].index("crop (")
