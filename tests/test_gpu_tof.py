"""GPU: tOF (tecogan_b200/tof.py -> tecogan_b200/csrc/farneback.cu) against cv2's flows and the reference loop's tOF
stored in tests/golden/tof.npz (rebuilt by tests/golden/make_golden_tof.py::load to within 3e-8 px of cv2's), and each
stage against the host restatement tests/golden/farneback_oracle.py.

Stage tolerances.  The kernels evaluate the restatement's operations in the same order, each correctly rounded, so the
stages normally agree bit for bit; the bounds allow the Gaussian and polynomial taps (computed by the C library's and by
numpy's exp) to differ in their last bit.  A result that sums T rounded terms of magnitude <= A is off by at most about
T * A * 2^-24 from such a tap change, which sets each bound:
  pyramid level   T = 2 (2r + 1) + 4 taps and the resize (r <= 9), A = 255
  expansion       T = 3 * 11 (vertical fp32 pass feeding the float64 horizontal one), A = max |coefficient|
  iteration       same R and flow in: bit-equal field, float64 sums; 1e-6 px leaves room for one ulp of the field
  flow resize     T = 6, A = max |flow|
End to end: |d| <= 1e-3 px against cv2 at every pixel whose final 2x2 system is well conditioned, <= 2e-2 px on the
near-singular pixels the fixture names (`ill<i>`: smallest eigenvalue of the box-mean matrix < 0.05, where cv2's own SIMD
and scalar builds differ by up to 1.3e-3 px), mean |d| <= 1e-5 px.  tOF: 1e-4 per frame, 1e-5 for the folder average."""
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24


def _g():
    from tests.golden import make_golden_tof as MG
    return MG.load()


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _case(g, name):
    names = [str(n) for n in g["names"]]
    i = [k for k, n in enumerate(names) if n.startswith(name)][0]
    return g["prev%d" % i], g["next%d" % i], g["flow%d" % i], g["ill%d" % i]


def test_grey_is_bit_exact_for_every_colour():
    from tecogan_b200 import tof as TOF
    c = torch.arange(1 << 24, device="cuda", dtype=torch.int64)
    rgb = torch.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1)
    want = ((9798 * rgb[:, 0] + 19235 * rgb[:, 1] + 3735 * rgb[:, 2] + 16384) >> 15).to(torch.uint8)
    got = TOF.grey(rgb.to(torch.uint8).reshape(1, 4096, 4096, 3))
    assert torch.equal(got.reshape(-1), want)
    img = rgb[:97 * 131 * 2].to(torch.uint8).reshape(2, 97, 131, 3)                 # through a window
    assert torch.equal(TOF.grey(img, (3, 5, 80, 100)), want[:97 * 131 * 2].reshape(2, 97, 131)[:, 3:83, 5:105])


def test_pyramid_levels_match_host_restatement():
    from tests.golden import farneback_oracle as F
    from tecogan_b200 import tof as TOF
    g = _g()
    for name in ("x2", "ragged", "32x32"):
        prev = _case(g, name)[0]
        for k in range(F.num_levels(*prev.shape[1:]) + 1):
            got = TOF.pyramid_level(_cu(prev), k).cpu().numpy()
            r = F.blur_params(k)[1] // 2
            bound = (2 * (2 * r + 1) + 4) * 255 * EPS
            for p in range(prev.shape[0]):
                want = F.pyramid_level(prev[p], k)
                assert got[p].shape == want.shape, (name, k)
                assert np.abs(got[p] - want).max() <= bound, (name, k, np.abs(got[p] - want).max())


def test_polynomial_expansion_matches_host_restatement():
    from tests.golden import farneback_oracle as F
    from tecogan_b200 import tof as TOF
    g = _g()
    for name in ("calendar", "ragged", "32x32"):
        prev = _case(g, name)[0]
        for k in range(F.num_levels(*prev.shape[1:]) + 1):
            lev = np.stack([F.pyramid_level(a, k) for a in prev])
            got = TOF.poly_exp(_cu(lev)).cpu().numpy()
            for p in range(prev.shape[0]):
                want = F.poly_exp(lev[p])
                for c in range(5):
                    bound = 33 * EPS * np.abs(want[..., c]).max() + 1e-30
                    assert np.abs(got[p, ..., c] - want[..., c]).max() <= bound, (name, k, c)


def test_one_iteration_matches_host_restatement():
    from tests.golden import farneback_oracle as F
    from tecogan_b200 import tof as TOF
    g = _g()
    for name in ("calendar", "large motion", "flat"):
        prev, nxt, flow, _ = _case(g, name)
        P = prev.shape[0]
        R = np.concatenate([np.stack([F.poly_exp(F.pyramid_level(a, 0)) for a in prev]),
                            np.stack([F.poly_exp(F.pyramid_level(b, 0)) for b in nxt])])
        pairs = [(p, P + p) for p in range(P)]
        for fin in (None, flow):
            out = torch.empty(flow.shape, device="cuda", dtype=torch.float32)
            TOF.iterate(_cu(R), pairs, None if fin is None else _cu(fin), out)
            got = out.cpu().numpy()
            for p in range(P):
                want = F.iterate(R[p], R[P + p], np.zeros_like(flow[p]) if fin is None else fin[p])
                assert np.abs(got[p] - want).max() <= 1e-6, (name, fin is None, np.abs(got[p] - want).max())


def test_flow_resize_matches_host_restatement():
    from tests.golden import farneback_oracle as F
    from tecogan_b200 import tof as TOF
    g = _g()
    for name in ("x2", "ragged", "large motion"):
        prev, _, flow, _ = _case(g, name)
        H, W = prev.shape[1:]
        for k in range(F.num_levels(H, W), 0, -1):
            sh, sw = F.level_size(H, W, k)
            h, w = F.level_size(H, W, k - 1)
            coarse = np.stack([F.resize_linear(f, sh, sw) for f in flow])
            got = TOF.flow_up(_cu(coarse), h, w).cpu().numpy()
            for p in range(flow.shape[0]):
                want = F.flow_up(coarse[p], h, w)
                assert np.abs(got[p] - want).max() <= 6 * EPS * np.abs(want).max() + 1e-30, (name, k)


def test_flows_match_cv2_on_every_fixture():
    from tecogan_b200 import tof as TOF
    g = _g()
    from tests.golden import make_golden_tof as MG
    for i in range(g["n_cases"]):
        name = str(g["names"][i])
        got = TOF.farneback(_cu(g["prev%d" % i]), _cu(g["next%d" % i])).cpu().numpy()
        ref, ill = g["flow%d" % i], g["ill%d" % i]
        assert got.shape == ref.shape, name
        assert np.abs(ref[:, ::MG.SAMPLE, ::MG.SAMPLE] - g["sample%d" % i]).max() <= 1e-7, name     # rebuilt = cv2
        for p in range(ref.shape[0]):
            d = np.abs(got[p] - ref[p]).max(-1)
            assert d[~ill[p]].max() <= 1e-3, (name, p, d[~ill[p]].max())
            assert not ill[p].any() or d[ill[p]].max() <= 2e-2, (name, p, d[ill[p]].max())
            assert d.mean() <= 1e-5, (name, p, d.mean())


def test_sequence_tof_matches_reference_loop():
    from tecogan_b200 import metrics as M
    g = _g()
    T, R, cut = _cu(g["seq_tgt"]), _cu(g["seq_out"]), int(g["cutfr"])
    want = g["seq_tof"]
    r = M.evaluate_sequence(T, R, cut, tof=True)
    assert len(r["tOF"]) == len(r["PSNR"]) - 1 == len(want)
    assert np.abs(np.array(r["tOF"]) - want).max() <= 1e-4
    assert abs(r["FolderAvg_tOF"] - want.mean()) <= 1e-5
    base = M.evaluate_sequence(T, R, cut)
    assert set(base) == {"PSNR", "SSIM", "FolderAvg_PSNR", "FolderAvg_SSIM"}        # the default is unchanged
    assert np.allclose(base["PSNR"], r["PSNR"], rtol=1e-12, atol=0) and np.allclose(base["SSIM"], r["SSIM"], rtol=1e-12, atol=0)
    # a larger result is cut to the target (metrics.py:139-140): padding it on the bottom / right changes nothing
    Rp = torch.nn.functional.pad(R.permute(0, 3, 1, 2), (0, 5, 0, 3)).permute(0, 2, 3, 1).contiguous()
    assert M.evaluate_sequence(T, Rp, cut, tof=True)["tOF"] == r["tOF"]


def test_batch_invariance():
    from tecogan_b200 import tof as TOF
    g = _g()
    from tests.golden import farneback_oracle as F
    prev, nxt = _case(g, "calendar")[:2]
    gs = F.grey(g["seq_tgt"])
    pa = np.concatenate([prev, gs[:-1], gs[0:4]])
    pb = np.concatenate([nxt, gs[1:], gs[2:6]])                                  # frames two apart
    assert pa.shape[0] == 12
    batch = TOF.farneback(_cu(pa), _cu(pb))
    for p in (0, 5, 11):
        alone = TOF.farneback(_cu(pa[p:p + 1]), _cu(pb[p:p + 1]))
        assert torch.equal(alone[0], batch[p]), p


def test_tof_rejects_a_frame_the_crop_empties():
    from tecogan_b200 import tof as TOF
    x = torch.zeros((3, 40, 64, 3), device="cuda", dtype=torch.uint8)
    with pytest.raises(ValueError, match="crop_8x8"):
        TOF.tof_sequence(x, x)
    with pytest.raises(ValueError):
        TOF.farneback(torch.zeros((2, 8, 8), device="cuda", dtype=torch.uint8), torch.zeros((2, 8, 9), device="cuda", dtype=torch.uint8))


def _write_pngs(tmp_path, T, R):
    from PIL import Image
    res, tar = tmp_path / "results" / "scene", tmp_path / "HR" / "scene"
    res.mkdir(parents=True)
    tar.mkdir(parents=True)
    for k in range(len(T)):
        Image.fromarray(T[k]).save(tar / ("%04d.png" % k))
        Image.fromarray(R[k]).save(res / ("output_%04d.png" % k))
    return res, tar


def test_metrics_command_line_with_tof_on_png_folders(tmp_path):
    """Root metrics.py --tof: tOF in the per-frame lines before psnr (metrics.py:169), tOF_00 / FolderAvg_tOF in
    metrics.csv, values equal to the reference loop's.  Without the flag the same folders give today's keys, lines and
    columns, with no tOF anywhere."""
    import metrics as CLI
    g = _g()
    T, R = g["seq_tgt"], g["seq_out"]
    res, tar = _write_pngs(tmp_path, T, R)
    with_log, plain_log = tmp_path / "with", tmp_path / "plain"
    r = CLI.main(["--output", str(with_log), "--results", str(res), "--targets", str(tar), "--tof"])
    p = CLI.main(["--output", str(plain_log), "--results", str(res), "--targets", str(tar)])
    assert list(r) == ["PSNR", "SSIM", "tOF"] and list(p) == ["PSNR", "SSIM"]
    assert abs(r["tOF"] - float(np.float32(g["seq_tof"]).mean())) <= 1e-5
    assert abs(r["PSNR"] - p["PSNR"]) <= 1e-5 and abs(r["SSIM"] - p["SSIM"]) <= 1e-6
    lines = open(with_log / "metricsfile.txt").read().splitlines()
    plain = open(plain_log / "metricsfile.txt").read().splitlines()
    frames = [l for l in lines if l.startswith("frame ")]
    assert len(frames) == 3
    assert "tOF" not in frames[0]
    for l, v in zip(frames[1:], g["seq_tof"]):
        assert (", tOF %02.2f, psnr " % v) in l, l
    assert not any("tOF" in l for l in plain)
    assert [re.sub(r"tOF [0-9.]+, ", "", l) for l in lines if not l.startswith("tOF")] == plain
    csv, plain_csv = open(with_log / "metrics.csv").read(), open(plain_log / "metrics.csv").read()
    for key in ("tOF_00", "Avg_tOF", "FolderAvg_tOF", "FrameAvg_tOF"):
        assert key in csv and key not in plain_csv, key
    assert csv.splitlines()[0] == ",PSNR_00,SSIM_00,tOF_00"
    assert plain_csv.splitlines()[0] == ",PSNR_00,SSIM_00"
