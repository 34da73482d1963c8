"""CPU: the numpy restatement of Farneback (tests/golden/farneback_oracle.py) against cv2's own flows stored in
tests/golden/tof.npz (exact values at every 7th row and column; make_golden_tof.py), the pyramid sizes of
tecogan_b200/tof.py, and the metrics command line's --tof flag.

Tolerances (same as the generator asserts): |d| <= 1e-3 px at every pixel whose final 2x2 system is well conditioned,
2e-2 px on the near-singular ones the fixture names (`ill<i>`), mean |d| <= 1e-5 px.  cv2's SIMD and scalar builds
differ by up to 1.3e-3 px on near-singular pixels of a large-motion pair, so the per-pixel bound cannot hold there."""
import numpy as np
import pytest


def _g():
    from tests.golden import make_golden_tof as MG
    return MG.load()


def test_oracle_matches_cv2_flows():
    """Against cv2's exact values at the sampled pixels (independent of the stored difference from the restatement),
    and the rebuilt full flow against the same samples."""
    from tests.golden import farneback_oracle as F
    from tests.golden import make_golden_tof as MG
    g = _g()
    levels = set()
    for i in range(g["n_cases"]):
        prev, nxt, ill, sample = g["prev%d" % i], g["next%d" % i], g["ill%d" % i], g["sample%d" % i]
        name = str(g["names"][i])
        for p in range(prev.shape[0]):
            mine = F.farneback(prev[p], nxt[p])[::MG.SAMPLE, ::MG.SAMPLE]
            bad = ill[p][::MG.SAMPLE, ::MG.SAMPLE]
            d = np.abs(mine - sample[p]).max(-1)
            assert d[~bad].max() <= 1e-3, (name, d[~bad].max())
            assert not bad.any() or d[bad].max() <= 2e-2, name
            assert d.mean() <= 1e-5, (name, d.mean())
            assert ill[p].mean() < 0.25                                       # the named pixels stay a minority
            assert np.abs(g["flow%d" % i][p][::MG.SAMPLE, ::MG.SAMPLE] - sample[p]).max() <= 1e-7, name
        levels.add(F.num_levels(*prev.shape[1:]))
    assert levels == {0, 1, 2, 3}                                              # every pyramid depth is covered


def test_oracle_sequence_tof_matches_reference_loop():
    from tests.golden import farneback_oracle as F
    g = _g()
    T, R, cut = g["seq_tgt"], g["seq_out"], int(g["cutfr"])
    gt, go = F.grey(T), F.grey(R)
    got = [F.tof_of_flows(F.farneback(gt[i - 1], gt[i]), F.farneback(go[i - 1], go[i])) for i in range(cut + 1, len(T) - cut)]
    assert len(got) == len(g["seq_tof"]) == len(T) - 2 * cut - 1
    assert np.allclose(got, g["seq_tof"], rtol=0, atol=1e-4)


def test_pyramid_sizes_follow_the_probed_rule():
    from tests.golden import farneback_oracle as F
    from tecogan_b200 import tof as TOF
    for h, w in ((32, 32), (63, 64), (64, 64), (97, 131), (128, 128), (144, 180), (288, 360), (576, 720), (1080, 1920)):
        want = [F.level_size(h, w, k) for k in range(F.num_levels(h, w) + 1)]
        assert TOF.pyramid_sizes(h, w) == want, (h, w)
    assert TOF.pyramid_sizes(97, 131) == [(97, 131), (48, 66)]                # 48.5 -> 48, 65.5 -> 66: half to even
    assert len(TOF.pyramid_sizes(576, 720)) == 4 and len(TOF.pyramid_sizes(32, 32)) == 1


def test_grey_formula_on_a_colour_sample():
    from tests.golden import farneback_oracle as F
    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (4096, 3)).astype(np.uint8)
    f = rgb.astype(np.float64)
    approx = 0.299 * f[:, 0] + 0.587 * f[:, 1] + 0.114 * f[:, 2]
    assert np.abs(F.grey(rgb).astype(np.float64) - approx).max() <= 0.5 + 0.01        # coefficients differ from 0.299 / 0.587 / 0.114 by < 2e-5


def test_metrics_command_line_tof_flag(tmp_path, capsys):
    import metrics as CLI
    assert CLI.metric_keys(False, False) == CLI.KEYS == ["PSNR", "SSIM"]
    assert CLI.metric_keys(True, False) == CLI.KEYS_LPIPS
    assert CLI.metric_keys(False, True) == ["PSNR", "SSIM", "tOF"]
    assert CLI.metric_keys(True, True) == ["PSNR", "SSIM", "LPIPS", "tOF", "tLP100"]     # metrics.py:120 order
    out = tmp_path / "log"
    with pytest.raises(SystemExit) as e:
        CLI.main(["--output", str(out), "--results", "r", "--targets", "t", "--tof=yes"])
    assert e.value.code == 2
    with pytest.raises(SystemExit) as e:
        CLI.main(["--output", str(out), "--results", "r", "--targets", "t", "--tof", "--lpips_lin", str(tmp_path / "w.pth")])
    assert e.value.code == 2
    assert "go together" in capsys.readouterr().err
    assert not out.exists()                                                      # refused before any work
