"""CPU: the float64 LPIPS / tLP100 oracle against the reference's own LPIPSmodels outputs (tests/golden/lpips.npz), the
weight loaders of tecogan_b200/lpips.py, and the metrics command line's LPIPS flags.

Tolerances: LPIPS and each d_l |d| <= 1e-6 |ref| + 1e-9 (the reference's fp32 LPIPS agrees with float64 runs to about
3e-7 relative; the stored d_l come from a float64 run of the reference network), tLP100 <= 1e-4 |ref| + 1e-7 (100 x a
difference of two fp32 distances)."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN


def _g():
    return np.load(os.path.join(GOLDEN, "lpips.npz"), allow_pickle=False)


def _lin(g):
    return {"lin%d.model.1.weight" % l: torch.from_numpy(g["lin%d" % l]).reshape(1, -1, 1, 1) for l in range(5)}


def _crop(img, win):
    y, x, h, w = (int(v) for v in win)
    return np.ascontiguousarray(img[y:y + h, x:x + w])


def test_oracle_matches_reference_lpips_and_layers():
    from tests.golden import lpips_oracle as LO
    g = _g()
    alex, lin = LO.lpips_test_weights(int(g["alex_seed"])), _lin(g)
    for i in range(int(g["n_cases"])):
        win = g["crop%d" % i]
        total, layers = LO.lpips(_crop(g["tgt%d" % i], win), _crop(g["out%d" % i], win), alex, lin)
        ref = float(g["lpips%d" % i])
        assert abs(total - ref) <= 1e-6 * abs(ref) + 1e-9, (i, total, ref)
        for l, (d, r) in enumerate(zip(layers, g["layers%d" % i])):
            assert abs(d - r) <= 1e-6 * abs(r) + 1e-9, (i, l, d, r)
    assert [tuple(g["crop%d" % i][2:]) for i in range(4)][2] == (32, 32)      # the 1x1-deep-layer case is present


def test_oracle_matches_reference_sequence_loop():
    from oracle import teco_oracle as O
    from tests.golden import lpips_oracle as LO
    g = _g()
    alex, lin = LO.lpips_test_weights(int(g["alex_seed"])), _lin(g)
    T, R, cut = g["seq_tgt"], g["seq_out"], int(g["cutfr"])
    crop = lambda a: np.ascontiguousarray(O.crop_8x8(a))                        # noqa: E731
    R = R[:, :T.shape[1], :T.shape[2]]                                           # metrics.py:134-135
    lp = [LO.lpips(crop(T[i]), crop(R[i]), alex, lin)[0] for i in range(cut, len(T) - cut)]
    tlp = [LO.tlp100(crop(T[i - 1]), crop(T[i]), crop(R[i - 1]), crop(R[i]), alex, lin) for i in range(cut + 1, len(T) - cut)]
    assert len(lp) == len(T) - 2 * cut and len(tlp) == len(lp) - 1
    for a, r in zip(lp, g["seq_lpips"]):
        assert abs(a - r) <= 1e-6 * abs(r) + 1e-9
    for a, r in zip(tlp, g["seq_tlp100"]):
        assert abs(a - r) <= 1e-4 * abs(r) + 1e-7


def test_oracle_feature_sizes_and_minimum_crop():
    from tests.golden import lpips_oracle as LO
    from tecogan_b200 import lpips as L
    alex = LO.lpips_test_weights(0)
    for h, w in ((31, 31), (32, 47), (71, 38)):
        got = [tuple(f.shape[1:3]) for f in LO.alexnet_features(np.zeros((h, w, 3), np.uint8), alex)]
        assert got == L.feature_sizes(h, w), (h, w)
    assert L.feature_sizes(31, 32)[2:] == [(1, 1)] * 3
    assert L.feature_sizes(544, 704) == [(135, 175), (67, 87), (33, 43), (33, 43), (33, 43)]
    with pytest.raises(ValueError):
        L.feature_sizes(30, 64)
    with pytest.raises(ValueError):
        LO.alexnet_features(np.zeros((64, 30, 3), np.uint8), alex)


def _torchvision_file(tmp_path, sd):
    """A torchvision-format AlexNet state dict on disk: features.* plus a classifier key the loader must ignore."""
    full = dict(sd)
    full["classifier.1.weight"] = torch.zeros(8, 4)
    path = tmp_path / "alexnet-owt-test.pth"
    torch.save(full, path)
    return str(path)


def test_load_alexnet_transposes_to_tf_layout_and_ignores_classifier(tmp_path):
    from tests.golden import lpips_oracle as LO
    from tecogan_b200 import lpips as L
    sd = LO.lpips_test_weights(7)
    convs = L.load_alexnet(_torchvision_file(tmp_path, sd))
    assert len(convs) == 5
    for (w, b), (name, cin, cout, k, _, _) in zip(convs, L.ALEXNET_CONVS):
        assert tuple(w.shape) == (k, k, cin, cout) and w.is_contiguous() and w.dtype == torch.float32
        src = sd[name + ".weight"]
        assert torch.equal(w[2, 1, :, 5 % cout], src[5 % cout, :, 2, 1])      # [ky,kx,ci,co] = torch[co,ci,ky,kx]
        assert torch.equal(w, src.permute(2, 3, 1, 0))
        assert torch.equal(b, sd[name + ".bias"])
    assert torch.equal(L.tf_layout(torch.arange(24.).reshape(2, 3, 2, 2))[1, 0], torch.arange(24.).reshape(2, 3, 2, 2)[:, :, 1, 0].T)


def test_load_alexnet_and_lin_reject_missing_or_misshapen_keys(tmp_path):
    from tests.golden import lpips_oracle as LO
    from tecogan_b200 import lpips as L
    sd = LO.lpips_test_weights(7)
    bad = dict(sd)
    del bad["features.8.bias"]
    with pytest.raises(ValueError, match="features.8.bias"):
        L.load_alexnet(bad)
    bad = dict(sd)
    bad["features.3.weight"] = torch.zeros(192, 64, 3, 3)
    with pytest.raises(ValueError, match="features.3.weight"):
        L.load_alexnet(bad)
    with pytest.raises(ValueError):
        L.load_alexnet([1, 2, 3])
    g = _g()
    path = tmp_path / "alex.pth"
    torch.save(_lin(g), path)
    lins = L.load_lin(str(path))
    assert [tuple(v.shape) for v in lins] == [(c,) for c in L.LIN_CHANNELS]
    assert np.array_equal(lins[2].numpy(), g["lin2"])
    bad = _lin(g)
    del bad["lin4.model.1.weight"]
    with pytest.raises(ValueError, match="lin4"):
        L.load_lin(bad)
    bad = _lin(g)
    bad["lin1.model.1.weight"] = torch.zeros(1, 64, 1, 1)
    with pytest.raises(ValueError, match="lin1"):
        L.load_lin(bad)


def test_metrics_command_line_needs_both_lpips_flags(tmp_path, capsys):
    import metrics as CLI
    out = tmp_path / "log"
    for flag in ("--lpips_alexnet", "--lpips_lin"):
        with pytest.raises(SystemExit) as e:
            CLI.main(["--output", str(out), "--results", "r", "--targets", "t", flag, str(tmp_path / "w.pth")])
        assert e.value.code == 2
        assert "go together" in capsys.readouterr().err
    assert not out.exists()                                                      # refused before any work
