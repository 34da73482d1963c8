"""Generate tests/golden/lpips.npz by executing the REFERENCE's own LPIPS code.

The reference computes LPIPS through LPIPSmodels (networks_basic.PNetLin, util.im2tensor; metrics.py:183-202).  Those
modules are imported from the checkout named by $TECOGAN_REFERENCE (never copied into the repo) with MagicMock stubs for
the optional imports that are not installed and that the LPIPS arithmetic never calls (skimage, IPython, matplotlib, and
cv2 / scipy.ndimage.interpolation where missing).  torchvision is needed here only, to build the AlexNet module.

The backbone is PNetLin(pnet_type='alex', pnet_rand=True, version='0.1') with its features loaded from the seeded test
weights tests/golden/lpips_oracle.py::lpips_test_weights(ALEX_SEED) -- about 10 MB, so only the seed is stored.  The linear weights
are the reference's real v0.1 values (LPIPSmodels/v0.1/alex.pth, 1152 floats), stored in the npz.
Stored: uncropped uint8 frame pairs with their crop_8x8 windows, the fp32 LPIPS the reference reports for each pair, the
per-layer d_l of each pair (float64 run, see below), and a 7-frame sequence with the loop's LPIPS and tLP100 lists.
The frame loop's LPIPS / tLP100 formulas (metrics.py:183-202) are restated around the reference's model call.
Run once:  TECOGAN_REFERENCE=/path/to/TecoGAN python tests/golden/make_golden_lpips.py
"""
import os
import sys
from unittest.mock import MagicMock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("TECOGAN_REFERENCE", "TecoGAN")
ALEX_SEED = 20261015
CUTFR = 2
# (seed, target h, target w, result h, result w, noise): a plain case, the ragged 144x180, a 48x60 frame whose crop is
# 32x32 (relu3..relu5 are 1x1), and a wide one.
CASES = [(0, 96, 128, 96, 128, 6.0), (1, 144, 180, 144, 180, 9.0), (2, 48, 60, 48, 60, 12.0), (3, 120, 232, 120, 232, 3.0)]
SEQ = (7, 66, 84, 68, 84)        # frames, target h, w, result h, w (the result is cut to the target, metrics.py:134-135)


def reference_modules():
    for name in ("skimage", "skimage.color", "skimage.measure", "skimage.transform", "IPython", "matplotlib",
                 "matplotlib.pyplot"):
        sys.modules[name] = MagicMock()
    for name in ("cv2", "scipy.ndimage.interpolation"):
        try:
            __import__(name)
        except ImportError:
            sys.modules[name] = MagicMock()
    sys.path.insert(0, REF)
    sys.path.insert(0, ROOT)
    import LPIPSmodels.networks_basic as nb
    import LPIPSmodels.util as util
    from tests.golden.make_golden_metrics import SRC, reference_functions
    assert os.path.exists(SRC), SRC
    return nb, util, reference_functions()["crop_8x8"]


def reference_model(nb, alex_sd, lin_sd):
    net = nb.PNetLin(pnet_type="alex", pnet_rand=True, use_gpu=False, spatial=False, version="0.1")
    backbone = net.net[0]
    # alexnet().features[k] sits in slice s of pretrained_networks.alexnet (pretrained_networks.py:67-76)
    slot = {0: 1, 3: 2, 6: 3, 8: 4, 10: 5}
    sd = {"slice%d.%d.%s" % (slot[int(k.split(".")[1])], int(k.split(".")[1]), k.split(".")[2]): v for k, v in alex_sd.items()}
    backbone.load_state_dict(sd)
    net.load_state_dict(lin_sd)
    net.eval()
    backbone.eval()
    return net


def frames(seed, h, w, oh, ow, noise):
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:oh, 0:ow]
    base = np.stack([127 + 90 * np.sin(xx / (5.0 + c) + c) * np.cos(yy / 4.0 - c) for c in range(3)], -1)
    big = np.clip(np.round(base + r.randn(oh, ow, 3) * 8), 0, 255).astype(np.uint8)
    out = np.clip(np.round(big.astype(np.float64) + r.randn(oh, ow, 3) * noise), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(big[:h, :w]), out


def main():
    nb, util, crop_8x8 = reference_modules()
    from tests.golden.lpips_oracle import lpips_test_weights
    lin_sd = torch.load(os.path.join(REF, "LPIPSmodels", "v0.1", "alex.pth"), map_location="cpu", weights_only=True)
    net = reference_model(nb, lpips_test_weights(ALEX_SEED), lin_sd)

    def dist(a, b):                     # DistModel.forward(..., retNumpy=True): dist_model.py:111-143
        with torch.no_grad():
            return net.forward(a, b).cpu().data.numpy().flatten()

    # Per-layer d_l: the spatial=True maps (networks_basic.py:160-165) averaged over the pixels, from a float64 copy of
    # the same network fed the same fp32 im2tensor inputs.  The fp32 run's d_l carry its own rounding: on the 32x32 crop,
    # where relu3..relu5 are one pixel and nothing averages it out, relu5's d_l is off by 5e-6 relative, while the fp32
    # and float64 runs of the summed LPIPS agree to below 1e-6.
    net64 = reference_model(nb, lpips_test_weights(ALEX_SEED), lin_sd).double()
    net64.net[0].double()
    net64.spatial = True

    def per_layer(a, b):
        with torch.no_grad():
            maps = net64.forward(a.double(), b.double())
        return np.float64([m.mean().item() for m in maps])

    kw = {"alex_seed": np.int64(ALEX_SEED), "cutfr": np.int64(CUTFR), "n_cases": np.int64(len(CASES))}
    for l in range(5):
        kw["lin%d" % l] = lin_sd["lin%d.model.1.weight" % l].numpy().reshape(-1).astype(np.float32)
    for i, (seed, h, w, oh, ow, noise) in enumerate(CASES):
        tgt, out = frames(seed, h, w, oh, ow, noise)
        ct, y, x = crop_8x8(tgt)
        co, _, _ = crop_8x8(out)
        a, b = util.im2tensor(ct), util.im2tensor(co)
        kw["tgt%d" % i], kw["out%d" % i] = tgt, out
        kw["crop%d" % i] = np.array([y, x, ct.shape[0], ct.shape[1]], dtype=np.int64)
        kw["lpips%d" % i] = np.float64(dist(a, b)[0])
        kw["layers%d" % i] = per_layer(a, b)

    n, h, w, oh, ow = SEQ
    T, R = [], []
    for k in range(n):
        t, o = frames(100 + k, h + 2 * k, w + 3 * k, oh + 2 * k, ow + 3 * k, 7.0)
        T.append(t[2 * k:, 3 * k:])      # the scene moves by (2, 3) pixels per frame
        R.append(o[2 * k:, 3 * k:])
    lp, tlp = [], []
    for i in range(CUTFR, n - CUTFR):    # metrics.py:131-202, LPIPS and tLP100 only
        output_img, target_img = R[i], T[i]
        if target_img.shape[0] < output_img.shape[0] or target_img.shape[1] < output_img.shape[1]:
            output_img = output_img[:target_img.shape[0], :target_img.shape[1]]
        target_img, _, _ = crop_8x8(target_img)
        output_img, _, _ = crop_8x8(output_img)
        img0, img1 = util.im2tensor(target_img), util.im2tensor(output_img)
        lp.append(dist(img0, img1)[0])
        if i > CUTFR:
            dist0t, dist1t = dist(pre_img0, img0), dist(pre_img1, img1)   # noqa: F821 (set on the previous frame)
            tlp.append((np.absolute(dist0t - dist1t) * 100.0)[0])
        pre_img0, pre_img1 = img0, img1
    kw["seq_tgt"], kw["seq_out"] = np.stack(T), np.stack(R)
    kw["seq_lpips"], kw["seq_tlp100"] = np.float64(lp), np.float64(tlp)
    path = os.path.join(HERE, "lpips.npz")
    np.savez_compressed(path, **kw)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
