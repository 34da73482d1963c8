"""CPU restatement of LPIPS-AlexNet v0.1 and tLP100 in float64 (reference metrics.py:183-202).  TEST INFRASTRUCTURE ONLY.

Written from the definition, not from LPIPSmodels: the input scaling of util.im2tensor and the v0.1 scaling layer,
torchvision alexnet().features[0:12] tapped after each ReLU, and the PNetLin head.  The network input is first rounded to
fp32 exactly as the reference does (im2tensor makes a float32 tensor, the scaling layer is fp32); every later step is
float64.  lpips_test_weights(seed) is the one definition of the seeded backbone that stands in for torchvision's ImageNet
AlexNet in tests/golden/lpips.npz (make_golden_lpips.py), the tests and tools/bench_lpips.py.

Checked against the reference's own LPIPSmodels outputs by tests/test_lpips_host.py.
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

LPIPS_SHIFT = np.float32([-.030, -.088, -.188])
LPIPS_SCALE = np.float32([.458, .448, .450])
# (state-dict prefix, Cin, Cout, kernel, stride, pad) of the five convolutions; MaxPool2d(3, 2) follows relu1 and relu2
ALEXNET_CONVS = [("features.0", 3, 64, 11, 4, 2), ("features.3", 64, 192, 5, 1, 2), ("features.6", 192, 384, 3, 1, 1),
                 ("features.8", 384, 256, 3, 1, 1), ("features.10", 256, 256, 3, 1, 1)]


def lpips_test_weights(seed):
    """The seeded stand-in for torchvision's ImageNet AlexNet: a torchvision-format state dict (features.* only) of fp32
    tensors, He-normal weights (std sqrt(2 / fan_in)) and N(0, 0.05) biases from numpy's default_rng(seed)."""
    rng = np.random.default_rng(seed)
    sd = OrderedDict()
    for name, cin, cout, k, _, _ in ALEXNET_CONVS:
        sd[name + ".weight"] = torch.from_numpy(rng.normal(0.0, math.sqrt(2.0 / (cin * k * k)), (cout, cin, k, k)).astype(np.float32))
        sd[name + ".bias"] = torch.from_numpy(rng.normal(0.0, 0.05, cout).astype(np.float32))
    return sd


def lpips_input(img_u8):
    """util.py:142-144 then networks_basic.py:131-132 on one uint8 RGB frame [h,w,3] -> fp32 [h,w,3]."""
    x = (np.asarray(img_u8) / 127.5 - 1.0).astype(np.float32)
    return (x - LPIPS_SHIFT) / LPIPS_SCALE


def alexnet_features(img_u8, alex):
    """relu1 .. relu5 of one already-cropped uint8 RGB frame, as float64 NHWC arrays [1,h_l,w_l,C_l]."""
    if min(img_u8.shape[0], img_u8.shape[1]) < 31:
        raise ValueError("LPIPS-AlexNet needs at least 31x31 pixels, got %dx%d" % img_u8.shape[:2])
    x = torch.from_numpy(lpips_input(img_u8).astype(np.float64)).permute(2, 0, 1)[None]
    feats = []
    for l, (name, _, _, _, stride, pad) in enumerate(ALEXNET_CONVS):
        if l in (1, 2):
            x = F.max_pool2d(x, 3, 2)
        w, b = alex[name + ".weight"].double(), alex[name + ".bias"].double()
        x = torch.relu(F.conv2d(x, w, b, stride=stride, padding=pad))
        feats.append(x.permute(0, 2, 3, 1).numpy())
    return feats


def lpips_from_features(fa, fb, lin):
    """The PNetLin head (networks_basic.py:150-177, util.py:72-75) on two feature lists: (LPIPS, [d_l])."""
    ds = []
    for l, (a, b) in enumerate(zip(fa, fb)):
        w = np.asarray(lin["lin%d.model.1.weight" % l], dtype=np.float64).reshape(-1)
        na = np.sqrt((a * a).sum(-1, keepdims=True)) + 1e-10
        nb = np.sqrt((b * b).sum(-1, keepdims=True)) + 1e-10
        ds.append(float(((a / na - b / nb) ** 2 * w).sum(-1).mean()))
    return sum(ds), ds


def lpips(img0_u8, img1_u8, alex, lin):
    """model.forward(im2tensor(img0), im2tensor(img1))[0] of metrics.py:186-188 on two cropped uint8 frames: (LPIPS, [d_l])."""
    return lpips_from_features(alexnet_features(img0_u8, alex), alexnet_features(img1_u8, alex), lin)


def tlp100(pre_tar_u8, tar_u8, pre_out_u8, out_u8, alex, lin):
    """metrics.py:194-198: 100 |LPIPS(previous target, target) - LPIPS(previous result, result)| on cropped frames."""
    return 100.0 * abs(lpips(pre_tar_u8, tar_u8, alex, lin)[0] - lpips(pre_out_u8, out_u8, alex, lin)[0])
