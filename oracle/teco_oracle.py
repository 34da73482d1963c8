"""CPU oracle for the TecoGAN recurrent video-SR hot path.  TEST INFRASTRUCTURE ONLY.

This file is a plain PyTorch-CPU fp32 (optionally fp64) restatement of the reference's
TF1 graph for the path named in BASELINE.json (SURVEY.md section 8a).  It is imported only by
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
leg -- as the checker or the timed CPU baseline, never by the product package
``tecogan_b200`` (which has no CPU fallback and fails loudly without its CUDA library).

PARITY UNPINNED: the reference ships no tests, golden vectors or stored outputs for this
path, and its arithmetic lives in an un-vendored, un-pinned dependency (``tensorflow`` 1.8+,
``tf.contrib.slim``, ``tf.contrib.image``; see reference README.md:36-37) that cannot be
installed here (Python 3.12, no network).  What *is* pinned: the graph wiring, by executing
the reference's own ``lib/frvsr.py`` / ``lib/ops.py`` / ``lib/Teco.py`` source under a
torch-backed TF shim (tests/golden/make_golden.py -> tests/golden/*.npz) and comparing to
this file.  The TF-primitive semantics (SAME padding, conv2d_transpose alignment, legacy
resize, dense_image_warp, fused batch-norm, Adam) are restated from the published TF 1.x
algorithms (SURVEY.md Appendix A) and are marked [TF-ext] below.

All tensors are NHWC like the reference (lib/ops.py:39,51).  Weights use the TF layouts and
the TF variable names of SURVEY.md Appendix C, held in a plain dict name -> torch.Tensor.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

VGG_MEAN = [123.68, 116.78, 103.94]  # lib/Teco.py:3


# --------------------------------------------------------------------------------------
# TF primitives [TF-ext]
# --------------------------------------------------------------------------------------
def _same_pad(n, k, s):
    """TF 'SAME' padding for one axis: (before, after).  [TF-ext] SURVEY A.2."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def conv2d(x, w, b=None, stride=1):
    """slim.conv2d(..., 'SAME', NHWC, activation_fn=None) -- lib/ops.py:47-56.
    x [N,H,W,Cin], w HWIO [kh,kw,Cin,Cout], cross-correlation."""
    kh, kw = w.shape[0], w.shape[1]
    pt, pb = _same_pad(x.shape[1], kh, stride)
    pl, pr = _same_pad(x.shape[2], kw, stride)
    xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xn, w.permute(3, 2, 0, 1), b, stride=stride)
    return y.permute(0, 2, 3, 1).contiguous()


def conv2d_transpose(x, w, b=None, stride=2):
    """slim.conv2d_transpose(..., 3x3, stride 2, 'SAME') -- lib/ops.py:35-44.  [TF-ext] SURVEY A.3.
    w is [kh,kw,Cout,Cin].  It is the input-gradient of a stride-2 SAME conv over a 2N-sized
    image (pad before 0, after 1), i.e. y[i] = sum_j x[j] w[i-2j], cropped to [0,2N)."""
    assert stride == 2 and w.shape[0] == 3 and w.shape[1] == 3
    n, h, wd, _ = x.shape
    y = F.conv_transpose2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, stride=2, padding=0)
    return y[:, :, : 2 * h, : 2 * wd].permute(0, 2, 3, 1).contiguous()


def lrelu(x, alpha=0.2):
    """keras LeakyReLU -- lib/ops.py:84-85."""
    return torch.where(x >= 0, x, alpha * x)


def maxpool(x):
    """slim.max_pool2d([2,2]) stride 2 VALID -- lib/ops.py:92-93."""
    return F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()


def resize_bilinear_legacy(x, oh, ow):
    """tf.image.resize_images default (bilinear, align_corners=False, legacy coordinates:
    src = dst * in/out).  [TF-ext] SURVEY A.5.  lib/frvsr.py:21-22, lib/Teco.py:244."""
    n, h, w, c = x.shape

    def axis(inn, out):
        src = torch.arange(out, dtype=x.dtype) * (inn / out)
        lo = torch.floor(src).long()
        hi = torch.clamp(lo + 1, max=inn - 1)
        return lo, hi, (src - lo.to(x.dtype))

    y0, y1, wy = axis(h, oh)
    x0, x1, wx = axis(w, ow)
    top = x[:, y0]
    bot = x[:, y1]
    wx_ = wx.view(1, 1, ow, 1)
    wy_ = wy.view(1, oh, 1, 1)
    t = top[:, :, x0] + (top[:, :, x1] - top[:, :, x0]) * wx_
    bt = bot[:, :, x0] + (bot[:, :, x1] - bot[:, :, x0]) * wx_
    return t + (bt - t) * wy_


def dense_image_warp(image, flow):
    """tf.contrib.image.dense_image_warp.  [TF-ext] SURVEY A.7.
    out[b,y,x] = bilinear(image[b], (y - flow[b,y,x,0], x - flow[b,y,x,1])), floor clamped to
    [0,size-2], alpha clamped to [0,1].  lib/Teco.py:120,140,224,254; main.py:215.
    Gradient to the query only where 0 < alpha_raw <= 1: TF clamps with minimum(maximum(0, a), 1), and at a tie
    Maximum's gradient goes to its first argument (the constant 0) and Minimum's to its first argument (a).
    torch.clamp would pass it at both ends, so at every integer query."""
    n, h, w, c = image.shape
    gy = torch.arange(h, dtype=image.dtype).view(1, h, 1)
    gx = torch.arange(w, dtype=image.dtype).view(1, 1, w)
    qy = gy - flow[..., 0]
    qx = gx - flow[..., 1]

    def split(q, size):
        fl = torch.clamp(torch.floor(q), 0, size - 2)
        a = q - fl
        al = torch.clamp(a, 0.0, 1.0)
        al = torch.where((a > 0) & (a <= 1), al, al.detach())
        return fl.long(), al

    y0, ay = split(qy, h)
    x0, ax = split(qx, w)
    bidx = torch.arange(n).view(n, 1, 1).expand(n, h, w)
    tl = image[bidx, y0, x0]
    tr = image[bidx, y0, x0 + 1]
    bl = image[bidx, y0 + 1, x0]
    br = image[bidx, y0 + 1, x0 + 1]
    ax = ax.unsqueeze(-1)
    ay = ay.unsqueeze(-1)
    top = ax * (tr - tl) + tl
    bot = ax * (br - bl) + bl
    return ay * (bot - top) + top


def batchnorm_train(x, beta, eps=1e-3):
    """slim.batch_norm(decay=.9, eps=1e-3, scale=False, fused=True, is_training=True)
    -- lib/ops.py:88-90.  [TF-ext] SURVEY A.10: biased batch variance, no gamma."""
    mean = x.mean(dim=(0, 1, 2), keepdim=True)
    var = ((x - mean) ** 2).mean(dim=(0, 1, 2), keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) + beta


# --------------------------------------------------------------------------------------
# in-tree ops (spelled out by the reference)
# --------------------------------------------------------------------------------------
def preprocess(x):  # lib/ops.py:13-16
    return x * 2 - 1


def deprocess(x):  # lib/ops.py:19-22
    return (x + 1) / 2


def upscale_four(x):
    """lib/ops.py:126-163: legacy bilinear x4, out[4i+k] = (1-k/4) x[i] + (k/4) x[min(i+1,n-1)]."""
    n, h, w, c = x.shape
    p = torch.cat((x, x[:, -1:]), dim=1)
    p = torch.cat((p, p[:, :, -1:]), dim=2)
    tl, tr, bl, br = x, p[:, :-1, 1:], p[:, 1:, :-1], p[:, 1:, 1:]
    outs = []
    for hi in range(4):
        for wj in range(4):
            outs.append(tl * (1.0 - 0.25 * hi) * (1.0 - 0.25 * wj) + tr * (1.0 - 0.25 * hi) * (0.25 * wj)
                        + bl * (0.25 * hi) * (1.0 - 0.25 * wj) + br * (0.25 * hi) * (0.25 * wj))
    hr = torch.stack(outs, dim=3).reshape(n, h, w, 4, 4, c).permute(0, 1, 3, 2, 4, 5)
    return hr.reshape(n, h * 4, w * 4, c)


_BICUBIC_R = 0.75
_BICUBIC_MAT = np.float32([[0, 1, 0, 0], [-_BICUBIC_R, 0, _BICUBIC_R, 0],
                           [2 * _BICUBIC_R, _BICUBIC_R - 3, 3 - 2 * _BICUBIC_R, -_BICUBIC_R],
                           [-_BICUBIC_R, 2 - _BICUBIC_R, _BICUBIC_R - 2, _BICUBIC_R]])
BICUBIC_WEIGHTS = [np.float32([1.0, t, t * t, t * t * t]).dot(_BICUBIC_MAT) for t in [0.0, 0.25, 0.5, 0.75]]


def bicubic_four(x):
    """lib/ops.py:166-212: x4 Keys bicubic (A=-0.75), legacy coordinates, edge replicate,
    rows first then columns."""
    n, h, w, c = x.shape
    p = torch.cat((x[:, :1], x), dim=1)
    p = torch.cat((p[:, :, :1], p), dim=2)
    p = torch.cat((p, p[:, -1:], p[:, -1:]), dim=1)
    p = torch.cat((p, p[:, :, -1:], p[:, :, -1:]), dim=2)
    bins = [p[:, bi:bi + h] for bi in range(4)]
    rows = []
    for hi in range(4):
        cw = BICUBIC_WEIGHTS[hi]
        rows.append(float(cw[0]) * bins[0] + float(cw[1]) * bins[1] + float(cw[2]) * bins[2] + float(cw[3]) * bins[3])
    hy = torch.stack(rows, dim=2).reshape(n, h * 4, w + 3, c)
    bins = [hy[:, :, bj:bj + w] for bj in range(4)]
    cols = []
    for hj in range(4):
        cw = BICUBIC_WEIGHTS[hj]
        cols.append(float(cw[0]) * bins[0] + float(cw[1]) * bins[1] + float(cw[2]) * bins[2] + float(cw[3]) * bins[3])
    return torch.stack(cols, dim=3).reshape(n, h * 4, w * 4, c)


def space_to_depth4(x):
    """tf.space_to_depth(x,4) (main.py:201) == reshape/transpose of lib/Teco.py:145-148:
    [B,4h,4w,3] -> [B,h,w,48], channel = (dy*4+dx)*3+c."""
    n, H, W, c = x.shape
    h, w = H // 4, W // 4
    return x.reshape(n, h, 4, w, 4, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h, w, 16 * c)


def gaussian_2dkernel(size=9, sig=1.5):
    """lib/ops.py:339-345 (scipy.signal.gaussian == exp(-x^2/2sig^2), unnormalised 1-D)."""
    ax = np.arange(size, dtype=np.float64) - (size - 1) / 2.0
    g = np.exp(-0.5 * (ax / sig) ** 2).reshape(size, 1)
    k = np.outer(g, g)
    return k / k.sum()


def gauss_down_by4(hr, sigma=1.5):
    """tf_data_gaussDownby4, lib/ops.py:347-367: 9x9 Gaussian, stride 4, VALID, per channel."""
    kw = 1 + 2 * int(sigma * 3.0)
    k = torch.tensor(np.float32(gaussian_2dkernel(kw, sigma)), dtype=hr.dtype)
    wt = torch.zeros(3, 3, kw, kw, dtype=hr.dtype)
    for c in range(3):
        wt[c, c] = k
    y = F.conv2d(hr.permute(0, 3, 1, 2), wt, stride=4)
    return y.permute(0, 2, 3, 1).contiguous()


# --------------------------------------------------------------------------------------
# parameters (TF variable names, SURVEY Appendix C)
# --------------------------------------------------------------------------------------
def _xavier(gen, shape, fan_in, fan_out, dtype):
    lim = math.sqrt(6.0 / (fan_in + fan_out))  # tf.contrib.layers.xavier_initializer (uniform)
    return ((torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1) * lim).to(dtype)


def _add_conv(p, gen, name, k, cin, cout, bias=True, transpose=False, bias_std=0.0, dtype=torch.float32):
    if transpose:   # [kh,kw,Cout,Cin]; slim fan_in/out computed from the stored shape
        p[name + "/weights"] = _xavier(gen, (k, k, cout, cin), k * k * cout, k * k * cin, dtype)
    else:
        p[name + "/weights"] = _xavier(gen, (k, k, cin, cout), k * k * cin, k * k * cout, dtype)
    if bias:
        b = torch.zeros(cout, dtype=dtype)
        if bias_std > 0:
            b = (torch.randn(cout, generator=gen, dtype=torch.float64) * bias_std).to(dtype)
        p[name + "/biases"] = b


def init_generator(seed=1234, num_resblock=16, bias_std=0.0, dtype=torch.float32):
    """Variables of generator_F (lib/frvsr.py:44-88) under scope 'generator' (main.py:203)."""
    gen = torch.Generator().manual_seed(seed)
    p = OrderedDict()
    g = "generator/generator_unit/"
    _add_conv(p, gen, g + "input_stage/conv/Conv", 3, 51, 64, bias_std=bias_std, dtype=dtype)
    for i in range(1, num_resblock + 1):
        _add_conv(p, gen, g + "resblock_%d/conv_1/Conv" % i, 3, 64, 64, bias_std=bias_std, dtype=dtype)
        _add_conv(p, gen, g + "resblock_%d/conv_2/Conv" % i, 3, 64, 64, bias_std=bias_std, dtype=dtype)
    for i in (1, 2):
        _add_conv(p, gen, g + "conv_tran2highres/conv_tran%d/Conv2d_transpose" % i, 3, 64, 64,
                  transpose=True, bias_std=bias_std, dtype=dtype)
    _add_conv(p, gen, g + "output_stage/conv/Conv", 3, 64, 3, bias_std=bias_std, dtype=dtype)
    return p


def damp_generator(p, gain=0.5):
    """Scale the residual-block and output-stage weights of a xavier-initialised generator.
    Why: with untrained xavier weights the RECURRENCE (output -> warp -> input) is expanding -- on the calendar
    32x32 clip the output std grows x1.5 per frame (0.4 -> 115 after 15 frames) and a 1e-6 input perturbation
    grows to 2e-2, so no two fp32 implementations can agree.  gain 0.5 gives a contractive, trained-like
    operating point (output std stays ~0.33, perturbations shrink) where parity over many frames is meaningful."""
    q = OrderedDict()
    for k, v in p.items():
        hit = k.endswith("/weights") and k.startswith("generator/") and ("/resblock_" in k or "/output_stage/" in k)
        q[k] = v * gain if hit else v
    return q


FNET_LAYERS = [("encoder_1", 6, 32), ("encoder_2", 32, 64), ("encoder_3", 64, 128),
               ("decoder_1", 128, 256), ("decoder_2", 256, 128), ("decoder_3", 128, 64)]


def init_fnet(seed=4321, bias_std=0.0, dtype=torch.float32):
    """Variables of fnet (lib/frvsr.py:4-41) under scope 'fnet' (main.py:210)."""
    gen = torch.Generator().manual_seed(seed)
    p = OrderedDict()
    f = "fnet/autoencode_unit/"
    for name, cin, cout in FNET_LAYERS:
        _add_conv(p, gen, f + name + "/conv_1/Conv", 3, cin, cout, bias_std=bias_std, dtype=dtype)
        _add_conv(p, gen, f + name + "/conv_2/Conv", 3, cout, cout, bias_std=bias_std, dtype=dtype)
    _add_conv(p, gen, f + "output_stage/conv1/Conv", 3, 64, 32, bias_std=bias_std, dtype=dtype)
    _add_conv(p, gen, f + "output_stage/conv2/Conv", 3, 32, 2, bias_std=bias_std, dtype=dtype)
    return p


DIS_BLOCKS = [("disblock_1", 64, 64), ("disblock_3", 64, 64), ("disblock_5", 64, 128), ("disblock_7", 128, 256)]


def init_discriminator(seed=777, cin=27, bias_std=0.0, dtype=torch.float32):
    """Variables of discriminator_F (lib/Teco.py:30-74) under 'tdiscriminator' (lib/Teco.py:226)."""
    gen = torch.Generator().manual_seed(seed)
    p = OrderedDict()
    d = "tdiscriminator/discriminator_unit/"
    _add_conv(p, gen, d + "input_stage/conv/Conv", 3, cin, 64, bias_std=bias_std, dtype=dtype)
    for name, ci, co in DIS_BLOCKS:
        _add_conv(p, gen, d + name + "/conv1/Conv", 4, ci, co, bias=False, dtype=dtype)
        beta = torch.zeros(co, dtype=dtype)
        if bias_std > 0:
            beta = (torch.randn(co, generator=gen, dtype=torch.float64) * bias_std).to(dtype)
        p[d + name + "/BatchNorm/beta"] = beta
    p[d + "dense_layer_2/dense/kernel"] = _xavier(gen, (256, 1), 256, 1, dtype)
    b = torch.zeros(1, dtype=dtype)
    if bias_std > 0:
        b = (torch.randn(1, generator=gen, dtype=torch.float64) * bias_std).to(dtype)
    p[d + "dense_layer_2/dense/bias"] = b
    return p


VGG_CFG = [(1, 2, 3, 64), (2, 2, 64, 128), (3, 4, 128, 256), (4, 4, 256, 512), (5, 4, 512, 512)]
VGG_TAPS = ["vgg_19/conv2/conv2_2", "vgg_19/conv3/conv3_4", "vgg_19/conv4/conv4_4", "vgg_19/conv5/conv5_4"]


def init_vgg19(seed=99, dtype=torch.float32):
    """slim vgg_19 conv trunk (lib/ops.py:319-328); random He-style weights stand in for
    vgg_19.ckpt (not on this box) -- frozen either way."""
    gen = torch.Generator().manual_seed(seed)
    p = OrderedDict()
    for blk, reps, cin, cout in VGG_CFG:
        c = cin
        for j in range(1, reps + 1):
            name = "vgg_19/conv%d/conv%d_%d" % (blk, blk, j)
            std = math.sqrt(2.0 / (9 * c))
            p[name + "/weights"] = (torch.randn((3, 3, c, cout), generator=gen, dtype=torch.float64) * std).to(dtype)
            p[name + "/biases"] = (torch.randn(cout, generator=gen, dtype=torch.float64) * 0.01).to(dtype)
            c = cout
    return p


# --------------------------------------------------------------------------------------
# networks
# --------------------------------------------------------------------------------------
def generator_F(p, gen_inputs, num_resblock=16):
    """lib/frvsr.py:44-88.  gen_inputs [B,h,w,51] -> [B,4h,4w,3] in ~[-1,1]."""
    g = "generator/generator_unit/"

    def cv(x, name):
        return conv2d(x, p[g + name + "/weights"], p[g + name + "/biases"])

    net = F.relu(cv(gen_inputs, "input_stage/conv/Conv"))
    for i in range(1, num_resblock + 1):
        r = F.relu(cv(net, "resblock_%d/conv_1/Conv" % i))
        net = cv(r, "resblock_%d/conv_2/Conv" % i) + net
    for i in (1, 2):
        n_ = g + "conv_tran2highres/conv_tran%d/Conv2d_transpose" % i
        net = F.relu(conv2d_transpose(net, p[n_ + "/weights"], p[n_ + "/biases"]))
    net = cv(net, "output_stage/conv/Conv")
    net = net + bicubic_four(gen_inputs[..., 0:3])
    return preprocess(net)


def fnet(p, fnet_input):
    """lib/frvsr.py:4-41.  [n,h,w,6] -> [n,8*(h//8),8*(w//8),2], tanh*24."""
    f = "fnet/autoencode_unit/"

    def cv(x, name):
        return conv2d(x, p[f + name + "/weights"], p[f + name + "/biases"])

    net = fnet_input
    for name in ("encoder_1", "encoder_2", "encoder_3"):
        net = lrelu(cv(net, name + "/conv_1/Conv"))
        net = lrelu(cv(net, name + "/conv_2/Conv"))
        net = maxpool(net)
    for name in ("decoder_1", "decoder_2", "decoder_3"):
        net = lrelu(cv(net, name + "/conv_1/Conv"))
        net = lrelu(cv(net, name + "/conv_2/Conv"))
        net = resize_bilinear_legacy(net, net.shape[1] * 2, net.shape[2] * 2)
    net = lrelu(cv(net, "output_stage/conv1/Conv"))
    net = cv(net, "output_stage/conv2/Conv")
    return torch.tanh(net) * 24.0


def discriminator_F(p, dis_inputs):
    """lib/Teco.py:30-74 -> (prob map [tb,h/16,w/16,1], [4 hidden layers])."""
    d = "tdiscriminator/discriminator_unit/"
    net = lrelu(conv2d(dis_inputs, p[d + "input_stage/conv/Conv/weights"], p[d + "input_stage/conv/Conv/biases"]))
    layers = []
    for name, _, _ in DIS_BLOCKS:
        net = conv2d(net, p[d + name + "/conv1/Conv/weights"], None, stride=2)
        net = lrelu(batchnorm_train(net, p[d + name + "/BatchNorm/beta"]))
        layers.append(net)
    net = net @ p[d + "dense_layer_2/dense/kernel"] + p[d + "dense_layer_2/dense/bias"]
    return torch.sigmoid(net), layers


def vgg19_features(p, x_pm1, norm_flag=True):
    """VGG19_slim (lib/Teco.py:5-24) + vgg_19 (lib/ops.py:287-334): returns the 4 tapped,
    channel-L2-normalised feature maps for an input in [-1,1]."""
    net = deprocess(x_pm1) * 255.0 - torch.tensor(VGG_MEAN, dtype=x_pm1.dtype)
    out = {}
    for blk, reps, _, _ in VGG_CFG:
        for j in range(1, reps + 1):
            name = "vgg_19/conv%d/conv%d_%d" % (blk, blk, j)
            net = F.relu(conv2d(net, p[name + "/weights"], p[name + "/biases"]))
            if name in VGG_TAPS:
                f = net
                if norm_flag:
                    f = f / torch.sqrt((f * f).sum(dim=3, keepdim=True) + 1e-12)
                out[name] = f
        if blk < 5:
            net = maxpool(net)
    return out


# --------------------------------------------------------------------------------------
# inference recurrence (main.py:185-216, 253-268)
# --------------------------------------------------------------------------------------
def pad_symmetric_br(x, oh, ow):
    """tf.pad(x, [[0,0],[0,oh],[0,ow],[0,0]], 'SYMMETRIC') -- edge-including mirror, main.py:212."""
    if oh:
        x = torch.cat((x, torch.flip(x[:, -oh:], dims=(1,))), dim=1)
    if ow:
        x = torch.cat((x, torch.flip(x[:, :, -ow:], dims=(2,))), dim=2)
    return x


def inference_sequence(pg, pf, frames, num_resblock=16, return_aux=False):
    """frames: list of [H,W,3] tensors in [0,1] (already including any warm-up frames).
    Returns list of [4H,4W,3] outputs in [0,1] (= deprocess(gen_output), main.py:207), one per
    input frame, following the ordering of main.py:253-260 / SURVEY A.9."""
    h, w = frames[0].shape[0], frames[0].shape[1]
    oh, ow = h - h // 8 * 8, w - w // 8 * 8
    dt = frames[0].dtype
    pre_inputs = torch.zeros(1, h, w, 3, dtype=dt)
    pre_gen = torch.zeros(1, 4 * h, 4 * w, 3, dtype=dt)
    pre_warp = torch.zeros(1, 4 * h, 4 * w, 3, dtype=dt)
    outs, aux = [], []
    for i, fr in enumerate(frames):
        cur = fr.unsqueeze(0)
        flow_lr = None
        if i != 0:
            flow_lr = fnet(pf, torch.cat((pre_inputs, cur), dim=-1))
            flow_lr = pad_symmetric_br(flow_lr, oh, ow)
            flow = upscale_four(flow_lr * 4.0)
            pre_warp = dense_image_warp(pre_gen, flow)
        inputs_all = torch.cat((cur, space_to_depth4(pre_warp)), dim=-1)
        gen_out = generator_F(pg, inputs_all, num_resblock)
        pre_inputs = cur
        pre_gen = deprocess(gen_out)
        outs.append(pre_gen[0])
        if return_aux:
            aux.append({"flow_lr": flow_lr, "pre_warp": pre_warp[0]})
    return (outs, aux) if return_aux else outs


def warmup_order(n):
    """lib/dataloader.py:42-44: prepend list indices 5,4,3,2,1 then 0..n-1."""
    return [5, 4, 3, 2, 1] + list(range(n))


def save_img_u8(img01):
    """lib/ops.py:521-523 without the BGR swap/imwrite: clip(255 x) -> uint8 (truncation)."""
    return np.clip(img01.detach().cpu().numpy() * 255.0, 0, 255).astype(np.uint8)


# --------------------------------------------------------------------------------------
# training graph (lib/Teco.py:77-517)
# --------------------------------------------------------------------------------------
class TrainFlags:
    """Config of record: runGan.py:142-234 (case 3) / 250-286 (case 4); defaults main.py:32-103."""

    def __init__(self, **kw):
        self.RNN_N = 10
        self.batch_size = 4
        self.crop_size = 32
        self.num_resblock = 16
        self.pingpang = True
        self.pp_scaling = 0.5
        self.vgg_scaling = 0.2
        self.warp_scaling = 1.0
        self.ratio = 0.01
        self.Dt_mergeDs = True
        self.Dt_ratio_0 = 1.0
        self.Dt_ratio_add = 0.0
        self.Dt_ratio_max = 1.0
        self.Dbalance = 0.4
        self.crop_dt = 0.75
        self.D_LAYERLOSS = True
        self.EPS = 1e-12
        self.learning_rate = 5e-5
        self.decay_step = 500000
        self.decay_rate = 1.0
        self.stair = True
        self.beta = 0.9
        self.adameps = 1e-8
        for k, v in kw.items():
            if not hasattr(self, k):
                raise ValueError("unknown flag " + k)
            setattr(self, k, v)

    @staticmethod
    def frvsr(**kw):  # runGan.py:250-286
        d = dict(num_resblock=10, ratio=-0.01, pingpang=False, vgg_scaling=-0.002, pp_scaling=1.0)
        d.update(kw)
        return TrainFlags(**d)


def tecogan_forward(params, r_inputs, r_targets, FLAGS, GAN_Flag=True, global_step=0):
    """Forward graph + losses of TecoGAN() (lib/Teco.py:77-413).  Returns a dict with
    gen_outputs, the scalar losses in reference order (update_list / update_list_name),
    gen_loss, fnet_loss, discrim_loss, t_balance."""
    B, crop = FLAGS.batch_size, FLAGS.crop_size
    T = FLAGS.RNN_N
    if FLAGS.pingpang:  # lib/Teco.py:80-85
        r_inputs = torch.cat((r_inputs, torch.flip(r_inputs[:, :-1], dims=(1,))), dim=1)
        r_targets = torch.cat((r_targets, torch.flip(r_targets[:, :-1], dims=(1,))), dim=1)
        T = FLAGS.RNN_N * 2 - 1
    H = crop * 4
    # fnet on all consecutive pairs, lib/Teco.py:102-117
    pre, cur = r_inputs[:, :-1], r_inputs[:, 1:]
    fnet_input = torch.cat((pre, cur), dim=-1).reshape(B * (T - 1), crop, crop, 6)
    gen_flow_lr = fnet(params, fnet_input)
    gen_flow = upscale_four(gen_flow_lr * 4.0).reshape(B, T - 1, H, H, 2)
    input_frames = cur.reshape(B * (T - 1), crop, crop, 3)
    s_input_warp = dense_image_warp(pre.reshape(B * (T - 1), crop, crop, 3), gen_flow_lr)  # :120-122
    # recurrent generator, lib/Teco.py:125-164
    input0 = torch.cat((r_inputs[:, 0], torch.zeros(B, crop, crop, 48, dtype=r_inputs.dtype)), dim=-1)
    gen_pre = generator_F(params, input0, FLAGS.num_resblock)
    gen_outputs, gen_warppre = [gen_pre], []
    for t in range(T - 1):
        warped = dense_image_warp(gen_pre, gen_flow[:, t])
        gen_warppre.append(warped)
        inputs = torch.cat((r_inputs[:, t + 1], space_to_depth4(deprocess(warped))), dim=-1)
        gen_pre = generator_F(params, inputs, FLAGS.num_resblock)
        gen_outputs.append(gen_pre)
    gen_outputs = torch.stack(gen_outputs, dim=1)
    s_gen_output = gen_outputs.reshape(B * T, H, H, 3)
    s_targets = r_targets.reshape(B * T, H, H, 3)

    update_list, update_list_name = [], []
    res = {"gen_outputs": gen_outputs, "gen_flow_lr": gen_flow_lr, "gen_warppre": gen_warppre}

    if FLAGS.vgg_scaling > 0.0:  # :174-178
        gen_vgg = vgg19_features(params, s_gen_output)
        target_vgg = vgg19_features(params, s_targets)

    dt_ratio = min(FLAGS.Dt_ratio_max, FLAGS.Dt_ratio_0 + FLAGS.Dt_ratio_add * float(global_step))
    if GAN_Flag:  # :180-313
        t_size = 3 * (T // 3)
        t_gen_output = gen_outputs[:, :t_size].reshape(B * t_size, H, H, 3)
        t_targets = r_targets[:, :t_size].reshape(B * t_size, H, H, 3)
        t_batch = B * t_size // 3
        if not FLAGS.pingpang:  # :190-204
            fb = torch.cat((r_inputs[:, 2:t_size:3], r_inputs[:, 1:t_size:3]), dim=-1).reshape(t_batch, crop, crop, 6)
            flow_back = upscale_four(fnet(params, fb) * 4.0).reshape(B, t_size // 3, H, H, 2)
            v_pre = gen_flow[:, 0:t_size:3]
            v_nxt = flow_back
        else:  # :206-209
            v_pre = gen_flow[:, 0:t_size:3]
            idx = list(range(T - 1))[-2:-1 - t_size:-3]
            v_nxt = gen_flow[:, idx]
        v_mid = torch.zeros_like(v_pre)
        T_vel = torch.stack((v_pre, v_mid, v_nxt), dim=2).reshape(B * t_size, H, H, 2).detach()  # :211-214
        if FLAGS.crop_dt < 1.0:  # :216-220
            crop_size_dt = int(crop * 4 * FLAGS.crop_dt)
            offset_dt = (crop * 4 - crop_size_dt) // 2
            crop_size_dt = crop * 4 - offset_dt * 2

        def triplet9(x):  # [tb*3,h,w,3] -> [tb,h,w,9] RRRGGGBBB, :227-229
            hh, ww = x.shape[1], x.shape[2]
            return x.reshape(t_batch, 3, hh, ww, 3).permute(0, 2, 3, 4, 1).reshape(t_batch, hh, ww, 9)

        def dst_inputs(frames):  # :224-245 / :254-269
            warp = triplet9(dense_image_warp(frames, T_vel))
            if FLAGS.crop_dt < 1.0:
                mask = torch.zeros(1, H, H, 1, dtype=warp.dtype)
                mask[:, offset_dt:offset_dt + crop_size_dt, offset_dt:offset_dt + crop_size_dt] = 1.0
                warp = warp * mask  # crop_to_bounding_box then tf.pad CONSTANT zeros
            before = triplet9(frames)
            t_input = triplet9(r_inputs[:, :t_size].reshape(B * t_size, crop, crop, 3))
            input_hi = resize_bilinear_legacy(t_input, H, H)
            return torch.cat((before, warp, input_hi), dim=-1)

        assert FLAGS.Dt_mergeDs, "oracle restates the Dst (merged) configuration of record"
        real_in = dst_inputs(t_targets)
        fake_in = dst_inputs(t_gen_output)
        d_real, real_layers = discriminator_F(params, real_in)
        d_fake, fake_layers = discriminator_F(params, fake_in)
        res.update(real_in=real_in, fake_in=fake_in, d_real=d_real, d_fake=d_fake,
                   real_layers=real_layers, fake_layers=fake_layers)
        if FLAGS.D_LAYERLOSS:  # :275-313
            layer_norm = [12.0, 14.0, 24.0, 100.0]
            sum_layer_loss = 0
            lll = []
            for li in range(4):
                ll = (real_layers[li] - fake_layers[li]).abs().sum(dim=3).mean()
                lll.append(ll)
                sum_layer_loss = sum_layer_loss + 0.02 * ll / layer_norm[li]
            update_list += lll
            update_list_name += ["D_layer_%d_loss" % i for i in range(4)]
            update_list += [sum_layer_loss]
            update_list_name += ["D_layer_loss_sum"]

    # generator losses :316-390
    content_loss = ((s_gen_output - s_targets) ** 2).sum(dim=3).mean()
    update_list += [content_loss]
    update_list_name += ["l2_content_loss"]
    gen_loss = content_loss
    warp_loss = ((input_frames - s_input_warp) ** 2).sum(dim=3).mean()
    update_list += [warp_loss]
    update_list_name += ["l2_warp_loss"]
    if FLAGS.vgg_scaling > 0.0:
        vgg_loss = 0
        vl = []
        for name in VGG_TAPS:
            d_ = 1.0 - (gen_vgg[name] * target_vgg[name]).sum(dim=3).mean()
            vl.append(d_)
            vgg_loss = vgg_loss + d_
        gen_loss = gen_loss + FLAGS.vgg_scaling * vgg_loss
        update_list += vl + [vgg_loss]
        update_list_name += ["vgg_loss_%d" % (i + 2) for i in range(4)] + ["vgg_all"]
    if FLAGS.pingpang:
        first = gen_outputs[:, 0:FLAGS.RNN_N - 1]
        last_rev = torch.flip(gen_outputs[:, FLAGS.RNN_N:], dims=(1,))  # [-1:-RNN_N:-1]
        pploss = (first - last_rev).abs().mean()
        if FLAGS.pp_scaling > 0:
            gen_loss = gen_loss + pploss * FLAGS.pp_scaling
        update_list += [pploss]
        update_list_name += ["PingPang"]
    discrim_loss = None
    t_balance = None
    if GAN_Flag:
        t_adv = (-torch.log(d_fake + FLAGS.EPS)).mean()
        gen_loss = gen_loss + FLAGS.ratio * t_adv * dt_ratio
        update_list += [t_adv]
        update_list_name += ["t_adversarial_loss"]
        if FLAGS.D_LAYERLOSS:
            gen_loss = gen_loss + sum_layer_loss * dt_ratio
        fake_l = torch.log(1 - d_fake + FLAGS.EPS)
        real_l = torch.log(d_real + FLAGS.EPS)
        discrim_loss = (-(fake_l + real_l)).mean()
        t_balance = real_l.mean() + t_adv
        update_list += [discrim_loss, d_real.mean(), d_fake.mean()]
        update_list_name += ["t_discrim_loss", "t_discrim_real_output", "t_discrim_fake_output"]
    update_list += [gen_loss]
    update_list_name += ["All_loss_Gen"]
    fnet_loss = FLAGS.warp_scaling * warp_loss + gen_loss  # :443
    res.update(update_list=update_list, update_list_name=update_list_name, gen_loss=gen_loss,
               fnet_loss=fnet_loss, discrim_loss=discrim_loss, t_balance=t_balance,
               content_loss=content_loss, warp_loss=warp_loss, dt_ratio=dt_ratio)
    return res


class TFAdam:
    """tf.train.AdamOptimizer [TF-ext] SURVEY A.12: lr_t = lr sqrt(1-b2^t)/(1-b1^t);
    theta -= lr_t m / (sqrt(v) + eps)."""

    def __init__(self, names, params, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        self.names, self.lr, self.b1, self.b2, self.eps = list(names), lr, beta1, beta2, eps
        self.m = {n: torch.zeros_like(params[n]) for n in self.names}
        self.v = {n: torch.zeros_like(params[n]) for n in self.names}
        self.t = 0

    def apply(self, params, grads):
        self.t += 1
        lr_t = self.lr * math.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        for n in self.names:
            g = grads[n]
            self.m[n] = self.b1 * self.m[n] + (1 - self.b1) * g
            self.v[n] = self.b2 * self.v[n] + (1 - self.b2) * g * g
            params[n] = params[n] - lr_t * self.m[n] / (torch.sqrt(self.v[n]) + self.eps)


class Trainer:
    """One-process restatement of the train op (lib/Teco.py:415-517): three TF-Adams,
    t_balance EMA (decay .99, zero init, no debias), adaptive-D branch tb < Dbalance decided
    on the EMA *before* this step's update (the tf.cond predicate reads the variable before
    update_tb runs inside the branch), all gradients from one forward with pre-update weights."""

    def __init__(self, params, FLAGS, GAN_Flag=True):
        self.p = OrderedDict((k, v.clone()) for k, v in params.items())
        self.FLAGS, self.GAN = FLAGS, GAN_Flag
        self.g_names = [k for k in self.p if k.startswith("generator/")]
        self.f_names = [k for k in self.p if k.startswith("fnet/")]
        self.d_names = [k for k in self.p if k.startswith("tdiscriminator/")]
        lr = FLAGS.learning_rate
        self.opt_g = TFAdam(self.g_names, self.p, lr, FLAGS.beta, eps=FLAGS.adameps)
        self.opt_f = TFAdam(self.f_names, self.p, lr, FLAGS.beta, eps=FLAGS.adameps)
        self.opt_d = TFAdam(self.d_names, self.p, lr, FLAGS.beta, eps=FLAGS.adameps) if GAN_Flag else None
        self.tb_ema = 0.0
        self.loss_ema = None
        self.global_step = 0
        self.counter_withD = 0
        self.counter_woD = 0

    def step(self, r_inputs, r_targets):
        F_ = self.FLAGS
        leaf = OrderedDict()
        for k, v in self.p.items():
            leaf[k] = v.clone().requires_grad_(not k.startswith("vgg_19/"))
        res = tecogan_forward(leaf, r_inputs, r_targets, F_, self.GAN, self.global_step)
        gf = self.g_names + self.f_names
        # d(fnet_loss)/d(gen vars) == d(gen_loss)/d(gen vars): warp_loss has no generator path (:334)
        g_grads = torch.autograd.grad(res["fnet_loss"], [leaf[n] for n in gf], retain_graph=self.GAN)
        grads = dict(zip(gf, g_grads))
        with_d = False
        if self.GAN:
            d_grads = torch.autograd.grad(res["discrim_loss"], [leaf[n] for n in self.d_names])
            grads.update(dict(zip(self.d_names, d_grads)))
            with_d = self.tb_ema < F_.Dbalance
            self.tb_ema = 0.99 * self.tb_ema + 0.01 * float(res["t_balance"].detach())
            if with_d:
                self.opt_d.apply(self.p, grads)
                self.counter_withD += 1
            else:
                self.counter_woD += 1
        self.opt_g.apply(self.p, grads)
        self.opt_f.apply(self.p, grads)
        vals = [float(v.detach()) if torch.is_tensor(v) else float(v) for v in res["update_list"]]
        if self.loss_ema is None:
            self.loss_ema = [0.0] * len(vals)
        self.loss_ema = [0.99 * a + 0.01 * b for a, b in zip(self.loss_ema, vals)]
        self.global_step += 1
        res["grads"] = grads
        res["with_d"] = with_d
        return res


# --------------------------------------------------------------------------------------
# metrics restated (metrics.py:37-70 PSNR on Y of uint8 images; metrics.py:77-92,143-169 tOF)
# --------------------------------------------------------------------------------------
_YCBCR_T = np.array([[0.256788235294118, 0.504129411764706, 0.097905882352941],
                     [-0.148223529411765, -0.290992156862745, 0.439215686274510],
                     [0.439215686274510, -0.367788235294118, -0.071427450980392]])


def _y_of_u8(img_u8):
    """metrics.py:37-55 (_rgb2ycbcr, maxVal=255) channel 0 after to_uint8(x,0,255) (:57-61)."""
    x = np.clip(np.round(np.asarray(img_u8).astype("float32")), 0, 255)
    return x.reshape(-1, 3).dot(_YCBCR_T.T)[:, 0].reshape(x.shape[:2]) + 16.0


def psnr_y(img_true_u8, img_pred_u8):
    """metrics.py:63-70: 20 log10(255 / rmse(Y_true - Y_pred)) on uint8 RGB frames."""
    d = _y_of_u8(img_true_u8) - _y_of_u8(img_pred_u8)
    rmse = math.sqrt(max(float(np.mean(d * d)), 1e-20))
    return 20.0 * math.log10(255.0 / rmse)


def ssim_y(img_true_u8, img_pred_u8):
    """metrics.py:72-75: skimage.measure.compare_ssim(Y_true, Y_pred, data_range=Y_pred.max()-Y_pred.min()).
    skimage is a third-party dependency that is not installed here (the reference imports skimage.measure.compare_ssim,
    i.e. scikit-image <= 0.15); its published algorithm is restated: float64, 7x7 uniform window (scipy.ndimage.
    uniform_filter), sample covariance (cov_norm = 49/48), K1 = 0.01, K2 = 0.03, mean of the S map cropped by 3 pixels.
    Pinned in tests/test_oracle_golden.py against a second derivation by direct 49-term window sums."""
    from scipy.ndimage import uniform_filter
    X, Y = _y_of_u8(img_true_u8).astype(np.float64), _y_of_u8(img_pred_u8).astype(np.float64)
    if min(X.shape) < 7:
        raise ValueError("win_size exceeds image extent.")
    R = float(Y.max() - Y.min())
    NP = 49.0
    cov_norm = NP / (NP - 1.0)
    ux, uy = uniform_filter(X, size=7), uniform_filter(Y, size=7)
    uxx, uyy, uxy = uniform_filter(X * X, size=7), uniform_filter(Y * Y, size=7), uniform_filter(X * Y, size=7)
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = (0.01 * R) ** 2, (0.03 * R) ** 2
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
    return float(S[3:-3, 3:-3].mean())


def crop_8x8(img):
    """metrics.py:77-92."""
    oh, ow = img.shape[0], img.shape[1]
    h, w = (oh // 32) * 32, (ow // 32) * 32
    while h > oh - 16:
        h -= 32
    while w > ow - 16:
        w -= 32
    y, x = (oh - h) // 2, (ow - w) // 2
    return img[y:y + h, x:x + w]


def tof(pre_tar_u8, tar_u8, pre_out_u8, out_u8):
    """metrics.py:143-169: mean L2 norm of the difference of Farneback flows (cv2, CPU)."""
    import cv2
    g = [cv2.cvtColor(np.ascontiguousarray(a), cv2.COLOR_RGB2GRAY) for a in (pre_tar_u8, tar_u8, pre_out_u8, out_u8)]
    t_of = cv2.calcOpticalFlowFarneback(g[0], g[1], None, 0.5, 3, 15, 3, 5, 1.2, 0)
    o_of = cv2.calcOpticalFlowFarneback(g[2], g[3], None, 0.5, 3, 15, 3, 5, 1.2, 0)
    d = np.absolute(crop_8x8(t_of) - crop_8x8(o_of))
    return float(np.sqrt(np.sum(d * d, axis=-1)).mean())


def psnr(a, b, peak=1.0):
    """Plain PSNR between two float arrays (harness metric: CUDA output vs oracle output)."""
    d = np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)
    mse = float(np.mean(d * d))
    return 10.0 * math.log10(peak * peak / max(mse, 1e-20))
