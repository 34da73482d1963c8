"""LPIPS (AlexNet, v0.1) and tLP100 on the device -- the perceptual and temporal-perceptual scores of the reference's
evaluation (metrics.py:183-202, LPIPSmodels/).  Frames are uint8 RGB CUDA tensors, exactly what tecogan_b200/metrics.py
takes; PyTorch only carries the buffers.

  input    teco_lpips_input_u8    float32(u8 / 127.5 - 1) (float64 arithmetic), then (x - shift) / scale in fp32, bit for bit
  relu1    teco_conv2d_f32        11x11 / 4, pad 2, 3 -> 64, ReLU
  relu2    teco_maxpool3s2_f32 +  5x5, pad 2, 64 -> 192, ReLU
  relu3    teco_maxpool3s2_f32 +  3x3, pad 1, 192 -> 384, ReLU
  relu4/5  teco_conv2d_f32        3x3, pad 1, 384 -> 256 -> 256, ReLU
  head     teco_lpips_head_f32    sum_l mean_pixels sum_c w_l[c] (f0/|f0| - f1/|f1|)^2, float64 accumulation

Everything is fp32 on the CUDA cores: tLP100 is 100 x the difference of two small distances, so bf16 / TF32 features would
show in its printed digits.  Each frame goes through AlexNet once; the distances between any two frames whose features
are kept (a frame and its result, a frame and its predecessor) come from the head alone.

Weights: torchvision's ImageNet AlexNet state dict (the file the reference downloads on its first metrics run, e.g.
alexnet-owt-*.pth under torch.hub.get_dir()/checkpoints) and LPIPSmodels/v0.1/alex.pth.  Parity with the reference is
pinned with seeded backbone weights and the real v0.1 linear weights (tests/golden/lpips.npz); parity with the real
ImageNet backbone is UNPINNED, because no copy of that file was available to check against.
"""
import ctypes as C
import os

import numpy as np
import torch

from ._ffi import ACT_RELU, call, ptr, stream_ptr
from .kernels import conv2d_raw

u8, f32, f64 = torch.uint8, torch.float32, torch.float64

# (state-dict prefix, Cin, Cout, kernel, stride, pad) of torchvision alexnet().features[0, 3, 6, 8, 10]
ALEXNET_CONVS = [("features.0", 3, 64, 11, 4, 2), ("features.3", 64, 192, 5, 1, 2), ("features.6", 192, 384, 3, 1, 1),
                 ("features.8", 384, 256, 3, 1, 1), ("features.10", 256, 256, 3, 1, 1)]
LIN_CHANNELS = (64, 192, 384, 256, 256)
MIN_SIZE = 31                    # smallest crop for which the second 3x3 / 2 pool has an output (torch raises below)
MAX_PAIRS = 256                  # pairs per teco_lpips_head_f32 launch


def _state_dict(path_or_dict):
    if isinstance(path_or_dict, (str, os.PathLike)):
        return torch.load(path_or_dict, map_location="cpu", weights_only=True)
    if not hasattr(path_or_dict, "keys"):
        raise ValueError("expected a state dict or the path of a torch.save'd one, got %s" % type(path_or_dict).__name__)
    return path_or_dict


def _tensor(sd, key, shape):
    if key not in sd:
        raise ValueError("state dict has no %r" % key)
    t = sd[key]
    t = t.detach() if torch.is_tensor(t) else torch.from_numpy(np.asarray(t))
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s has shape %s, expected %s" % (key, tuple(t.shape), tuple(shape)))
    return t.to(device="cpu", dtype=f32).contiguous()


def tf_layout(w):
    """torch conv weight [Cout,Cin,kh,kw] -> [kh,kw,Cin,Cout], the layout teco_conv2d_f32 reads."""
    return w.permute(2, 3, 1, 0).contiguous()


def load_alexnet(path_or_dict):
    """features.{0,3,6,8,10}.{weight,bias} of a torchvision AlexNet state dict (classifier.* is ignored) ->
    five (weight [kh,kw,Cin,Cout], bias [Cout]) pairs of CPU fp32 tensors.  A missing key or a wrong shape raises ValueError."""
    sd = _state_dict(path_or_dict)
    return [(tf_layout(_tensor(sd, name + ".weight", (cout, cin, k, k))), _tensor(sd, name + ".bias", (cout,)))
            for name, cin, cout, k, _, _ in ALEXNET_CONVS]


def load_lin(path_or_dict):
    """lin{0..4}.model.1.weight of LPIPS v0.1 (LPIPSmodels/v0.1/alex.pth, each [1,C,1,1]) -> five CPU fp32 [C] tensors."""
    sd = _state_dict(path_or_dict)
    return [_tensor(sd, "lin%d.model.1.weight" % l, (1, c, 1, 1)).reshape(c) for l, c in enumerate(LIN_CHANNELS)]


def feature_sizes(h, w):
    """(H, W) of relu1 .. relu5 for an h x w input; ValueError below MIN_SIZE, where torch's second pool raises."""
    if h < MIN_SIZE or w < MIN_SIZE:
        raise ValueError("LPIPS-AlexNet needs a crop of at least %dx%d pixels, got %dx%d" % (MIN_SIZE, MIN_SIZE, h, w))
    c1 = ((h + 4 - 11) // 4 + 1, (w + 4 - 11) // 4 + 1)
    p1 = ((c1[0] - 3) // 2 + 1, (c1[1] - 3) // 2 + 1)
    p2 = ((p1[0] - 3) // 2 + 1, (p1[1] - 3) // 2 + 1)
    return [c1, p1, p2, p2, p2]


def _frames(t, name):
    if not torch.is_tensor(t) or t.dtype != u8:
        raise ValueError("%s must be a uint8 tensor (decoded RGB frames)" % name)
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor: LPIPS has no CPU path" % name)
    if t.dim() == 3:
        t = t[None]
    if t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError("%s must be [H,W,3] or [N,H,W,3], got %s" % (name, tuple(t.shape)))
    return t.contiguous()


class LPIPS:
    """LPIPS-AlexNet v0.1 on the current CUDA device.  `alexnet` / `lin`: what load_alexnet / load_lin return, or anything
    they accept (a state dict or its path)."""

    def __init__(self, alexnet, lin):
        if not torch.cuda.is_available():
            raise ValueError("LPIPS needs a CUDA device: there is no CPU path")
        self.device = torch.device("cuda", torch.cuda.current_device())
        convs = alexnet if isinstance(alexnet, (list, tuple)) else load_alexnet(alexnet)
        lins = lin if isinstance(lin, (list, tuple)) else load_lin(lin)
        if len(convs) != 5 or len(lins) != 5:
            raise ValueError("LPIPS needs five AlexNet convolutions and five linear weights")
        self.convs = [(w.to(self.device, f32).contiguous(), b.to(self.device, f32).contiguous()) for w, b in convs]
        self.lin = [v.to(self.device, f32).contiguous() for v in lins]
        self._bufs = {}

    def _buffers(self, N, h, w):
        """Network input and the two pool outputs, kept per (N, h, w); the five feature maps are allocated per call so
        that callers may keep them."""
        key = (N, h, w)
        if key not in self._bufs:
            sz = feature_sizes(h, w)
            e = lambda *s: torch.empty(s, device=self.device, dtype=f32)   # noqa: E731
            self._bufs = {key: (e(N, h, w, 3), e(N, sz[1][0], sz[1][1], 64), e(N, sz[2][0], sz[2][1], 192))}
        return self._bufs[key]

    def features(self, frames_u8, window=None):
        """relu1 .. relu5 (fp32 NHWC) of every frame, all in one batched pass.  `frames_u8`: a uint8 CUDA tensor [N,H,W,3]
        (or [H,W,3]) or a list of them, whose frames are stacked in order; they may differ in size as long as the window
        (y0, x0, h, w) fits all of them.  window=None: the whole frame (all frames the same size)."""
        srcs = [_frames(f, "frames_u8") for f in (frames_u8 if isinstance(frames_u8, (list, tuple)) else [frames_u8])]
        if not srcs:
            raise ValueError("features: no frames")
        if window is None:
            if len({tuple(s.shape[1:3]) for s in srcs}) != 1:
                raise ValueError("features: frames of different sizes need a window")
            window = (0, 0, srcs[0].shape[1], srcs[0].shape[2])
        y0, x0, h, w = (int(v) for v in window)
        for s in srcs:
            if s.device != self.device:
                raise ValueError("features: frames on %s, model on %s" % (s.device, self.device))
            if y0 < 0 or x0 < 0 or y0 + h > s.shape[1] or x0 + w > s.shape[2]:
                raise ValueError("features: window %s does not fit %dx%d frames" % ((y0, x0, h, w), s.shape[1], s.shape[2]))
        sz = feature_sizes(h, w)
        N = sum(s.shape[0] for s in srcs)
        x, pool1, pool2 = self._buffers(N, h, w)
        n0, st = 0, stream_ptr()
        for s in srcs:
            n = s.shape[0]
            call("teco_lpips_input_u8", ptr(s, u8), n, s.shape[1], s.shape[2], y0, x0, h, w, ptr(x[n0:n0 + n], f32), st)
            n0 += n
        feats, inp = [], x
        for l, ((wt, b), (_, _, cout, _, stride, pad)) in enumerate(zip(self.convs, ALEXNET_CONVS)):
            if l in (1, 2):
                pooled = pool1 if l == 1 else pool2
                _, H, W, Cc = inp.shape
                call("teco_maxpool3s2_f32", ptr(inp, f32), ptr(pooled, f32), N, H, W, Cc, st)
                inp = pooled
            y = torch.empty((N, sz[l][0], sz[l][1], cout), device=self.device, dtype=f32)
            conv2d_raw(inp, wt, b, y, stride=stride, pad_t=pad, pad_l=pad, OH=sz[l][0], OW=sz[l][1], act=ACT_RELU)
            feats.append(y)
            inp = y
        return feats

    def distances(self, feats_a, feats_b, pairs, per_layer=False):
        """LPIPS of each pair (i, j) = (frame i of feats_a, frame j of feats_b), as a list of floats (and, with per_layer,
        the list of the five d_l of each pair).  One head launch per layer and 256 pairs; one device sync."""
        if len(feats_a) != 5 or len(feats_b) != 5:
            raise ValueError("distances: expected the five feature maps of LPIPS.features")
        for a, b in zip(feats_a, feats_b):
            if a.shape[1:] != b.shape[1:]:
                raise ValueError("distances: feature maps %s and %s differ (frames of different crop sizes)"
                                 % (tuple(a.shape), tuple(b.shape)))
        Na, Nb = feats_a[0].shape[0], feats_b[0].shape[0]
        pairs = [(int(i), int(j)) for i, j in pairs]
        if not pairs:
            return ([], []) if per_layer else []
        for i, j in pairs:
            if not (0 <= i < Na and 0 <= j < Nb):
                raise ValueError("distances: pair (%d, %d) outside %d x %d frames" % (i, j, Na, Nb))
        P = len(pairs)
        out = torch.zeros((5, P), device=self.device, dtype=f64)
        st = stream_ptr()
        for s in range(0, P, MAX_PAIRS):
            chunk = pairs[s:s + MAX_PAIRS]
            ia = (C.c_int32 * len(chunk))(*[i for i, _ in chunk])
            ib = (C.c_int32 * len(chunk))(*[j for _, j in chunk])
            for l in range(5):
                a, b = feats_a[l], feats_b[l]
                _, H, W, Cc = a.shape
                call("teco_lpips_head_f32", ptr(a, f32), Na, ptr(b, f32), Nb, C.cast(ia, C.c_void_p), C.cast(ib, C.c_void_p),
                     len(chunk), H, W, Cc, ptr(self.lin[l], f32), ptr(out[l, s:s + len(chunk)], f64), st)
        d = out.cpu().numpy()
        layers = [[float(d[l, p]) for l in range(5)] for p in range(P)]
        total = [(((v[0] + v[1]) + v[2]) + v[3]) + v[4] for v in layers]       # networks_basic.py:167-171 order
        return (total, layers) if per_layer else total

    def __call__(self, img_true, img_pred):
        """model.forward(im2tensor(img_true), im2tensor(img_pred))[0] of metrics.py:186-188 on already-cropped uint8
        frames [H,W,3]; a larger result is cut to the target (metrics.py:134-135)."""
        t, p = _frames(img_true, "img_true"), _frames(img_pred, "img_pred")
        if t.shape[0] != 1 or p.shape[0] != 1:
            raise ValueError("LPIPS(img_true, img_pred) takes one frame each; use features / distances for batches")
        f = self.features([t, p], (0, 0, min(t.shape[1], p.shape[1]), min(t.shape[2], p.shape[2])))
        return self.distances(f, f, [(0, 1)])[0]

    def sequence(self, targets, results, window, chunk=8):
        """LPIPS and tLP100 lists of consecutive frame pairs (metrics.py:183-202): LPIPS_k of (targets[k], results[k]) and,
        for k >= 1, tLP100_k = 100 |LPIPS(targets[k-1], targets[k]) - LPIPS(results[k-1], results[k])|, every frame
        through AlexNet once (`chunk` target / result pairs per batched pass)."""
        t, p = _frames(targets, "targets"), _frames(results, "results")
        if t.shape[0] != p.shape[0]:
            raise ValueError("sequence: %d target frames but %d result frames" % (t.shape[0], p.shape[0]))
        lp, tlp, prev = [], [], None
        for s in range(0, t.shape[0], chunk):
            k = min(chunk, t.shape[0] - s)
            f = self.features([t[s:s + k], p[s:s + k]], window)          # targets at 0..k-1, results at k..2k-1
            same = [(j, k + j) for j in range(k)]
            tt = [(j - 1, j) for j in range(1, k)]
            oo = [(k + j - 1, k + j) for j in range(1, k)]
            d = self.distances(f, f, same + tt + oo)
            lp += d[:k]
            dt, do = d[k:2 * k - 1], d[2 * k - 1:]
            if prev is not None:                                          # the first frame of this chunk and its predecessor
                pf, pk = prev
                dt0, do0 = self.distances(pf, f, [(pk - 1, 0), (2 * pk - 1, k)])
                dt, do = [dt0] + dt, [do0] + do
            tlp += [100.0 * abs(a - b) for a, b in zip(dt, do)]
            prev = (f, k)
        return lp, tlp
