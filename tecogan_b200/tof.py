"""tOF on the device -- the temporal optical-flow score of the reference's evaluation (metrics.py:143-169): the mean,
over the crop_8x8 window, of |flow(target[i-1], target[i]) - flow(result[i-1], result[i])|, with the flows of
cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0) on cv2's RGB2GRAY frames.  PyTorch only
carries the buffers; every stage is a kernel of tecogan_b200/csrc/farneback.cu:

  grey      teco_tof_grey_u8            (9798 R + 19235 G + 3735 B + 16384) >> 15, through a window
  level k   teco_farneback_pyramid_u8   Gaussian of the full frame, INTER_LINEAR to round(H / 2^k) x round(W / 2^k)
  expand    teco_farneback_polyexp_f32  5 polynomial coefficients per pixel, once per frame and level
  iterate   teco_farneback_iterate_f32  per-pixel field, 15x15 box mean (float64), regularised 2x2 solve; 3 per level
  up        teco_farneback_flow_up_f32  INTER_LINEAR to the next level, x 2
  tOF       teco_tof_reduce_f32         crop window, per-pixel norm, float64 mean without atomics

The flow of a frame pair is computed on the whole frame and cropped afterwards, as the reference does: the pyramid sees
the borders, so the flow of a crop would differ inside as well.  Only the reference's parameters exist.  DESIGN.md 4.4
lists what was established about cv2's algorithm and how closely this follows it.
"""
import ctypes as C

import torch

from ._ffi import call, ptr, stream_ptr
from .metrics import crop_window

u8, f32, f64 = torch.uint8, torch.float32, torch.float64

LEVELS = 3                       # levels above the full-resolution one (pyr_scale 0.5)
MIN_SIZE = 32                    # a level whose width or height would fall below this is dropped
ITERATIONS = 3
MAX_PAIRS = 256                  # pairs per teco_farneback_iterate_f32 launch
RED_CHUNKS = 32                  # partial sums per pair of teco_tof_reduce_f32
MAX_BATCH = 65535                # frames per polyexp launch / pairs per reduction launch (grid z / y)


def pyramid_sizes(h, w):
    """[(h_k, w_k)] for k = 0 .. the coarsest level kept: level k is round-half-to-even(h / 2^k) x (w / 2^k), and a
    level is kept while both scaled sides stay >= 32."""
    sizes, scale = [(h, w)], 1.0
    for _ in range(LEVELS):
        scale *= 0.5
        if w * scale < MIN_SIZE or h * scale < MIN_SIZE:
            break
        sizes.append((int(round(h * scale)), int(round(w * scale))))
    return sizes


def _check_grey(t, name):
    if not torch.is_tensor(t) or t.dtype != u8 or not t.is_cuda:
        raise ValueError("%s must be a uint8 CUDA tensor (grey frames)" % name)
    if t.dim() == 2:
        t = t[None]
    if t.dim() != 3:
        raise ValueError("%s must be [H,W] or [P,H,W], got %s" % (name, tuple(t.shape)))
    if t.shape[1] < 2 or t.shape[2] < 2:
        raise ValueError("%s: Farneback flow needs frames of at least 2x2 pixels, got %dx%d" % (name, t.shape[1], t.shape[2]))
    return t.contiguous()


def grey(frames_u8, window=None):
    """cv2.cvtColor(RGB2GRAY) of uint8 RGB CUDA frames [N,H,W,3] (or [H,W,3]) read through `window` (y0, x0, h, w;
    None: the whole frame) -> uint8 [N,h,w]."""
    if not torch.is_tensor(frames_u8) or frames_u8.dtype != u8 or not frames_u8.is_cuda:
        raise ValueError("frames_u8 must be a uint8 CUDA tensor (decoded RGB frames)")
    t = frames_u8[None] if frames_u8.dim() == 3 else frames_u8
    if t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError("frames_u8 must be [H,W,3] or [N,H,W,3], got %s" % (tuple(frames_u8.shape),))
    t = t.contiguous()
    N, H, W, _ = t.shape
    y0, x0, h, w = (0, 0, H, W) if window is None else (int(v) for v in window)
    out = torch.empty((N, h, w), device=t.device, dtype=u8)
    call("teco_tof_grey_u8", ptr(t, u8), N, H, W, y0, x0, h, w, ptr(out, u8), stream_ptr())
    return out


def pyramid_level(grey_u8, level):
    """Level `level` of grey frames [N,H,W] -> fp32 [N,h_k,w_k] (the stage alone, for tests and tools)."""
    g = _check_grey(grey_u8, "grey_u8")
    N, H, W = g.shape
    lh, lw = (int(round(H * 0.5 ** level)), int(round(W * 0.5 ** level)))
    out = torch.empty((N, lh, lw), device=g.device, dtype=f32)
    call("teco_farneback_pyramid_u8", ptr(g, u8), N, H, W, int(level), lh, lw, ptr(out, f32), stream_ptr())
    return out


def poly_exp(img_f32):
    """Polynomial expansion of fp32 images [N,h,w] -> [N,h,w,5] (coefficients of y, x, yy, xx, xy)."""
    img = img_f32[None] if img_f32.dim() == 2 else img_f32
    img = img.contiguous()
    N, h, w = img.shape
    R = torch.empty((N, h, w, 5), device=img.device, dtype=f32)
    for s in range(0, N, MAX_BATCH):
        n = min(MAX_BATCH, N - s)
        call("teco_farneback_polyexp_f32", ptr(img[s:s + n], f32), n, h, w, ptr(R[s:s + n], f32), stream_ptr())
    return R


def iterate(R, pairs, flow_in, flow_out):
    """One update iteration of the frame pairs `pairs` [(i0, i1)] of the expansions R [Nf,h,w,5]: flow_in [P,h,w,2]
    (None: zero) -> flow_out [P,h,w,2]."""
    Nf, h, w, _ = R.shape
    st = stream_ptr()
    for s in range(0, len(pairs), MAX_PAIRS):
        chunk = pairs[s:s + MAX_PAIRS]
        ia = (C.c_int32 * len(chunk))(*[a for a, _ in chunk])
        ib = (C.c_int32 * len(chunk))(*[b for _, b in chunk])
        fin = None if flow_in is None else flow_in[s:s + len(chunk)]
        call("teco_farneback_iterate_f32", ptr(R, f32), Nf, h, w, C.cast(ia, C.c_void_p), C.cast(ib, C.c_void_p),
             len(chunk), ptr(fin, f32), ptr(flow_out[s:s + len(chunk)], f32), st)
    return flow_out


def flow_up(flow, h, w):
    """Flow of the coarser level [P,sh,sw,2] -> [P,h,w,2]: INTER_LINEAR, x 1 / pyr_scale."""
    flow = flow.contiguous()
    P, sh, sw, _ = flow.shape
    out = torch.empty((P, h, w, 2), device=flow.device, dtype=f32)
    call("teco_farneback_flow_up_f32", ptr(flow, f32), P, sh, sw, ptr(out, f32), h, w, stream_ptr())
    return out


def flows(grey_u8, pairs):
    """Farneback flows [P,H,W,2] fp32 of the frame pairs `pairs` [(i0, i1)] of grey frames [Nf,H,W]: each frame is
    expanded once per level, whatever number of pairs it takes part in."""
    g = _check_grey(grey_u8, "grey_u8")
    Nf, H, W = g.shape
    pairs = [(int(a), int(b)) for a, b in pairs]
    if not pairs:
        raise ValueError("flows: no frame pairs")
    for a, b in pairs:
        if not (0 <= a < Nf and 0 <= b < Nf):
            raise ValueError("flows: pair (%d, %d) outside %d frames" % (a, b, Nf))
    sizes, flow = pyramid_sizes(H, W), None
    for k in range(len(sizes) - 1, -1, -1):
        lh, lw = sizes[k]
        img = torch.empty((Nf, lh, lw), device=g.device, dtype=f32)
        call("teco_farneback_pyramid_u8", ptr(g, u8), Nf, H, W, k, lh, lw, ptr(img, f32), stream_ptr())
        R = poly_exp(img)
        a = torch.empty((len(pairs), lh, lw, 2), device=g.device, dtype=f32)
        b = torch.empty_like(a) if flow is None else flow_up(flow, lh, lw)
        cur = None if flow is None else b                  # the coarsest level starts from the zero flow
        for it in range(ITERATIONS):                       # ping-pong: b -> a -> b -> a
            cur = iterate(R, pairs, cur, a if it % 2 == 0 else b)
        flow = cur
    return flow


def farneback(prev_u8, next_u8):
    """cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0) of P pairs at once: uint8 CUDA grey
    frames [P,H,W] (or [H,W]) -> fp32 [P,H,W,2] (x, y displacement)."""
    a, b = _check_grey(prev_u8, "prev_u8"), _check_grey(next_u8, "next_u8")
    if a.shape != b.shape:
        raise ValueError("farneback: prev %s and next %s differ in shape" % (tuple(a.shape), tuple(b.shape)))
    P = a.shape[0]
    return flows(torch.cat([a, b]), [(p, P + p) for p in range(P)])


def tof_of_flows(flow_t, flow_o, window):
    """tOF of flow pairs [P,H,W,2] over `window` (y0, x0, h, w): list of P floats."""
    flow_t, flow_o = flow_t.contiguous(), flow_o.contiguous()
    P, H, W, _ = flow_t.shape
    y0, x0, h, w = (int(v) for v in window)
    out = torch.empty(P, device=flow_t.device, dtype=f64)
    part = torch.empty((P, RED_CHUNKS), device=flow_t.device, dtype=f64)
    for s in range(0, P, MAX_BATCH):
        n = min(MAX_BATCH, P - s)
        call("teco_tof_reduce_f32", ptr(flow_t[s:s + n], f32), ptr(flow_o[s:s + n], f32), n, H, W, y0, x0, h, w,
             ptr(part[s:s + n], f64), ptr(out[s:s + n], f64), stream_ptr())
    return [float(v) for v in out.cpu()]


def tof_sequence(targets, results, window=None):
    """tOF list of consecutive frames (metrics.py:143-169): entry k-1 is the tOF of frame k against frame k-1, for
    k = 1 .. N-1, so the list is one shorter than the frames.  targets / results: uint8 RGB CUDA frames [N,H,W,3].
    Both are read through `window` (y0, x0, h, w) -- by default the common top-left area, which is the reference's cut
    of a larger result to the target; a result smaller than the target (where the reference fails) is compared on the
    area the two share.  The flows of the whole window are cropped with crop_8x8 before the norm.  All 2(N-1) flows run
    as one batch."""
    t, p = targets, results
    for name, v in (("targets", t), ("results", p)):
        if not torch.is_tensor(v) or v.dtype != u8 or v.dim() != 4 or v.shape[-1] != 3:
            raise ValueError("%s must be a uint8 tensor [N,H,W,3]" % name)
    if t.shape[0] != p.shape[0]:
        raise ValueError("tof_sequence: %d target frames but %d result frames" % (t.shape[0], p.shape[0]))
    N = t.shape[0]
    if window is None:
        window = (0, 0, min(t.shape[1], p.shape[1]), min(t.shape[2], p.shape[2]))
    cy, cx, ch, cw = crop_window(int(window[2]), int(window[3]))
    if ch <= 0 or cw <= 0:
        raise ValueError("crop_8x8 leaves nothing of %dx%d flows" % (int(window[2]), int(window[3])))
    if N < 2:
        return []
    g = torch.cat([grey(t, window), grey(p, window)])
    pairs = [(k - 1, k) for k in range(1, N)] + [(N + k - 1, N + k) for k in range(1, N)]
    f = flows(g, pairs)
    return tof_of_flows(f[:N - 1], f[N - 1:], (cy, cx, ch, cw))
