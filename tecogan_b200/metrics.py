"""Evaluation metrics of the reference's `metrics.py` computed on the device (SURVEY.md 8f-3): PSNR and SSIM on the Y channel
of the uint8 result / target frames here, given an `lpips.LPIPS` model LPIPS and tLP100 (tecogan_b200/lpips.py), and with
tof=True the Farneback-flow tOF (tecogan_b200/tof.py).
Same function names and argument order as the reference (`psnr(img_true, img_pred)`, `ssim(img_true, img_pred)`,
`crop_8x8(img)`, metrics.py:63-92); frames are uint8 RGB CUDA tensors `[H,W,3]` (or `[N,H,W,3]` for the batched calls),
i.e. exactly what `main.py` inference writes through `save_img`.
"""
import math

import torch

from ._ffi import call, ptr, stream_ptr

u8, f64 = torch.uint8, torch.float64


def crop_window(ori_h, ori_w):
    """(y, x, h, w) of the reference's crop_8x8 (metrics.py:77-92): multiples of 32, at least 16 pixels smaller, centred."""
    h, w = (ori_h // 32) * 32, (ori_w // 32) * 32
    while h > ori_h - 16:
        h -= 32
    while w > ori_w - 16:
        w -= 32
    return (ori_h - h) // 2, (ori_w - w) // 2, h, w


def crop_8x8(img):
    """Reference signature: returns (crop_img, y, x).  `img` is any [H,W,...] tensor or array; the crop is a view."""
    y, x, h, w = crop_window(img.shape[0], img.shape[1])
    if h <= 0 or w <= 0:
        raise ValueError("crop_8x8: a %dx%d frame leaves nothing after the crop" % (img.shape[0], img.shape[1]))
    return img[y:y + h, x:x + w], y, x


def _as_batch(t, name):
    if not torch.is_tensor(t) or t.dtype != u8:
        raise ValueError("%s must be a uint8 tensor (decoded RGB frames)" % name)
    if t.dim() == 3:
        t = t[None]
    if t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError("%s must be [H,W,3] or [N,H,W,3], got %s" % (name, tuple(t.shape)))
    return t


def psnr_ssim_sums(img_true, img_pred, window=None, with_ssim=True):
    """Launches the two kernels and returns the raw accumulator [N,4] (float64, on device, no host sync) together with the
    window (y, x, h, w).  `window=None` means the whole common area of the two frames (the reference crops first with
    crop_8x8 and then calls psnr/ssim on the crops: pass `crop_window(...)` for that)."""
    t, p = _as_batch(img_true, "img_true"), _as_batch(img_pred, "img_pred")
    if t.shape[0] != p.shape[0]:
        raise ValueError("psnr/ssim: %d target frames but %d result frames" % (t.shape[0], p.shape[0]))
    N, tH, tW, _ = t.shape
    _, oH, oW, _ = p.shape
    if window is None:
        window = (0, 0, min(tH, oH), min(tW, oW))          # metrics.py:134-135: the result is cut to the target
    y0, x0, h, w = window
    acc = torch.empty((N, 4), device=t.device, dtype=f64)
    args = (ptr(t, u8), tH, tW, ptr(p, u8), oH, oW, N, y0, x0, h, w, ptr(acc, f64), stream_ptr())
    call("teco_metrics_psnr_y_u8", *args)
    if with_ssim:
        call("teco_metrics_ssim_y_u8", *args)
    return acc, window


def _finish(acc, window, with_ssim):
    _, _, h, w = window
    a = acc.cpu()
    ps, ss = [], []
    for n in range(a.shape[0]):
        mse = float(a[n, 0]) / (h * w)
        ps.append(20.0 * math.log10(255.0 / math.sqrt(mse)) if mse > 0.0 else float("inf"))   # numpy: 255/0 -> inf
        if with_ssim:
            ss.append(float(a[n, 3]) / ((h - 6) * (w - 6)))
    return ps, ss


def psnr(img_true, img_pred):
    """metrics.py:63-70 on one pair of uint8 RGB frames (already cropped, like the reference's call site :172)."""
    acc, win = psnr_ssim_sums(img_true, img_pred, with_ssim=False)
    return _finish(acc, win, False)[0][0]


def ssim(img_true, img_pred):
    """metrics.py:72-75 (skimage compare_ssim on Y, data_range = Y_pred.max() - Y_pred.min())."""
    acc, win = psnr_ssim_sums(img_true, img_pred)
    return _finish(acc, win, True)[1][0]


def frame_metrics(targets, results, crop=True):
    """PSNR and SSIM of N frame pairs in two launches: ([psnr_n], [ssim_n]).  crop=True applies crop_8x8 (as a window,
    without copying) exactly as the evaluation loop metrics.py:171-180 does before calling psnr/ssim."""
    t, p = _as_batch(targets, "targets"), _as_batch(results, "results")
    win = crop_window(min(t.shape[1], p.shape[1]), min(t.shape[2], p.shape[2])) if crop else None
    if crop and (win[2] <= 0 or win[3] <= 0):
        raise ValueError("crop_8x8 leaves nothing of %dx%d frames" % (t.shape[1], t.shape[2]))
    acc, win = psnr_ssim_sums(t, p, win)
    return _finish(acc, win, True)


def evaluate_sequence(targets, results, cutfr=2, lpips=None, tof=False):
    """The reference's per-folder loop (metrics.py:124-202): frames cutfr .. N-cutfr-1, crop_8x8, per-frame lists and
    their means (the 'FolderAvg' numbers).  PSNR and SSIM always; with `lpips` (an lpips.LPIPS model) also LPIPS and
    tLP100, and with tof=True also tOF; the temporal lists start at frame cutfr+1 and so are one shorter."""
    t, p = _as_batch(targets, "targets"), _as_batch(results, "results")
    n = t.shape[0]
    if n - 2 * cutfr <= 0:
        raise ValueError("evaluate_sequence: %d frames with cutfr=%d leave nothing to evaluate" % (n, cutfr))
    ps, ss = frame_metrics(t[cutfr:n - cutfr], p[cutfr:n - cutfr])
    r = {"PSNR": ps, "SSIM": ss, "FolderAvg_PSNR": sum(ps) / len(ps), "FolderAvg_SSIM": sum(ss) / len(ss)}
    if lpips is not None:
        win = crop_window(min(t.shape[1], p.shape[1]), min(t.shape[2], p.shape[2]))
        lp, tlp = lpips.sequence(t[cutfr:n - cutfr], p[cutfr:n - cutfr], win)
        r.update({"LPIPS": lp, "tLP100": tlp, "FolderAvg_LPIPS": sum(lp) / len(lp),
                  "FolderAvg_tLP100": sum(tlp) / len(tlp) if tlp else float("nan")})
    if tof:
        from .tof import tof_sequence
        of = tof_sequence(t[cutfr:n - cutfr], p[cutfr:n - cutfr])
        r.update({"tOF": of, "FolderAvg_tOF": sum(of) / len(of) if of else float("nan")})
    return r
