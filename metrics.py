#!/usr/bin/env python
"""Mirror of the reference's metrics.py command line (flags --output / --results / --targets, metrics.py:9-12), computed on
the GPU: PSNR and SSIM on the Y channel (tecogan_b200/metrics.py: teco_metrics_psnr_y_u8 / teco_metrics_ssim_y_u8) and,
with --lpips_alexnet and --lpips_lin, LPIPS and tLP100 (tecogan_b200/lpips.py: AlexNet and the LPIPS v0.1 head in CUDA).
Same frame selection (cutfr = 2, metrics.py:117,131), same cut of the result to the target size (:134-135), same crop_8x8
(:171-172), same per-frame / per-folder / total printout and metrics.csv layout (:205-242) restricted to
keys = ["PSNR", "SSIM"], plus "LPIPS" and "tLP100" with the two LPIPS flags and "tOF" with --tof, in the reference's
order PSNR, SSIM, LPIPS, tOF, tLP100.  Each folder's frames are decoded once, on the device (read_folder), and run
through AlexNet once; tLP100 reuses the previous frame's features.  With --tof all the folder's Farneback flows
(tecogan_b200/tof.py) run as one batch; the per-frame line then carries "tOF %02.2f, " before psnr, as the reference prints it.  Without
--tof nothing about the output changes.  Unlike the reference, which fails there, a result smaller than its target is
compared on the area the two share, for tOF as for the other metrics.

  python metrics.py --output results/metric_log/ --results results/calendar --targets HR/calendar [--tof] \
      [--lpips_alexnet ~/.cache/torch/hub/checkpoints/alexnet-owt-7be5be79.pth --lpips_lin LPIPSmodels/v0.1/alex.pth]
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

KEYS = ["PSNR", "SSIM"]
KEYS_LPIPS = ["PSNR", "SSIM", "LPIPS", "tLP100"]
CUTFR = 2


def listPNGinDir(dirpath):
    """metrics.py:28-35: *.png, not starting with IB, ordered by the digits in the name."""
    names = sorted(n for n in os.listdir(dirpath) if n.endswith(".png") and not n.startswith("IB"))
    names.sort(key=lambda f: int(''.join(filter(str.isdigit, f)) or -1))
    return [os.path.join(dirpath, n) for n in names]


def read_rgb(path):
    try:
        import cv2
        return np.ascontiguousarray(cv2.imread(path)[:, :, ::-1])
    except ImportError:
        from PIL import Image
        return np.ascontiguousarray(np.asarray(Image.open(path).convert("RGB")))


def metric_keys(lpips, tof):
    """The reference's key order (metrics.py:120) restricted to what is computed."""
    return KEYS + (["LPIPS"] if lpips else []) + (["tOF"] if tof else []) + (["tLP100"] if lpips else [])


def read_folder(paths):
    """[H, W, 3] uint8 RGB CUDA tensors of the PNG files at `paths`: decoded on the device in byte-bounded batches
    (tecogan_b200/png.py::decode_png), with read_rgb for the files the device does not take."""
    from tecogan_b200.png import decode_png
    return decode_png(paths, host_decode=read_rgb)


def folder_tof(tars, outs):
    """tOF list of one scene's decoded frames cutfr .. n-cutfr-1 (one shorter than PSNR's): all flows in one batch on
    the common area of result and target."""
    import torch
    from tecogan_b200 import tof as TOF
    if not tars:
        return []
    for name, frames in (("target", tars), ("result", outs)):
        if len({tuple(f.shape) for f in frames}) != 1:
            raise ValueError("tOF: the %s frames of one folder differ in size" % name)
    return TOF.tof_sequence(torch.stack(tars), torch.stack(outs))


def evaluate_folder(result_dir, target_dir, log=print, lpips=None, tof=False):
    """Per-frame lists of one scene (frames cutfr .. n-cutfr-1): PSNR / SSIM, LPIPS / tLP100 when `lpips` (a
    tecogan_b200.lpips.LPIPS model) is given, and tOF with tof=True.  The previous frame's target and result features
    are kept for tLP100."""
    import torch
    from tecogan_b200 import metrics as M
    result, target = listPNGinDir(result_dir), listPNGinDir(target_dir)
    lists = {k: [] for k in metric_keys(lpips is not None, tof)}
    idx = list(range(CUTFR, len(target) - CUTFR))
    frames = read_folder([target[i] for i in idx] + [result[i] for i in idx])   # every frame decoded once
    tars, outs = frames[:len(idx)], frames[len(idx):]
    tof_all = folder_tof(tars, outs) if tof else None
    prev = None
    for n, i in enumerate(idx):
        t, o = tars[n], outs[n]
        tar, out = t.shape, o.shape
        msg = "frame %d, tar %s, out %s, " % (i, str(tuple(tar)), str(tuple(out)))
        if tof and i > CUTFR:                     # metrics.py:143-169
            lists["tOF"].append(tof_all[i - CUTFR - 1])
            msg += "tOF %02.2f, " % lists["tOF"][-1]
        ps, ss = M.frame_metrics(t, o)            # window = crop_8x8 of the common area; no cropped copies
        win = M.crop_window(min(tar[0], out[0]), min(tar[1], out[1]))
        lists["PSNR"].append(ps[0])
        lists["SSIM"].append(ss[0])
        log(result[i])
        msg += "psnr %02.2f, ssim %02.2f" % (ps[0], ss[0])
        if lpips is not None:                     # metrics.py:183-202
            feats = lpips.features([t, o], win)   # target at 0, result at 1
            lists["LPIPS"].append(lpips.distances(feats, feats, [(0, 1)])[0])
            msg += ", lpips %02.2f" % lists["LPIPS"][-1]
            if prev is not None:
                d_tar, d_out = lpips.distances(prev, feats, [(0, 0), (1, 1)])
                lists["tLP100"].append(100.0 * abs(d_tar - d_out))
                msg += ", tLPx100 %02.2f" % lists["tLP100"][-1]
            prev = feats
        log(msg + ", crop (%d, %d)" % win[:2])
    return lists


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--output", required=True, help="the path of output directory")
    ap.add_argument("--results", required=True, help="the list of paths of result directory")
    ap.add_argument("--targets", required=True, help="the list of paths of target directory")
    ap.add_argument("--lpips_alexnet", default=None,
                    help="torchvision ImageNet AlexNet state dict (alexnet-owt-*.pth); with --lpips_lin adds LPIPS and tLP100")
    ap.add_argument("--lpips_lin", default=None, help="LPIPS v0.1 linear weights (LPIPSmodels/v0.1/alex.pth)")
    ap.add_argument("--tof", action="store_true", help="also compute tOF (Farneback optical flow on the GPU)")
    F = ap.parse_args(argv)
    if (F.lpips_alexnet is None) != (F.lpips_lin is None):
        ap.error("--lpips_alexnet and --lpips_lin go together: give both for LPIPS / tLP100, or neither")
    lpips = None
    if F.lpips_alexnet is not None:
        from tecogan_b200.lpips import LPIPS
        lpips = LPIPS(F.lpips_alexnet, F.lpips_lin)
    keys = metric_keys(lpips is not None, F.tof)
    import pandas as pd
    os.makedirs(F.output, exist_ok=True)
    logf = open(os.path.join(F.output, "metricsfile.txt"), "a")

    def log(m):
        print(m)
        logf.write(m + "\n")
    result_list, target_list = F.results.split(','), F.targets.split(',')
    folder_n = len(result_list)
    sum_d = {"FrameAvg_" + k: 0.0 for k in keys}
    len_d = {k: 0 for k in keys}
    avg_d = {"Avg_" + k: [] for k in keys}
    folder_d = {"FolderAvg_" + k: 0.0 for k in keys}
    csv = os.path.join(F.output, "metrics.csv")
    for fi in range(folder_n):
        lists = evaluate_folder(result_list[fi], target_list[fi], log, lpips, F.tof)
        pd_dict = {}
        for k in keys:
            cur = np.float32(lists[k])
            pd_dict["%s_%02d" % (k, fi)] = pd.Series(cur)
            mean = cur.sum() / cur.shape[0]
            log("%s_%02d, max %02.4f, min %02.4f, avg %02.4f" % (k, fi, cur.max(), cur.min(), mean))
            avg_d["Avg_" + k].append(mean)
            sum_d["FrameAvg_" + k] += cur.sum()
            len_d[k] += cur.shape[0]
            folder_d["FolderAvg_" + k] += mean
        pd.DataFrame(pd_dict).to_csv(csv, mode='w' if fi == 0 else 'a')
    for k in keys:
        sum_d["FrameAvg_" + k] = pd.Series([sum_d["FrameAvg_" + k] / len_d[k]])
        folder_d["FolderAvg_" + k] = pd.Series([folder_d["FolderAvg_" + k] / folder_n])
        avg_d["Avg_" + k] = pd.Series(np.float32(avg_d["Avg_" + k]))
        log("%s, total frame %d, total avg %02.4f, folder avg %02.4f" % (k, len_d[k], sum_d["FrameAvg_" + k][0], folder_d["FolderAvg_" + k][0]))
    for d in (avg_d, folder_d, sum_d):
        pd.DataFrame(d).to_csv(csv, mode='a')
    log("Finished.")
    logf.close()
    return {k: float(sum_d["FrameAvg_" + k][0]) for k in keys}


if __name__ == "__main__":
    main()
