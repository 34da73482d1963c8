"""The inference input read on the device (tecogan_b200.lib.dataloader.inference_data_loader: PNG decode, then
teco_frames_to_f32 or teco_gauss_blur_down4) against the host formula it replaced, restated below as the baseline.

  python tools/bench_inference_input.py [--reps 3] [--out results/bench_inference_input.json]

Prints the card's name and power limit, then, on seeded PNG sequences written by cv2.imwrite (smooth frames with noise)
-- 41 x 144x180 LR, 41 x 576x720 HR, 24 x 1080x1920 HR:
  * the loader end to end (files to resident float32 CUDA frames), against the baseline: cv.imread(name, 3), astype,
    cv.GaussianBlur for HR, / 255 on one host thread, then each frame uploaded from pageable memory as the per-frame loop
    of main.py did -- alternated in each rep, median of the reps; both must give identical frames;
  * for the HR sizes, teco_gauss_blur_down4 alone on the whole sequence in one launch (CUDA events, 20 launches);
  * the wall time of `main.py --mode inference --input_dir_HR` on the 576x720 sequence (num_resblock 16, random
    weights, PNG output), with the loader and with the baseline patched in; the written files must be identical.
Temporary files only.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import png_cases as PC  # noqa: E402

SEQS = [("lr", 144, 180, 41), ("hr", 576, 720, 41), ("hr", 1080, 1920, 24)]

# main.py with the baseline loader patched in: argv[1:] are main.py's arguments
HOST_MAIN = """
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import torch
import main as M
import bench_inference_input as B
from tecogan_b200.lib import dataloader as DL
DL.read_inputs = lambda paths, down: [torch.from_numpy(a) for a in B.host_formula(paths, down)]
M.main(sys.argv[1:])
"""


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def write_frames(d, h, w, n, seed):
    os.makedirs(d, exist_ok=True)
    g = np.random.default_rng(seed)
    base = PC.smooth(h, w + 3 * n, seed).astype(np.int64)
    for k in range(n):
        f = np.clip(base[:, 3 * k:3 * k + w] + g.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(d, "%04d.png" % (k + 1)), np.ascontiguousarray(f[:, :, ::-1]))
    return d


def host_formula(paths, down):
    """The parent's loader: reference lib/dataloader.py:38-43 on the host, one frame at a time."""
    out = []
    for name in paths:
        im = cv2.imread(name, 3).astype(np.float32)[:, :, ::-1]
        if down:
            im = cv2.GaussianBlur(im, (0, 0), sigmaX=1.5)[::4, ::4, ::]
        out.append(np.ascontiguousarray(im / 255.0))
    return out


def baseline(paths, down):
    """host_formula, then each frame uploaded as main.py's per-frame loop did (np.array([frame]) -> .cuda())."""
    return [torch.from_numpy(np.array([im]).astype(np.float32)).cuda()[0] for im in host_formula(paths, down)]


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t) * 1e3


def bench_loader(d, down, reps):
    from tecogan_b200.lib.dataloader import read_inputs
    paths = sorted(os.path.join(d, f) for f in os.listdir(d))
    dev, host = read_inputs(paths, down), baseline(paths, down)       # warm-up, and the identity check
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(dev, host)), "frames differ"
    del dev, host
    t_dev, t_host = [], []
    for _ in range(reps):
        t_dev.append(timed(lambda: read_inputs(paths, down))[1])
        t_host.append(timed(lambda: baseline(paths, down))[1])
    return {"loader_ms": float(np.median(t_dev)), "baseline_ms": float(np.median(t_host)),
            "speedup": float(np.median(t_host) / np.median(t_dev))}


def bench_kernel(d):
    from tecogan_b200 import kernels as K
    from tecogan_b200.png import decode_png
    paths = sorted(os.path.join(d, f) for f in os.listdir(d))
    frames = torch.stack(decode_png(paths))
    K.gauss_blur_down4(frames)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        K.gauss_blur_down4(frames)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 20
    n, h, w, _ = frames.shape
    # bytes a perfect kernel moves: every input byte read once, every output float written once
    nbytes = frames.numel() + n * ((h + 3) // 4) * ((w + 3) // 4) * 3 * 4
    return {"kernel_ms": ms, "kernel_us_per_frame": ms * 1e3 / n, "min_bytes_GBps": nbytes / ms / 1e6}


def bench_main(d, tmp, reps):
    args = ["--mode", "inference", "--checkpoint", "random:5", "--num_resblock", "16", "--input_dir_HR", d,
            "--output_pre", "", "--output_ext", "png", "--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")]
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    host = py + ["-c", HOST_MAIN % (ROOT, os.path.join(ROOT, "tools"))]
    dev = py + [os.path.join(ROOT, "main.py")]
    t = {"device": [], "baseline": []}
    for r in range(reps):
        for key, cmd in (("device", dev), ("baseline", host)):
            out = os.path.join(tmp, "main_%s_%d" % (key, r))
            t0 = time.perf_counter()
            p = subprocess.run(cmd + args + ["--output_dir", out], capture_output=True, text=True, cwd=tmp)
            t[key].append(time.perf_counter() - t0)
            assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    a, b = os.path.join(tmp, "main_device_0"), os.path.join(tmp, "main_baseline_0")
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)) and names
    assert all(open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read() for n in names)
    return {"main_device_s": float(np.median(t["device"])), "main_baseline_s": float(np.median(t["baseline"])),
            "files": len(names)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inference_input: needs a CUDA device")
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for kind, h, w, n in SEQS:
            d = write_frames(os.path.join(tmp, "%s_%dx%d" % (kind, h, w)), h, w, n, seed=h + w)
            r = bench_loader(d, kind == "hr", a.reps)
            if kind == "hr":
                r.update(bench_kernel(d))
            key = "%s %dx%d x%d" % (kind, h, w, n)
            res[key] = r
            print("%s: %s" % (key, json.dumps({k: round(v, 3) for k, v in r.items()})), flush=True)
        r = bench_main(os.path.join(tmp, "hr_576x720"), tmp, max(1, a.reps - 1))
        res["main.py --input_dir_HR 41 x 576x720"] = r
        print("main.py --input_dir_HR 41 x 576x720: %s" % json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
