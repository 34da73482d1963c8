"""PNG encode on the device (tecogan_b200.png) against cv2.imencode on the host, for the same seeded smooth frames.

  python tools/bench_png.py [--reps 50] [--out results/bench_png.json]

Prints the card's name and power limit, then per frame size: the device encode (CUDA events around the encoder's
launches, warmed, median of --reps), encode_png including the copy back, cv2.imencode, and a per-kernel split from a
separate torch.profiler run.  Then the wall time of `main.py --mode inference --output_ext png` (and jpg, the default)
on seeded 41-frame sequences of 144x180 and 270x480.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def device_encode_ms(frame, reps):
    from tecogan_b200 import _ffi, png
    png.encode_png(frame)
    st = png._state
    h, w = frame.shape[:2]
    args = lambda: (_ffi.ptr(frame), h, w, _ffi.ptr(st["ws"]), st["ws"].numel(), _ffi.ptr(st["out"]), st["out"].numel(),
                    _ffi.ptr(st["n"]), _ffi.stream_ptr())
    for _ in range(5):
        _ffi.call("teco_png_encode_rgb8", *args())
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _ffi.call("teco_png_encode_rgb8", *args())
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def stage_split(frame):
    from tecogan_b200 import png
    from torch.profiler import ProfilerActivity, profile
    png.encode_png(frame)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            png.encode_png(frame)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(png_\w+)", e.key)
        if m:
            out[m.group(1)] = round(e.device_time_total / 10.0, 2)     # us per frame
    return out


def main_wall(ext, h, w, n=41):
    with tempfile.TemporaryDirectory() as d:
        from tests.png_cases import smooth
        p = os.path.join(d, "LR")
        os.makedirs(p)
        base = smooth(h + 48, w + 48, 1)
        for i in range(n):
            cv2.imwrite(os.path.join(p, "%04d.png" % (i + 1)), base[i:i + h, i:i + w][:, :, ::-1])
        cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--mode", "inference", "--checkpoint", "random:1",
               "--input_dir_LR", p, "--output_dir", os.path.join(d, "out"), "--output_ext", ext]
        t = time.time()
        r = subprocess.run(cmd, cwd=d, capture_output=True, text=True)
        wall = time.time() - t
        assert r.returncode == 0, r.stderr[-2000:]
        return wall


def run():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from tests.png_cases import smooth
    from tecogan_b200.png import encode_png
    res = {"card": card(), "sizes": {}}
    print("card:", res["card"])
    for h, w in ((576, 720), (1080, 1920), (2160, 3840)):
        rgb = smooth(h, w, 3)
        fr = torch.from_numpy(rgb).cuda()
        med, best = device_encode_ms(fr, a.reps)
        t = time.perf_counter()
        for _ in range(10):
            data = encode_png(fr)
        api = (time.perf_counter() - t) / 10 * 1e3
        bgr = np.ascontiguousarray(rgb[:, :, ::-1])
        t = time.perf_counter()
        for _ in range(5):
            ref = cv2.imencode(".png", bgr)[1].tobytes()
        host = (time.perf_counter() - t) / 5 * 1e3
        assert data == ref
        r = {"device_ms_median": med, "device_ms_min": best, "encode_png_ms": api, "cv2_ms": host,
             "bytes": len(data), "stages_us": stage_split(fr)}
        res["sizes"]["%dx%d" % (h, w)] = r
        print("%dx%d" % (h, w), json.dumps(r))
    for h, w in ((144, 180), (270, 480)):
        for ext in ("png", "jpg", "png", "jpg"):
            wall = main_wall(ext, h, w)
            res.setdefault("main_wall_s", []).append({"lr": "%dx%d" % (h, w), "ext": ext, "s": round(wall, 2)})
            print("main.py inference %dx%d --output_ext %s: %.2f s" % (h, w, ext, wall))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    run()
