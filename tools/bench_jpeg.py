"""JPEG encode on the device (tecogan_b200.jpeg) against cv2.imencode('.jpg') on the host, for the same seeded frames.

  python tools/bench_jpeg.py [--reps 30] [--out results/bench_jpeg.json]

Prints the card's name, power limit and max SM clock, then per frame (seeded smooth frames at 576x720, 1080x1920 and
2160x3840, and a uniform-noise frame at 1080x1920, the most expensive content): the device encode (CUDA events around
the encoder's launches, warmed, median of --reps) alternating with cv2.imencode on the host, encode_jpeg including its
copies back, and a per-kernel split from a separate torch.profiler run.  The bytes are asserted equal.  Then the wall
time of `main.py --mode inference` with --output_ext jpg and png, alternating, on seeded 41-frame sequences of 144x180
and 270x480.
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


def device_vs_cv2(frame, rgb, reps):
    """(device ms per encode, cv2 ms per encode) lists, the two alternating."""
    from tecogan_b200 import _ffi, jpeg
    jpeg.encode_jpeg(frame)
    st = jpeg._state
    h, w = frame.shape[:2]
    args = lambda: (_ffi.ptr(frame), h, w, _ffi.ptr(st["ws"]), st["ws"].numel(), _ffi.ptr(st["out"]), st["out"].numel(),
                    _ffi.ptr(st["n"]), _ffi.stream_ptr())
    bgr = np.ascontiguousarray(rgb[:, :, ::-1])
    for _ in range(5):
        _ffi.call("teco_jpeg_encode_rgb8", *args())
        cv2.imencode(".jpg", bgr)
    dev, host = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _ffi.call("teco_jpeg_encode_rgb8", *args())
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
        t = time.perf_counter()
        cv2.imencode(".jpg", bgr)
        host.append((time.perf_counter() - t) * 1e3)
    return dev, host


def stage_split(frame):
    from tecogan_b200 import jpeg
    from torch.profiler import ProfilerActivity, profile
    jpeg.encode_jpeg(frame)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            jpeg.encode_jpeg(frame)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(jpeg_\w+)", e.key)
        if m:
            out[m.group(1)] = round(out.get(m.group(1), 0) + e.device_time_total / 10.0, 2)     # us per frame
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
        assert len(os.listdir(os.path.join(d, "out"))) == n
        return wall


def run():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from tests.png_cases import noise, smooth
    from tecogan_b200.jpeg import encode_jpeg
    res = {"card": card(), "frames": {}}
    print("card:", res["card"])
    frames = [("smooth", h, w, smooth(h, w, 3)) for h, w in ((576, 720), (1080, 1920), (2160, 3840))]
    frames.append(("noise", 1080, 1920, noise(1080, 1920, 4)))
    for kind, h, w, rgb in frames:
        fr = torch.from_numpy(rgb).cuda()
        dev, host = device_vs_cv2(fr, rgb, a.reps)
        t = time.perf_counter()
        for _ in range(10):
            data = encode_jpeg(fr)
        api = (time.perf_counter() - t) / 10 * 1e3
        assert data == cv2.imencode(".jpg", np.ascontiguousarray(rgb[:, :, ::-1]))[1].tobytes()
        r = {"device_ms_median": float(np.median(dev)), "device_ms_min": float(np.min(dev)),
             "cv2_ms_median": float(np.median(host)), "cv2_ms_min": float(np.min(host)), "encode_jpeg_ms": api,
             "bytes": len(data), "stages_us": stage_split(fr)}
        key = "%s_%dx%d" % (kind, h, w)
        res["frames"][key] = r
        print(key, json.dumps(r))
    for h, w in ((144, 180), (270, 480)):
        for ext in ("jpg", "png", "jpg", "png"):
            wall = main_wall(ext, h, w)
            res.setdefault("main_wall_s", []).append({"lr": "%dx%d" % (h, w), "ext": ext, "s": round(wall, 2)})
            print("main.py inference %dx%d --output_ext %s: %.2f s" % (h, w, ext, wall))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    run()
