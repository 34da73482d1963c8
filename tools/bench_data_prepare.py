#!/usr/bin/env python
"""Time the training-data preparation on seeded generated videos (mp4v, 1920x1080 and 3840x2160 sources, a few scenes
each), in one run:
  * dataPrepare.py's main() in a subprocess of its own with this table (CUDA start-up included), wall time per output
    frame; and prepare() again in this process, once CUDA is initialised;
  * teco_area_half_u8 alone, CUDA events over repeated launches on one window of decoded frames, per frame;
  * the reference's loop restated on the host (a seek before every frame, cv2.resize INTER_AREA, cv2.imwrite), wall
    time per output frame, and its files compared with the command's by SHA-256.
Everything is written under a temporary directory; prints one JSON line (with the card's name and power limit).

    python tools/bench_data_prepare.py [--duration 30] [--threads 4] [--out results.json]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {"1080p": (1920, 1080), "2160p": (3840, 2160)}
STARTS = [0, 40, 80]                   # three scenes per video


def write_video(path, w, h, n, seed):
    import cv2
    import numpy as np
    g = np.random.default_rng(seed)
    base = cv2.resize(g.integers(0, 256, ((h + 64) // 8, (w + 64) // 8, 3)).astype(np.uint8), (w + 64, h + 64),
                      interpolation=cv2.INTER_CUBIC)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 25, (w, h))
    for i in range(n):
        vw.write(base[(3 * i) % 64:(3 * i) % 64 + h, (5 * i) % 64:(5 * i) % 64 + w])
    vw.release()


def reference_loop(path, out, start_id, starts, duration):
    import cv2
    for k, start in enumerate(starts):
        d = os.path.join(out, "scene_%04d/" % (start_id + k))
        os.makedirs(d)
        cam = cv2.VideoCapture(path)
        for i in range(duration):
            cam.set(1, i + start)
            ok, f = cam.read()
            assert ok, (path, i + start)
            cv2.imwrite(d + "col_high_%04d.png" % i,
                        cv2.resize(f, (0, 0), fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA))
        cam.release()


def digests(root):
    res = {}
    for r, _, fs in os.walk(root):
        for n in fs:
            if n.endswith(".png"):
                with open(os.path.join(r, n), "rb") as f:
                    res[os.path.relpath(os.path.join(r, n), root)] = hashlib.sha256(f.read()).hexdigest()
    return res


def kernel_ms_per_frame(w, h, n=8, reps=50):
    import torch
    from tecogan_b200 import kernels as K
    frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((n, K.area_half_size(h), K.area_half_size(w), 3), dtype=torch.uint8, device="cuda")
    for _ in range(5):
        K.area_half(frames, swap_rb=True, out=out)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        K.area_half(frames, swap_rb=True, out=out)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps / n
    return ms, 3 * h * w * 1.25 / (ms * 1e-3) / 1e9      # bytes read + written (a quarter of the read) per second


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--duration", type=int, default=30)
    ap.add_argument("--threads", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    res = {"gpu": torch.cuda.get_device_name(0)}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit"] = "unknown"
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "src")
        os.makedirs(src)
        for k, (vid, (w, h)) in enumerate(SIZES.items()):
            write_video(os.path.join(src, vid + ".mp4"), w, h, STARTS[-1] + a.duration + 5, k)
        for vid, (w, h) in SIZES.items():
            disk = os.path.join(tmp, "disk_" + vid)
            os.makedirs(disk)
            os.symlink(os.path.join(src, vid + ".mp4"), os.path.join(disk, vid + ".mp4"))
            t = time.perf_counter()
            argv = ["--disk_path", disk, "--duration", str(a.duration), "--threads", str(a.threads)]
            code = "import dataPrepare; dataPrepare.main(%r, videos={%r: %r})" % (argv, vid, STARTS)
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
            t_cmd = time.perf_counter() - t
            assert r.returncode == 0, r.stderr[-2000:]
            ref = os.path.join(tmp, "ref_" + vid)
            t = time.perf_counter()
            reference_loop(os.path.join(src, vid + ".mp4"), ref, 2000, STARTS, a.duration)
            t_ref = time.perf_counter() - t
            got, want = digests(disk), digests(ref)
            from tecogan_b200 import data_prepare
            disk2 = os.path.join(tmp, "inproc_" + vid)
            os.makedirs(disk2)
            os.symlink(os.path.join(src, vid + ".mp4"), os.path.join(disk2, vid + ".mp4"))
            t = time.perf_counter()
            data_prepare.prepare({vid: STARTS}, disk2, 2000, a.duration, threads=a.threads)
            t_in = time.perf_counter() - t
            k_ms, k_gbs = kernel_ms_per_frame(w, h)
            n = len(STARTS) * a.duration
            res["%dx%d" % (w, h)] = {
                "frames": n, "command_ms_per_frame": 1e3 * t_cmd / n, "prepare_in_process_ms_per_frame": 1e3 * t_in / n,
                "reference_loop_ms_per_frame": 1e3 * t_ref / n, "kernel_ms_per_frame": k_ms,
                "kernel_GBps": k_gbs, "files_identical": got == want and len(got) == n}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
