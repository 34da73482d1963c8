#!/usr/bin/env python
"""The scan of `dataPrepare.py --scene_threshold` (DESIGN.md section 4.14), measured.

  python tools/bench_data_scan.py [--frames 300] [--reps 3] [--out results/bench_data_scan.json]

Prints the card's name, power limit and SM clocks (nvidia-smi, in the same call), then:
  * kernel: teco_frame_sads_u8 alone on windows of halved frames, 540x960 (from a 1080p source) and 1080x1920 (from a
    2160p source): the window pass 1 uses (WINDOW_BYTES of source frames) and a 32-frame one, with the previous
    window's last frame as prev.  CUDA events over 200 launches replayed from one CUDA graph after 20 warm-up launches
    (tools/bench_y4m.py::timed); the bytes are the n + 1 distinct frames a window reads (each frame is loaded by two
    pairs, the second time most likely from L2), and that rate's fraction of the H100 SXM's 3.35 TB/s data-sheet HBM3
    bandwidth;
  * pass 1: scan_video on one seeded `--frames`-frame 1920x1080 MJPG video with a cut every 60 frames, against a loop
    that only calls cv2.VideoCapture.read on the same file, alternated `--reps` times; wall time and frames/s of each,
    and whether the scan found the planted cuts.  If the two times match, the device work hides under decoding.
Temporary files only.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_y4m as BY  # noqa: E402

SOURCE = (1080, 1920)
SHOT = 60
THRESHOLD = 10.0


def bench_kernel():
    from tecogan_b200 import data_prepare as D
    from tecogan_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(1)
    res = {}
    for h, w in [(540, 960), (1080, 1920)]:
        fb = 3 * h * w
        for n in sorted({max(1, D.WINDOW_BYTES // (3 * 2 * h * 2 * w)), 32}):
            frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
            prev = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
            out = torch.empty(n, dtype=torch.int64, device="cuda")
            r = BY.timed(lambda: K.frame_sads_u8(frames, prev, out), (n + 1) * fb)
            r["us_per_pair"] = round(r["us_per_frame"] / n, 2)
            r["us_per_window"] = r.pop("us_per_frame")
            res["frame_sads_u8 %d x %dx%d" % (n, h, w)] = r
            print("kernel %d x %dx%d: %s" % (n, h, w, json.dumps(r)), flush=True)
    return res


def write_video(path, n, seed):
    """n seeded 1920x1080 MJPG frames: smooth noise drifting (1, 2) pixels a frame, a new texture every SHOT frames."""
    h, w = SOURCE
    g = np.random.default_rng(seed)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 25, (w, h))
    for k in range(n):
        j = k % SHOT
        if j == 0:
            small = g.integers(0, 256, ((h + 2 * SHOT) // 16 + 1, (w + 2 * SHOT) // 16 + 1, 3)).astype(np.uint8)
            base = cv2.resize(small, (w + 2 * SHOT, h + 2 * SHOT), interpolation=cv2.INTER_CUBIC)
            base = base // 2 + (128 if (k // SHOT) % 2 else 0)
        vw.write(base[j:j + h, 2 * j:2 * j + w])
    vw.release()
    return path


def read_only(path):
    cam = cv2.VideoCapture(path)
    n = 0
    while cam.read()[0]:
        n += 1
    cam.release()
    return n


def bench_pass1(frames, reps):
    from tecogan_b200 import data_prepare as D
    dev = torch.device("cuda", torch.cuda.current_device())
    with tempfile.TemporaryDirectory() as tmp:
        path = write_video(os.path.join(tmp, "v.avi"), frames, seed=7)
        warm = write_video(os.path.join(tmp, "warm.avi"), 8, seed=3)
        D.scan_video(warm, dev)                  # module loads, pinned and device buffers, the first launches
        read_only(warm)
        runs = {"cv2_read_only": [], "scan_video": []}
        cuts = None
        for rep in range(reps):
            t0 = time.perf_counter()
            n = read_only(path)
            runs["cv2_read_only"].append({"wall_s": round(time.perf_counter() - t0, 3), "frames": n})
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sads, values = D.scan_video(path, dev)
            wall = time.perf_counter() - t0     # scan_video ends with a synchronise of its stream
            scores = D.frame_scores(sads, values)
            cuts = [i for i, s in enumerate(scores) if i > 0 and s >= THRESHOLD]
            runs["scan_video"].append({"wall_s": round(wall, 3), "frames": len(sads), "sm_clock_after": BY.sm_clock()})
            for k in runs:
                runs[k][-1]["fps"] = round(runs[k][-1]["frames"] / runs[k][-1]["wall_s"], 1)
            print("pass 1 rep %d: %s" % (rep, json.dumps({k: v[-1] for k, v in runs.items()})), flush=True)
    med = {k: float(np.median([r["wall_s"] for r in v])) for k, v in runs.items()}
    return {"video": "%d x %dx%d MJPG, a cut every %d frames" % (frames, SOURCE[1], SOURCE[0], SHOT), "runs": runs,
            "median_wall_s": med, "scan_over_read": round(med["scan_video"] / med["cv2_read_only"], 3),
            "planted_cuts_found": cuts == list(range(SHOT, frames, SHOT))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_data_scan: needs a CUDA device")
    res = {"card": BY.card()}
    print("card:", res["card"], flush=True)
    res["kernel"] = bench_kernel()
    res["pass1"] = bench_pass1(a.frames, a.reps)
    print("pass 1: %s" % json.dumps({k: v for k, v in res["pass1"].items() if k != "runs"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
