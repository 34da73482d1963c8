"""Time the tOF evaluation of one sequence on the GPU: the seeded 41-frame 576x720 sequence of tools/bench_lpips.py
(calendar's length and HR size) already on the device, frames 2..38 evaluated as metrics.py does.  Each evaluated frame
after the first costs two Farneback flows (target pair and result pair) on the whole frame and the crop_8x8 reduction;
every frame is expanded once per pyramid level and serves both pairs it belongs to.

  python tools/bench_tof.py --out DIR [--host-only]

Prints and writes DIR/tof_bench.json: the card's name and power limit read in the same run, ms per evaluated frame from
CUDA events over --repeats timed passes (after one warm-up pass), and the per-kernel split of one separate pass under
torch.profiler.  If cv2 is importable, cv2.calcOpticalFlowFarneback's host time per evaluated frame (two flows, the
reference's parameters) on the first --cv2-frames frames is reported beside it.  --host-only skips the GPU and times
cv2 alone, on frames drawn the same way from the CPU generator (same distribution, different values)."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def frames(n, H, W, device):
    gen = torch.Generator(device=device).manual_seed(0)
    T = torch.randint(0, 256, (n, H, W, 3), generator=gen, device=device, dtype=torch.int32)
    R = (T + torch.randint(-12, 13, T.shape, generator=gen, device=device, dtype=torch.int32)).clamp_(0, 255)
    return T.to(torch.uint8), R.to(torch.uint8)


def cv2_ms_per_frame(T, R, count):
    """Host time of the reference's per-frame tOF work (two cvtColor pairs are negligible; two flows dominate)."""
    try:
        import cv2
    except ImportError:
        return None
    t, r = T.cpu().numpy(), R.cpu().numpy()
    grey = lambda a: cv2.cvtColor(np.ascontiguousarray(a), cv2.COLOR_RGB2GRAY)    # noqa: E731
    gt, gr = [grey(a) for a in t[:count + 1]], [grey(a) for a in r[:count + 1]]
    cv2.calcOpticalFlowFarneback(gt[0], gt[1], None, 0.5, 3, 15, 3, 5, 1.2, 0)     # warm-up
    t0 = time.perf_counter()
    for i in range(1, count + 1):
        cv2.calcOpticalFlowFarneback(gt[i - 1], gt[i], None, 0.5, 3, 15, 3, 5, 1.2, 0)
        cv2.calcOpticalFlowFarneback(gr[i - 1], gr[i], None, 0.5, 3, 15, 3, 5, 1.2, 0)
    return {"cv2_version": cv2.__version__, "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count(),
            "frames_timed": count, "ms_per_frame": (time.perf_counter() - t0) * 1e3 / count}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--frames", type=int, default=41)
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=720)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cv2-frames", type=int, default=4)
    ap.add_argument("--host-only", action="store_true")
    args = ap.parse_args()
    n, H, W, cut = args.frames, args.height, args.width, 2
    res = {"frame": [H, W], "frames_evaluated": n - 2 * cut}
    if args.host_only:
        T, R = frames(n, H, W, "cpu")
        res["cv2_host"] = cv2_ms_per_frame(T[cut:], R[cut:], args.cv2_frames)
    else:
        if not torch.cuda.is_available():
            sys.exit("bench_tof.py needs a GPU (or --host-only)")
        from tecogan_b200 import tof as TOF
        torch.cuda.set_device(0)
        T, R = frames(n, H, W, "cuda")
        ts, rs = T[cut:n - cut], R[cut:n - cut]
        tof_frames = n - 2 * cut - 1

        def run():
            return TOF.tof_sequence(ts, rs)

        run()                                   # warm-up: module load, allocator, first launches
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
                m = re.search(r"\w+_kernel", ev.name)
                name = m.group(0) if m else ev.name[:60]
                split[name] = split.get(name, 0.0) + ev.device_time
        kernel_us = sum(split.values())
        res.update({"gpu": card(), "tof_frames": tof_frames, "repeats": args.repeats,
                    "ms_per_frame_median": float(np.median(ms)) / tof_frames, "ms_per_frame_min": min(ms) / tof_frames,
                    "ms_per_frame_runs": [m / tof_frames for m in ms],
                    "profiled_kernel_ms_per_frame": {k: v / 1000.0 / tof_frames
                                                     for k, v in sorted(split.items(), key=lambda kv: -kv[1])},
                    "profiled_kernel_share": {k: v / kernel_us for k, v in split.items()},
                    "cv2_host": cv2_ms_per_frame(ts, rs, args.cv2_frames)})
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "tof_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
