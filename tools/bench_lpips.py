"""Time the LPIPS + tLP100 evaluation of one sequence on the GPU: a seeded 41-frame 576x720 sequence (calendar's length and
HR size) already on the device, frames 2..38 evaluated as metrics.py does (crop_8x8 -> 544x704).  Each evaluated frame
costs one AlexNet pass for the target, one for the result and three head evaluations (LPIPS, and the two distances of
tLP100 from the second frame on).  Backbone: the seeded test weights (tests/golden/lpips_oracle.py); the arithmetic and its
cost do not depend on the values.

  python tools/bench_lpips.py --out DIR

Prints and writes DIR/lpips_bench.json: the card's name and power limit read in the same run, ms per evaluated frame
from CUDA events over --repeats timed passes (after one warm-up pass), and the per-kernel split of one separate pass
under torch.profiler (conv1 .. conv5 are told apart by launch order: features() launches them in that order)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.golden.lpips_oracle import lpips_test_weights  # noqa: E402
from tecogan_b200 import metrics as M  # noqa: E402
from tecogan_b200.lpips import LPIPS, feature_sizes  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def macs_per_image(h, w):
    sz, cin, k = feature_sizes(h, w), (3, 64, 192, 384, 256), (11, 5, 3, 3, 3)
    cout = (64, 192, 384, 256, 256)
    return sum(sz[l][0] * sz[l][1] * cout[l] * cin[l] * k[l] * k[l] for l in range(5))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--frames", type=int, default=41)
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--width", type=int, default=720)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lpips.py needs a GPU")
    torch.cuda.set_device(0)
    g = np.load(os.path.join(ROOT, "tests", "golden", "lpips.npz"))
    lin = {"lin%d.model.1.weight" % l: torch.from_numpy(g["lin%d" % l]).reshape(1, -1, 1, 1) for l in range(5)}
    model = LPIPS(lpips_test_weights(1), lin)
    gen = torch.Generator(device="cuda").manual_seed(0)
    n, H, W = args.frames, args.height, args.width
    T = torch.randint(0, 256, (n, H, W, 3), generator=gen, device="cuda", dtype=torch.int32)
    R = (T + torch.randint(-12, 13, T.shape, generator=gen, device="cuda", dtype=torch.int32)).clamp_(0, 255)
    T, R = T.to(torch.uint8), R.to(torch.uint8)
    cut = 2
    win = M.crop_window(H, W)
    ts, rs = T[cut:n - cut], R[cut:n - cut]
    frames = n - 2 * cut

    def run():
        return model.sequence(ts, rs, win)

    run()                                       # warm-up: module load, buffers, first launches
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
    evs = sorted((ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0),
                 key=lambda ev: ev.time_range.start)
    split, nconv, npool = {}, 0, 0
    for ev in evs:
        if "conv2d_f32_kernel" in ev.name:
            key, nconv = "conv%d" % (nconv % 5 + 1), nconv + 1
        elif "maxpool3s2_kernel" in ev.name:
            key, npool = "pool%d" % (npool % 2 + 1), npool + 1
        elif "lpips_head_kernel" in ev.name:
            key = "head"
        elif "lpips_input_kernel" in ev.name:
            key = "input"
        else:
            key = "other: " + ev.name[:60]
        split[key] = split.get(key, 0.0) + ev.device_time
    kernel_us = sum(split.values())
    macs = macs_per_image(win[2], win[3])
    best = min(ms) / frames
    res = {"gpu": card(), "frames_evaluated": frames, "frame": [H, W], "crop": list(win[2:]), "repeats": args.repeats,
           "ms_per_frame_median": float(np.median(ms)) / frames, "ms_per_frame_min": best,
           "ms_per_frame_runs": [m / frames for m in ms],
           "alexnet_gflop_per_frame": 2 * 2 * macs / 1e9,
           "alexnet_tflops_at_min": 2 * 2 * macs / (best * 1e-3) / 1e12,
           "profiled_kernel_ms_per_frame": {k: v / 1000.0 / frames for k, v in sorted(split.items(), key=lambda kv: -kv[1])},
           "profiled_kernel_share": {k: v / kernel_us for k, v in split.items()}}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "lpips_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
